// The pool of call contexts behind every entry point that takes no handle (call_context.h).
#include "call_context.h"
#include "vbx_plan.h"

#include <memory>
#include <mutex>
#include <vector>

namespace fa {

int CallContext::init(int worker_lim) {
    FA_CUDA_TRY(cudaGetDevice(&device));
    int st = stream.create();
    for (auto &e : ev)
        if (st == FA_OK) st = e.create();
    if (st == FA_OK) st = vbx::set_smem_limits();
    if (st == FA_OK) st = solver.init(stream, worker_lim);
    if (st != FA_OK) return st;
    worker_limit = worker_lim;
    ready = true;
    return FA_OK;
}

static std::mutex g_pool_mutex;
static std::vector<std::unique_ptr<CallContext>> g_pool;   // idle contexts

struct Lease {
    std::unique_ptr<CallContext> ctx;
    int status = FA_OK;
    explicit Lease(int worker_limit) {
        int dev = 0;
        const cudaError_t e = cudaGetDevice(&dev);
        if (e != cudaSuccess) {
            status = cuda_failure(e, "cudaGetDevice", __FILE__, __LINE__);
            return;
        }
        {
            std::lock_guard<std::mutex> lock(g_pool_mutex);
            for (size_t i = 0; i < g_pool.size(); ++i)
                if (g_pool[i]->device == dev && g_pool[i]->worker_limit == worker_limit) {
                    ctx = std::move(g_pool[i]);
                    g_pool.erase(g_pool.begin() + i);
                    break;
                }
        }
        if (!ctx) {
            ctx.reset(new CallContext());
            status = ctx->init(worker_limit);
        }
    }
    ~Lease() {
        if (ctx && ctx->ready && status != FA_CUDA_ERROR) {
            std::lock_guard<std::mutex> lock(g_pool_mutex);
            g_pool.push_back(std::move(ctx));
        }
    }
};

int with_context(int worker_limit, const std::function<int(CallContext &)> &body) {
    Lease lease(worker_limit);
    if (lease.status != FA_OK) return lease.status;
    lease.status = body(*lease.ctx);
    return lease.status;
}

} // namespace fa
