// Device probe of fluidaudio_b200/csrc/fa_float.cuh for tests/test_gpu_float_rounding.py: evaluates f_exp, f_log or
// f_log1p on the H100 over a range of float32 bit patterns (or a list of them), and compares each result on the device
// with an uploaded reference.  Built for sm_90a by __graft_entry__.build() into tests/device/libfa_float_probe.so; the
// library itself never links it.
#include "../../fluidaudio_b200/csrc/fa_float.cuh"

#include <cuda_runtime.h>

#include <cmath>
#include <cstdint>

namespace {

// policy 0: the library's helper.  policy 1: the old (float)f((double)x), CUDA's float64 libm rounded once.
__device__ float eval(int fn, int policy, float x) {
    if (policy == 1) return (float)(fn == 0 ? exp((double)x) : fn == 1 ? log((double)x) : log1p((double)x));
    return fn == 0 ? fa::fp::f_exp(x) : fn == 1 ? fa::fp::f_log(x) : fa::fp::f_log1p(x);
}

__global__ void probe_kernel(int fn, int policy, uint64_t start, uint64_t count, const uint32_t *inputs,
                             const uint32_t *ref, uint32_t *out, uint32_t *bad, int cap, unsigned long long *n_bad) {
    for (uint64_t i = blockIdx.x * (uint64_t)blockDim.x + threadIdx.x; i < count; i += (uint64_t)gridDim.x * blockDim.x) {
        const uint32_t xb = inputs ? inputs[i] : (uint32_t)(start + i);
        const uint32_t g = __float_as_uint(eval(fn, policy, __uint_as_float(xb)));
        if (out) out[i] = g;
        if (!ref) continue;
        const uint32_t w = ref[i];
        if (g == w || (isnan(__uint_as_float(g)) && isnan(__uint_as_float(w)))) continue;
        const unsigned long long k = atomicAdd(n_bad, 1ull);
        if (k < (unsigned long long)cap) {
            bad[3 * k] = xb;
            bad[3 * k + 1] = g;
            bad[3 * k + 2] = w;
        }
    }
}

} // namespace

// Evaluates fn (0 exp, 1 log, 2 log1p) under policy at count inputs: inputs[0, count) when inputs is not null, else
// the bit patterns start .. start + count - 1.  Host arrays in and out; out (results) and ref (compared on the device,
// mismatches counted into *n_bad and the first cap written to bad as (input, got, expected)) may each be null.
// Returns 0, or the CUDA error.
extern "C" int fa_float_probe(int fn, int policy, uint64_t start, uint64_t count, const uint32_t *inputs,
                              const uint32_t *ref, uint32_t *out, uint32_t *bad, int cap, unsigned long long *n_bad) {
    uint32_t *d_in = nullptr, *d_ref = nullptr, *d_out = nullptr, *d_bad = nullptr;
    unsigned long long *d_n = nullptr;
    const size_t bytes = count * sizeof(uint32_t);
    cudaError_t e = cudaSuccess;
    auto step = [&](cudaError_t r) { if (e == cudaSuccess) e = r; };
    step(cudaMalloc(&d_n, sizeof(*d_n)));
    step(cudaMalloc(&d_bad, 3 * sizeof(uint32_t) * (cap > 0 ? cap : 1)));
    step(cudaMemset(d_n, 0, sizeof(*d_n)));
    if (inputs) step(cudaMalloc(&d_in, bytes)), step(cudaMemcpy(d_in, inputs, bytes, cudaMemcpyHostToDevice));
    if (ref) step(cudaMalloc(&d_ref, bytes)), step(cudaMemcpy(d_ref, ref, bytes, cudaMemcpyHostToDevice));
    if (out) step(cudaMalloc(&d_out, bytes));
    if (e == cudaSuccess && count > 0) {
        probe_kernel<<<132 * 16, 256>>>(fn, policy, start, count, d_in, d_ref, d_out, d_bad, cap, d_n);
        step(cudaGetLastError());
        step(cudaDeviceSynchronize());
    }
    if (out) step(cudaMemcpy(out, d_out, bytes, cudaMemcpyDeviceToHost));
    unsigned long long n = 0;
    step(cudaMemcpy(&n, d_n, sizeof(n), cudaMemcpyDeviceToHost));
    if (n_bad) *n_bad = n;
    if (bad && cap > 0 && n > 0)
        step(cudaMemcpy(bad, d_bad, 3 * sizeof(uint32_t) * (n < (unsigned long long)cap ? n : cap), cudaMemcpyDeviceToHost));
    cudaFree(d_in);
    cudaFree(d_ref);
    cudaFree(d_out);
    cudaFree(d_bad);
    cudaFree(d_n);
    return (int)e;
}
