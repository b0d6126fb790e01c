// Microbenchmark of the AHC scan step's instruction schedule: 128 threads of one CTA, each a sequential chain
// sum = sum + (x_k - v_k)^2 over D = 256 with x in a k-major shared-memory tile (stride SP) and v broadcast — the loop
// of ahc_merge_kernel — in several source forms.  Reports cycles per element (clock64, one SM).
// nvcc -gencode arch=compute_90a,code=sm_90a -O3 -o scan_sched scan_sched.cu && ./scan_sched
#include <cstdio>
#include <cuda_runtime.h>
constexpr int D = 256, SP = 112, kReps = 16;
__device__ __forceinline__ double sq_step(double sum, double a, double b) {
    const double diff = __dsub_rn(a, b);
    return __dadd_rn(sum, __dmul_rn(diff, diff));
}
template <int kMode>
__global__ void __launch_bounds__(128) scan(const double *g, double *out, long long *cycles) {
    extern __shared__ double sm[];
    double *sv = sm;              // [D x SP]
    double *v = sm + D * SP;      // [D]
    for (int i = threadIdx.x; i < D * SP; i += 128) sv[i] = g[i % 4096] * 1e-3;
    for (int i = threadIdx.x; i < D; i += 128) v[i] = g[i] * 2e-3;
    __syncthreads();
    const double *col = sv + (threadIdx.x % SP);
    double total = 0.0;
    const long long t0 = clock64();
#pragma unroll 1
    for (int rep = 0; rep < kReps; ++rep) {
        double sum = 0.0;
        if (kMode == 0) {   // the kernel's form: eight loads, eight steps
            for (int k = 0; k + 8 <= D; k += 8) {
                double x[8];
#pragma unroll
                for (int u = 0; u < 8; ++u) x[u] = col[(k + u) * SP];
#pragma unroll
                for (int u = 0; u < 8; ++u) sum = sq_step(sum, x[u], v[k + u]);
            }
        } else if (kMode == 1) {   // explicit software pipeline: p one element ahead, d two ahead
            double d = __dsub_rn(col[SP], v[1]);
            double d0 = __dsub_rn(col[0], v[0]);
            double p = __dmul_rn(d0, d0);
#pragma unroll 8
            for (int k = 0; k < D - 2; ++k) {
                sum = __dadd_rn(sum, p);
                p = __dmul_rn(d, d);
                d = __dsub_rn(col[(k + 2) * SP], v[k + 2]);
            }
            sum = __dadd_rn(sum, p);
            sum = __dadd_rn(sum, __dmul_rn(d, d));
        } else if (kMode == 2) {   // same, the three instructions of a step pinned in one asm statement
            double d = __dsub_rn(col[SP], v[1]);
            double d0 = __dsub_rn(col[0], v[0]);
            double p = __dmul_rn(d0, d0);
#pragma unroll 8
            for (int k = 0; k < D - 2; ++k) {
                const double xn = col[(k + 2) * SP], vn = v[k + 2];
                asm volatile("add.rn.f64 %0, %0, %1;\n\tmul.rn.f64 %1, %2, %2;\n\tsub.rn.f64 %2, %3, %4;"
                             : "+d"(sum), "+d"(p), "+d"(d) : "d"(xn), "d"(vn));
            }
            sum = __dadd_rn(sum, p);
            sum = __dadd_rn(sum, __dmul_rn(d, d));
        } else if (kMode == 3) {   // sixteen loads, sixteen steps
            for (int k = 0; k + 16 <= D; k += 16) {
                double x[16];
#pragma unroll
                for (int u = 0; u < 16; ++u) x[u] = col[(k + u) * SP];
#pragma unroll
                for (int u = 0; u < 16; ++u) sum = sq_step(sum, x[u], v[k + u]);
            }
        } else if (kMode == 4) {   // squares of a block of eight first, then the eight chain adds (upper bound of bad)
            for (int k = 0; k + 8 <= D; k += 8) {
                double p[8];
#pragma unroll
                for (int u = 0; u < 8; ++u) { const double d = __dsub_rn(col[(k + u) * SP], v[k + u]); p[u] = __dmul_rn(d, d); }
#pragma unroll
                for (int u = 0; u < 8; ++u) sum = __dadd_rn(sum, p[u]);
            }
        } else {   // squares one BLOCK ahead: while the chain eats block b, the side work of block b+1 fills the pipe
            double p[8], q[8];
#pragma unroll
            for (int u = 0; u < 8; ++u) { const double d = __dsub_rn(col[u * SP], v[u]); p[u] = __dmul_rn(d, d); }
            for (int k = 8; k + 8 <= D; k += 8) {
#pragma unroll
                for (int u = 0; u < 8; ++u) {
                    sum = __dadd_rn(sum, p[u]);
                    const double d = __dsub_rn(col[(k + u) * SP], v[k + u]);
                    q[u] = __dmul_rn(d, d);
                }
#pragma unroll
                for (int u = 0; u < 8; ++u) p[u] = q[u];
            }
#pragma unroll
            for (int u = 0; u < 8; ++u) sum = __dadd_rn(sum, p[u]);
        }
        total += sum;
    }
    const long long t1 = clock64();
    out[threadIdx.x] = total;
    if (threadIdx.x == 0) cycles[0] = t1 - t0;
}
int main() {
    double *g, *out; long long *cyc;
    cudaMalloc(&g, 4096 * 8); cudaMalloc(&out, 1024); cudaMalloc(&cyc, 8);
    double h[4096]; for (int i = 0; i < 4096; ++i) h[i] = 1.0 + (i % 97) * 1e-2;
    cudaMemcpy(g, h, sizeof(h), cudaMemcpyHostToDevice);
    const size_t smem = (size_t)(D * SP + D) * 8;
    const char *names[6] = {"kernel form (8 loads, 8 steps)", "software pipeline in source", "pipeline, asm-pinned triple",
                            "16 loads, 16 steps", "8 squares then 8 adds", "squares one block ahead"};
    auto run = [&](int mode) {
        void (*f)(const double *, double *, long long *) = mode == 0 ? scan<0> : mode == 1 ? scan<1> : mode == 2 ? scan<2> : mode == 3 ? scan<3> : mode == 4 ? scan<4> : scan<5>;
        cudaFuncSetAttribute(f, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
        long long hc = 0;
        for (int rep = 0; rep < 2; ++rep) { f<<<1, 128, smem>>>(g, out, cyc); cudaDeviceSynchronize(); }
        cudaMemcpy(&hc, cyc, 8, cudaMemcpyDeviceToHost);
        printf("%-36s %6.2f cycles per element  (%s)\n", names[mode], (double)hc / (kReps * D), cudaGetErrorString(cudaGetLastError()));
    };
    for (int m = 0; m < 6; ++m) run(m);
    return 0;
}
