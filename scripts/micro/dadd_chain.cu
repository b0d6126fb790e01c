// Microbenchmark: latency of a dependent FP64 add chain on one SM, alone and with the scan's two independent FP64
// operations per step (d = x - v, p = d * d), at 1 / 2 / 4 warps per SM sub-partition.
// nvcc -gencode arch=compute_90a,code=sm_90a -O3 -o dadd_chain dadd_chain.cu && ./dadd_chain
#include <cstdio>
#include <cuda_runtime.h>
constexpr int kSteps = 4096;
template <int kMode>
__global__ void chain(const double *x, const double *v, double *out, long long *cycles) {
    __shared__ double xs[256], vs[256];
    for (int i = threadIdx.x; i < 256; i += blockDim.x) { xs[i] = x[i]; vs[i] = v[i]; }
    __syncthreads();
    double sum = x[threadIdx.x & 255];
    const long long t0 = clock64();
#pragma unroll 1
    for (int r = 0; r < kSteps / 256; ++r) {
#pragma unroll 8
        for (int k = 0; k < 256; ++k) {
            if (kMode == 0) {
                sum = __dadd_rn(sum, vs[k]);                       // chain only (operand from shared memory)
            } else if (kMode == 1) {
                const double d = __dadd_rn(xs[(k + threadIdx.x) & 255], -vs[k]);
                sum = __dadd_rn(sum, __dmul_rn(d, d));             // the scan's step
            } else if (kMode == 2) {
                sum = __fma_rn(sum, 1.0000000001, vs[k]);          // dependent DFMA chain
            } else {
                const float d = __fadd_rn((float)xs[(k + threadIdx.x) & 255], -(float)vs[k]);
                sum = __dadd_rn(sum, (double)__fmul_rn(d, d));     // FP32 side work: chain + conversions only
            }
        }
    }
    const long long t1 = clock64();
    out[blockIdx.x * blockDim.x + threadIdx.x] = sum;
    if (threadIdx.x == 0) cycles[blockIdx.x] = t1 - t0;
}
int main() {
    double *x, *v, *out; long long *cyc;
    cudaMalloc(&x, 2048); cudaMalloc(&v, 2048); cudaMalloc(&out, 8 * 1024 * 148); cudaMalloc(&cyc, 8 * 148);
    double h[256]; for (int i = 0; i < 256; ++i) h[i] = 1.0 + i * 1e-3;
    cudaMemcpy(x, h, 2048, cudaMemcpyHostToDevice); cudaMemcpy(v, h, 2048, cudaMemcpyHostToDevice);
    const char *names[4] = {"DADD chain", "scan step (DADD d, DMUL p, DADD chain)", "DFMA chain", "chain + FP32 side work"};
    for (int mode = 0; mode < 4; ++mode)
        for (int threads : {32, 128, 256, 512}) {
            long long hc = 0;
            for (int rep = 0; rep < 2; ++rep) {
                if (mode == 0) chain<0><<<1, threads>>>(x, v, out, cyc);
                if (mode == 1) chain<1><<<1, threads>>>(x, v, out, cyc);
                if (mode == 2) chain<2><<<1, threads>>>(x, v, out, cyc);
                if (mode == 3) chain<3><<<1, threads>>>(x, v, out, cyc);
                cudaDeviceSynchronize();
            }
            cudaMemcpy(&hc, cyc, 8, cudaMemcpyDeviceToHost);
            printf("%-44s %3d threads/SM: %6.2f cycles per step\n", names[mode], threads, (double)hc / kSteps);
        }
    return 0;
}
