// DMMA (mma.sync m8n8k4.f64 and m16n8k16.f64) throughput micro-benchmark used to decide between DFMA and DMMA kernels:
//   nvcc -gencode arch=compute_90a,code=sm_90a -O3 -DTRY_M16 -o scripts/mb/dmma_bench scripts/mb/dmma.cu
#include <cstdio>
#include <cuda_runtime.h>
__device__ __forceinline__ void dmma884(double& c0, double& c1, double a, double b) {
    asm volatile("mma.sync.aligned.m8n8k4.row.col.f64.f64.f64.f64 {%0,%1}, {%2}, {%3}, {%0,%1};" : "+d"(c0), "+d"(c1) : "d"(a), "d"(b));
}
template <int NACC>
__global__ void __launch_bounds__(256) k_dmma(double* out, int iters) {
    double c[NACC][2];
    for (int i = 0; i < NACC; ++i) c[i][0] = c[i][1] = 0.0;
    double a = threadIdx.x * 1e-9, b = 1.0000001;
    for (int it = 0; it < iters; ++it) {
#pragma unroll
        for (int i = 0; i < NACC; ++i) dmma884(c[i][0], c[i][1], a, b);
    }
    double s = 0; for (int i = 0; i < NACC; ++i) s += c[i][0] + c[i][1];
    out[blockIdx.x * blockDim.x + threadIdx.x] = s;
}
#ifdef TRY_M16
__device__ __forceinline__ void dmma16816(double (&c)[4], const double (&a)[8], const double (&b)[4]) {
    asm volatile("mma.sync.aligned.m16n8k16.row.col.f64.f64.f64.f64 {%0,%1,%2,%3}, {%4,%5,%6,%7,%8,%9,%10,%11}, {%12,%13,%14,%15}, {%0,%1,%2,%3};"
       : "+d"(c[0]), "+d"(c[1]), "+d"(c[2]), "+d"(c[3]) : "d"(a[0]),"d"(a[1]),"d"(a[2]),"d"(a[3]),"d"(a[4]),"d"(a[5]),"d"(a[6]),"d"(a[7]),"d"(b[0]),"d"(b[1]),"d"(b[2]),"d"(b[3]));
}
template <int NACC>
__global__ void __launch_bounds__(256) k_dmma16(double* out, int iters) {
    double c[NACC][4];
    for (int i = 0; i < NACC; ++i) for (int j = 0; j < 4; ++j) c[i][j] = 0.0;
    double a[8], b[4];
    for (int j = 0; j < 8; ++j) a[j] = threadIdx.x * 1e-9 + j;
    for (int j = 0; j < 4; ++j) b[j] = 1.0000001 + j;
    for (int it = 0; it < iters; ++it) {
#pragma unroll
        for (int i = 0; i < NACC; ++i) dmma16816(c[i], a, b);
    }
    double s = 0; for (int i = 0; i < NACC; ++i) for (int j = 0; j < 4; ++j) s += c[i][j];
    out[blockIdx.x * blockDim.x + threadIdx.x] = s;
}
#endif
template <class F> float timeit(F f) { cudaEvent_t a, b; cudaEventCreate(&a); cudaEventCreate(&b); f(); cudaDeviceSynchronize(); float best = 1e30; for (int r = 0; r < 3; ++r) { cudaEventRecord(a); f(); cudaEventRecord(b); cudaEventSynchronize(b); float ms; cudaEventElapsedTime(&ms, a, b); if (ms < best) best = ms; } return best; }
int main() {
    int sms = 0;
    cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, 0);
    double* out; cudaMalloc(&out, (size_t)sms * 4 * 256 * 8);  // largest grid below: 4 CTAs of 256 threads per SM
    const int iters = 4096;
    for (int bps : {1, 2, 4}) {
        int blocks = sms * bps;
        float ms = timeit([&] { k_dmma<8><<<blocks, 256>>>(out, iters); });
        printf("m8n8k4 NACC=8 blocks/SM=%d: %.2f TFLOP/s\n", bps, 2.0 * 256 * 8 * iters * (double)blocks * 8 / ms / 1e9);
        ms = timeit([&] { k_dmma<1><<<blocks, 256>>>(out, iters); });
        printf("m8n8k4 NACC=1 (dependent) blocks/SM=%d: %.2f TFLOP/s; cycles/dmma at 1.965GHz = %.1f\n", bps, 2.0 * 256 * 1 * iters * (double)blocks * 8 / ms / 1e9, ms * 1e-3 * 1.965e9 / iters);
        ms = timeit([&] { k_dmma<16><<<blocks, 256>>>(out, iters); });
        printf("m8n8k4 NACC=16 blocks/SM=%d: %.2f TFLOP/s\n", bps, 2.0 * 256 * 16 * iters * (double)blocks * 8 / ms / 1e9);
#ifdef TRY_M16
        ms = timeit([&] { k_dmma16<4><<<blocks, 256>>>(out, iters); });
        printf("m16n8k16 NACC=4 blocks/SM=%d: %.2f TFLOP/s\n", bps, 2.0 * 16 * 8 * 16 * 4 * iters * (double)blocks * 8 / ms / 1e9);
#endif
    }
    printf("err %s\n", cudaGetErrorString(cudaGetLastError()));
}
