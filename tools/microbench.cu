// microbench.cu - dependent-chain latencies of the scalar fp64 / shared-memory / shuffle operations the plan
// search is made of.  One warp, clock64 around an unrolled chain; prints cycles per operation.
// Build: nvcc -gencode arch=compute_90a,code=sm_90a -O3 -fmad=false -o microbench tools/microbench.cu ; run on the
// GPU.  Not part of the product.
#include <cuda_runtime.h>
#include <stdio.h>
#include <stdint.h>

constexpr int N = 4096;

__global__ void k_dadd(double *out, double a, double b, long long *cyc) {
    double x = a;
    const long long t0 = clock64();
#pragma unroll 64
    for (int i = 0; i < N; ++i) x = x - b;
    const long long t1 = clock64();
    if (threadIdx.x == 0) { *cyc = t1 - t0; }
    out[threadIdx.x] = x;
}

__global__ void k_cmpsub(double *out, double a, double b, long long *cyc) {
    double x = a;
    int n = 0;
    const long long t0 = clock64();
#pragma unroll 64
    for (int i = 0; i < N; ++i) { if (x > b) { x = x - b; ++n; } }
    const long long t1 = clock64();
    if (threadIdx.x == 0) { *cyc = t1 - t0; }
    out[threadIdx.x] = x + n;
}

__global__ void k_dmul(double *out, double a, double b, long long *cyc) {
    double x = a;
    const long long t0 = clock64();
#pragma unroll 64
    for (int i = 0; i < N; ++i) x = x * b;
    const long long t1 = clock64();
    if (threadIdx.x == 0) { *cyc = t1 - t0; }
    out[threadIdx.x] = x;
}

__global__ void k_ddiv(double *out, double a, double b, long long *cyc) {
    double x = a;
    const long long t0 = clock64();
#pragma unroll 16
    for (int i = 0; i < N / 8; ++i) x = x / b;
    const long long t1 = clock64();
    if (threadIdx.x == 0) { *cyc = (t1 - t0) * 8; }
    out[threadIdx.x] = x;
}

__global__ void k_d2i(double *out, double a, long long *cyc) {
    double x = a;
    const long long t0 = clock64();
#pragma unroll 64
    for (int i = 0; i < N; ++i) x = (double)((int)x) + 0.5;
    const long long t1 = clock64();
    if (threadIdx.x == 0) { *cyc = t1 - t0; }     // D2I + I2D + DADD
    out[threadIdx.x] = x;
}

__global__ void k_lds(int *out, long long *cyc) {
    __shared__ int chain[1024];
    for (int i = threadIdx.x; i < 1024; i += 32) chain[i] = (i * 37 + 11) & 1023;
    __syncwarp();
    int p = threadIdx.x;
    const long long t0 = clock64();
#pragma unroll 64
    for (int i = 0; i < N; ++i) p = chain[p];
    const long long t1 = clock64();
    if (threadIdx.x == 0) { *cyc = t1 - t0; }
    out[threadIdx.x] = p;
}

__global__ void k_lds64_dadd(double *out, long long *cyc) {
    __shared__ double v[1024];
    for (int i = threadIdx.x; i < 1024; i += 32) v[i] = 1.0 / (i + 3);
    __syncwarp();
    double f = 0.0;
    const long long t0 = clock64();
#pragma unroll 32
    for (int i = 0; i < N; ++i) f = f + v[i & 1023];       // address independent of data: loads can run ahead
    const long long t1 = clock64();
    if (threadIdx.x == 0) { *cyc = t1 - t0; }
    out[threadIdx.x] = f;
}

__global__ void k_neumaier(double *out, long long *cyc) {
    __shared__ double v[1024];
    for (int i = threadIdx.x; i < 1024; i += 32) v[i] = 1.0 / (i + 3);
    __syncwarp();
    double f = 0.0, c = 0.0;
    const long long t0 = clock64();
#pragma unroll 16
    for (int i = 0; i < N; ++i) {
        const double x = v[i & 1023];
        const double t = f + x;
        if (fabs(f) >= fabs(x)) c += (f - t) + x; else c += (x - t) + f;
        f = t;
    }
    const long long t1 = clock64();
    if (threadIdx.x == 0) { *cyc = t1 - t0; }
    out[threadIdx.x] = f + c;
}

__global__ void k_shfl(int *out, long long *cyc) {
    int p = threadIdx.x;
    const long long t0 = clock64();
#pragma unroll 64
    for (int i = 0; i < N; ++i) p = __shfl_sync(0xFFFFFFFFu, p, (p + 1) & 31);
    const long long t1 = clock64();
    if (threadIdx.x == 0) { *cyc = t1 - t0; }
    out[threadIdx.x] = p;
}

__global__ void k_ballot(int *out, long long *cyc) {
    unsigned p = threadIdx.x;
    const long long t0 = clock64();
#pragma unroll 64
    for (int i = 0; i < N; ++i) p = __ballot_sync(0xFFFFFFFFu, (p >> (threadIdx.x & 7)) & 1) + i;
    const long long t1 = clock64();
    if (threadIdx.x == 0) { *cyc = t1 - t0; }
    out[threadIdx.x] = p;
}

__global__ void k_syncwarp_sts_lds(int *out, long long *cyc) {
    __shared__ int box[64];
    int p = threadIdx.x;
    const long long t0 = clock64();
#pragma unroll 16
    for (int i = 0; i < N; ++i) {                  // lane hand-over through shared memory: store, syncwarp, load
        box[threadIdx.x] = p;
        __syncwarp();
        p = box[(threadIdx.x + 1) & 31] + 1;
        __syncwarp();
    }
    const long long t1 = clock64();
    if (threadIdx.x == 0) { *cyc = t1 - t0; }
    out[threadIdx.x] = p;
}

__global__ void k_iadd(int *out, int a, long long *cyc) {
    int x = a;
    const long long t0 = clock64();
#pragma unroll 64
    for (int i = 0; i < N; ++i) x = (x + a) ^ i;
    const long long t1 = clock64();
    if (threadIdx.x == 0) { *cyc = t1 - t0; }
    out[threadIdx.x] = x;
}

// throughput: W warps per block of dependent DADD chains, one block per SM
__global__ void k_dadd_tput(double *out, double a, double b, long long *cyc) {
    double x = a + threadIdx.x;
    __syncthreads();
    const long long t0 = clock64();
#pragma unroll 64
    for (int i = 0; i < N; ++i) x = x - b;
    const long long t1 = clock64();
    if (threadIdx.x == 0 && blockIdx.x == 0) { *cyc = t1 - t0; }
    out[blockIdx.x * blockDim.x + threadIdx.x] = x;
}

int main() {
    double *dout; int *iout; long long *cyc, h;
    int sms = 0;
    cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, 0);
    cudaMalloc(&dout, 8 * 1024 * sms); cudaMalloc(&iout, 4 * 1024); cudaMalloc(&cyc, 8);
#define RUN(name, call, per)                                                         \
    for (int rep = 0; rep < 2; ++rep) { call; cudaDeviceSynchronize(); }             \
    cudaMemcpy(&h, cyc, 8, cudaMemcpyDeviceToHost);                                  \
    printf("%-28s %8.2f cycles/op  (%s)\n", name, (double)h / (per), cudaGetErrorString(cudaGetLastError()));
    RUN("DADD dependent", (k_dadd<<<1, 32>>>(dout, 1e9, 1.25, cyc)), N);
    RUN("DSETP+DADD (if x>b x-=b)", (k_cmpsub<<<1, 32>>>(dout, 1e9, 1.25, cyc)), N);
    RUN("DMUL dependent", (k_dmul<<<1, 32>>>(dout, 1.0, 1.0000001, cyc)), N);
    RUN("DDIV dependent", (k_ddiv<<<1, 32>>>(dout, 1.0, 1.0000001, cyc)), N);
    RUN("D2I+I2D+DADD", (k_d2i<<<1, 32>>>(dout, 12345.25, cyc)), N);
    RUN("LDS pointer chase", (k_lds<<<1, 32>>>(iout, cyc)), N);
    RUN("LDS.64 + DADD (addr indep)", (k_lds64_dadd<<<1, 32>>>(dout, cyc)), N);
    RUN("Neumaier step (LDS+4 DADD)", (k_neumaier<<<1, 32>>>(dout, cyc)), N);
    RUN("SHFL dependent", (k_shfl<<<1, 32>>>(iout, cyc)), N);
    RUN("BALLOT dependent", (k_ballot<<<1, 32>>>(iout, cyc)), N);
    RUN("STS+syncwarp+LDS+syncwarp", (k_syncwarp_sts_lds<<<1, 32>>>(iout, cyc)), N);
    RUN("IADD+LOP dependent", (k_iadd<<<1, 32>>>(iout, 3, cyc)), N);
    for (int w = 1; w <= 32; w *= 2) {
        char name[64]; snprintf(name, sizeof(name), "DADD chain x %2d warps/SM", w);
        RUN(name, (k_dadd_tput<<<sms, 32 * w>>>(dout, 1e9, 1.25, cyc)), N);
    }
    return 0;
}
