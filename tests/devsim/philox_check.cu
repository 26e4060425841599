// philox_check.cu - TEST-ONLY: the device Philox4x32-10 of metis_noise.cuh next to curand's curand_Philox4x32_10 on
// the same counters and keys.  Compiled with the library's nvcc flags and loaded only by tests/test_profile_noise.py.
#include <cuda_runtime.h>
#include <curand_philox4x32_x.h>

#include <cstdint>

#include "../../metis_b200/csrc/metis_noise.cuh"

__global__ void philox_pair_kernel(const uint32_t *ctr, const uint32_t *key, uint32_t *ours, uint32_t *theirs, int n) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const metis::Philox4 r = metis::philox4x32_10(
        metis::Philox4{{ctr[4 * i], ctr[4 * i + 1], ctr[4 * i + 2], ctr[4 * i + 3]}}, key[2 * i], key[2 * i + 1]);
    const uint4 c = curand_Philox4x32_10(make_uint4(ctr[4 * i], ctr[4 * i + 1], ctr[4 * i + 2], ctr[4 * i + 3]),
                                         make_uint2(key[2 * i], key[2 * i + 1]));
    for (int k = 0; k < 4; ++k) ours[4 * i + k] = r.v[k];
    theirs[4 * i] = c.x;
    theirs[4 * i + 1] = c.y;
    theirs[4 * i + 2] = c.z;
    theirs[4 * i + 3] = c.w;
}

// n counters (4 words each) and keys (2 words each), host pointers; 0, or the CUDA error code
extern "C" int philox_check(const uint32_t *ctr, const uint32_t *key, uint32_t *ours, uint32_t *theirs, int n) {
    uint32_t *d = nullptr;
    const size_t words = (size_t)n * 14;
    cudaError_t e = cudaMalloc(&d, words * sizeof(uint32_t));
    if (e != cudaSuccess) return (int)e;
    uint32_t *dc = d, *dk = d + 4 * (size_t)n, *dours = dk + 2 * (size_t)n, *dtheirs = dours + 4 * (size_t)n;
    cudaMemcpy(dc, ctr, 4 * (size_t)n * sizeof(uint32_t), cudaMemcpyHostToDevice);
    cudaMemcpy(dk, key, 2 * (size_t)n * sizeof(uint32_t), cudaMemcpyHostToDevice);
    philox_pair_kernel<<<(n + 127) / 128, 128>>>(dc, dk, dours, dtheirs, n);
    cudaMemcpy(ours, dours, 4 * (size_t)n * sizeof(uint32_t), cudaMemcpyDeviceToHost);
    e = cudaMemcpy(theirs, dtheirs, 4 * (size_t)n * sizeof(uint32_t), cudaMemcpyDeviceToHost);
    cudaFree(d);
    return (int)e;
}
