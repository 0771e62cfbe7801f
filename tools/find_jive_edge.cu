// find_jive_edge.cu — searches for an RpJive64_256 merge input whose Jive sum (rpj_compress, rpjive.cuh) reaches the window of
// its last add: x + y in [p, 2^64), with x = in[i] + in[4 + i] and y = out[i] + out[4 + i] (both reduced). There the sum needs
// canonicalising without having wrapped 2^64. Both operands come from the same permutation input, so the window cannot be aimed at
// backwards; about 2^31 inputs are tried (seconds on one GPU). The input found is a test vector of tests/test_gpu_hash_edges.py.
// Build: nvcc -gencode arch=compute_90a,code=sm_90a -O3 -std=c++17 -o find_jive_edge tools/find_jive_edge.cu
// Run on a GPU: prints the 8 input words, the lane and x + y as one JSON line.
#include <cuda_runtime.h>
#include <stdint.h>
#include <stdio.h>

#include "../winterfell_b200/csrc/rpjive.cuh"

__device__ __forceinline__ void base_state(u64 t, u64 s[8]) {   // a fixed canonical state, word 0 = the trial counter
    s[0] = t;
#pragma unroll
    for (int k = 1; k < 8; k++) s[k] = 0x9e3779b97f4a7c15ULL * (k + 1) % GL_P;
}

__global__ void search(u64 t0, unsigned long long* found) {
    const u64 t = t0 + (u64)blockIdx.x * blockDim.x + threadIdx.x;
    u64 in[8], s[8];
    base_state(t, in);
#pragma unroll
    for (int k = 0; k < 8; k++) s[k] = in[k];
    rpj_permute(s);
#pragma unroll
    for (int i = 0; i < 4; i++) {
        const u64 x = gl_add(in[i], in[4 + i]), y = gl_add(s[i], s[4 + i]);
        if (x + y >= x && x + y >= GL_P) atomicMin(found, (unsigned long long)t << 2 | i);
    }
}

int main() {
    unsigned long long* d;
    cudaMalloc(&d, 8);
    unsigned long long h = ~0ULL;
    const u64 chunk = 1ULL << 28;
    for (u64 t0 = 1; t0 < (1ULL << 36) && h == ~0ULL; t0 += chunk) {
        cudaMemcpy(d, &h, 8, cudaMemcpyHostToDevice);
        search<<<(unsigned)(chunk / 256), 256>>>(t0, d);
        cudaMemcpy(&h, d, 8, cudaMemcpyDeviceToHost);
        if (cudaGetLastError() != cudaSuccess) { printf("{\"error\": \"launch\"}\n"); return 1; }
    }
    cudaFree(d);
    if (h == ~0ULL) { printf("{\"found\": false}\n"); return 1; }
    const u64 t = h >> 2;
    u64 in[8];
    in[0] = t;
    for (int k = 1; k < 8; k++) in[k] = 0x9e3779b97f4a7c15ULL * (k + 1) % GL_P;
    printf("{\"found\": true, \"lane\": %llu, \"input\": [", h & 3);
    for (int k = 0; k < 8; k++) printf("%s%llu", k ? ", " : "", (unsigned long long)in[k]);
    printf("]}\n");
    return 0;
}
