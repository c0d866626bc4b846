// Diagnostic only: tiny "foreign" CUDA module used by tools/tune_k1_diag3.py to find out which property of another
// module loaded into the same context slows k_g1_validate_main (DESIGN.md, "foreign module effect").
#include <cassert>
#include <cstdio>
#include <cuda_runtime.h>
__global__ void k_plain(int* p) { p[threadIdx.x] = threadIdx.x; }
__global__ void k_assert(int* p) { assert(p != nullptr); p[threadIdx.x] = 1; }
__global__ void k_printf(int* p) { if (p == nullptr) printf("never\n"); else p[threadIdx.x] = 2; }
__global__ void k_malloc(int* p) { int* q = (int*)malloc(16); if (q) { q[0] = 3; p[threadIdx.x] = q[0]; free(q); } }
__global__ void k_lmem(int* p) {
    volatile int big[8192];  // 32 KiB of local memory per thread
    for (int i = 0; i < 8192; i++) big[i] = i + threadIdx.x;
    int s = 0; for (int i = 0; i < 8192; i += 97) s += big[i];
    p[threadIdx.x] = s;
}
__global__ void k_smem(int* p) { extern __shared__ int sh[]; sh[threadIdx.x] = threadIdx.x; __syncthreads(); p[threadIdx.x] = sh[31 - threadIdx.x]; }
extern "C" int foreign_run(int kind) {
    static int* d = nullptr;
    if (!d) cudaMalloc(&d, 4096);
    switch (kind) {
        case 0: k_plain<<<1, 32>>>(d); break;
        case 1: k_assert<<<1, 32>>>(d); break;
        case 2: k_printf<<<1, 32>>>(d); break;
        case 3: k_malloc<<<1, 32>>>(d); break;
        case 4: k_lmem<<<1, 32>>>(d); break;
        case 5: cudaFuncSetAttribute(k_smem, cudaFuncAttributeMaxDynamicSharedMemorySize, 200 * 1024);
                k_smem<<<1, 32, 200 * 1024>>>(d); break;
        case 6: { cudaStream_t s; cudaStreamCreate(&s); k_plain<<<1, 32, 0, s>>>(d); cudaStreamSynchronize(s); } break;
    }
    return (int)cudaDeviceSynchronize();
}
