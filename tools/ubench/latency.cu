// dependent-load latency microbenchmark for sm_90a: one warp follows a random cycle of indices, every lane at the
// same address (a warp-uniform field, as in the pair kernel's resolve turn), through one kind of load at a time;
// SM cycles and ns per load reported.
//
//   nvcc -O3 -gencode arch=compute_90a,code=sm_90a -o tools/ubench/latency tools/ubench/latency.cu
//
//   generic param   LD.E of a __grid_constant__ parameter through its generic address (a `const ScanParams &`)
//   LDC param       the same field read from the constant bank (the parameter indexed directly)
//   LDS             shared memory
//   LDG L2          global memory, ld.global.cg (L1 bypassed), one 128-byte line per step, the chain resident in L2
//   LDG L1          global memory, ld.global.ca, a chain that fits L1
#include <cstdio>
#include <cstdint>
#include <vector>
#include <cuda_runtime.h>

constexpr int kParamN = 128;               // 512 B of indices in the parameter block
constexpr int kIters = 4096;
constexpr uint32_t kL2Lines = 1u << 16;    // 8 MiB of 128-byte lines: past L1, inside the 50 MB L2
constexpr uint32_t kL1Lines = 256;         // 32 KiB
struct Chain { uint32_t next[kParamN]; };

__device__ __forceinline__ uint32_t ld_generic(const uint32_t *a) {
    uint32_t v;
    asm volatile("ld.u32 %0, [%1];" : "=r"(v) : "l"(a));
    return v;
}
__device__ __forceinline__ uint32_t ld_cg(const uint32_t *a) {
    uint32_t v;
    asm volatile("ld.global.cg.u32 %0, [%1];" : "=r"(v) : "l"(a));
    return v;
}
__device__ __forceinline__ uint32_t ld_ca(const uint32_t *a) {
    uint32_t v;
    asm volatile("ld.global.ca.u32 %0, [%1];" : "=r"(v) : "l"(a));
    return v;
}
__device__ __forceinline__ unsigned long long global_ns() {
    unsigned long long t;
    asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t));
    return t;
}

template <int KIND>
__device__ __forceinline__ uint32_t step(const Chain &c, const uint32_t *s, const uint32_t *g, uint32_t j) {
    if (KIND == 0) return ld_generic(&c.next[j]);
    if (KIND == 1) return c.next[j];
    if (KIND == 2) { uint32_t v; asm volatile("ld.shared.u32 %0, [%1];" : "=r"(v) : "r"((uint32_t)__cvta_generic_to_shared(s + j))); return v; }
    if (KIND == 3) return ld_cg(g + j);
    return ld_ca(g + j);
}

template <int KIND>
__global__ void chase(const __grid_constant__ Chain c, const uint32_t *g, unsigned long long *res, uint32_t *sink) {
    __shared__ uint32_t s[kParamN];
    for (int i = threadIdx.x; i < kParamN; i += blockDim.x) s[i] = c.next[i];
    __syncthreads();
    uint32_t j = 0;
    for (int it = 0; it < kIters; it++) j = step<KIND>(c, s, g, j);     // warm-up lap: the same addresses as below
    asm volatile("mov.u32 %0, 0;" : "=r"(j));                          // back to the start (opaque to the compiler)
    __syncwarp();
    const unsigned long long c0 = clock64(), t0 = global_ns();
    for (int it = 0; it < kIters; it++) j = step<KIND>(c, s, g, j);
    const unsigned long long c1 = clock64(), t1 = global_ns();
    sink[threadIdx.x] = j;
    if (threadIdx.x == 0) { res[0] = c1 - c0; res[1] = t1 - t0; }
}

// a random cyclic permutation of 0..n-1 (Sattolo), scaled by `mul` (word index of the next element)
static std::vector<uint32_t> cycle(uint32_t n, uint32_t mul, uint64_t seed) {
    std::vector<uint32_t> perm(n);
    for (uint32_t i = 0; i < n; i++) perm[i] = i;
    for (uint32_t i = n - 1; i > 0; i--) {
        seed = seed * 6364136223846793005ull + 1442695040888963407ull;
        const uint32_t k = (uint32_t)((seed >> 33) % i);
        const uint32_t t = perm[i]; perm[i] = perm[k]; perm[k] = t;
    }
    std::vector<uint32_t> next((size_t)n * mul, 0);
    for (uint32_t i = 0; i < n; i++) next[(size_t)perm[i] * mul] = perm[(i + 1) % n] * mul;
    return next;
}

template <int KIND>
static void run(const char *name, const Chain &c, const uint32_t *g, unsigned long long *d_res, uint32_t *d_sink) {
    chase<KIND><<<1, 32>>>(c, g, d_res, d_sink);
    cudaDeviceSynchronize();
    chase<KIND><<<1, 32>>>(c, g, d_res, d_sink);
    cudaDeviceSynchronize();
    unsigned long long r[2] = {0, 0};
    cudaMemcpy(r, d_res, sizeof(r), cudaMemcpyDeviceToHost);
    printf("%-16s %7.1f cycles %7.1f ns per dependent load (%s)\n", name, (double)r[0] / kIters, (double)r[1] / kIters,
           cudaGetErrorString(cudaGetLastError()));
}

int main() {
    cudaDeviceProp prop;
    cudaGetDeviceProperties(&prop, 0);
    printf("%s, %d SMs\n", prop.name, prop.multiProcessorCount);
    Chain c;
    const std::vector<uint32_t> pc = cycle(kParamN, 1, 1);
    for (int i = 0; i < kParamN; i++) c.next[i] = pc[i];
    const std::vector<uint32_t> l2 = cycle(kL2Lines, 32, 2), l1 = cycle(kL1Lines, 32, 3);
    uint32_t *d_l2, *d_l1, *d_sink;
    unsigned long long *d_res;
    cudaMalloc(&d_l2, l2.size() * 4); cudaMalloc(&d_l1, l1.size() * 4); cudaMalloc(&d_sink, 32 * 4); cudaMalloc(&d_res, 16);
    cudaMemcpy(d_l2, l2.data(), l2.size() * 4, cudaMemcpyHostToDevice);
    cudaMemcpy(d_l1, l1.data(), l1.size() * 4, cudaMemcpyHostToDevice);
    run<0>("generic param", c, d_l2, d_res, d_sink);
    run<1>("LDC param", c, d_l2, d_res, d_sink);
    run<2>("LDS", c, d_l2, d_res, d_sink);
    run<3>("LDG L2 (.cg)", c, d_l2, d_res, d_sink);
    run<4>("LDG L1 (.ca)", c, d_l1, d_res, d_sink);
    cudaFree(d_l2); cudaFree(d_l1); cudaFree(d_sink); cudaFree(d_res);
    return 0;
}
