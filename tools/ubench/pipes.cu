// instruction issue-rate microbenchmark for sm_90a: N independent chains of one PTX instruction per thread,
// 8 warps per SM sub-partition, cycles per warp-instruction per sub-partition reported.
#include <cstdio>
#include <cstdint>
#include <cuda_runtime.h>
#define ITERS 4096
#define CHAINS 8
template <int OP>
__global__ void k(uint32_t *out, uint32_t seed, unsigned long long *cyc) {
    uint32_t x[CHAINS];
    uint32_t y = seed | 1u, z = seed * 2654435761u | 1u;
#pragma unroll
    for (int i = 0; i < CHAINS; i++) x[i] = seed + i * 977u + threadIdx.x;
    unsigned long long t0 = clock64();
    for (int it = 0; it < ITERS; it++) {
#pragma unroll
        for (int i = 0; i < CHAINS; i++) {
            if (OP == 0) asm volatile("mul.lo.u32 %0, %0, %1;" : "+r"(x[i]) : "r"(y));
            if (OP == 1) asm volatile("mad.lo.u32 %0, %0, %1, %2;" : "+r"(x[i]) : "r"(y), "r"(z));
            if (OP == 2) asm volatile("mul.hi.u32 %0, %0, %1;" : "+r"(x[i]) : "r"(y));
            if (OP == 3) { unsigned long long w; asm volatile("mul.wide.u32 %0, %1, %2;" : "=l"(w) : "r"(x[i]), "r"(y)); x[i] = (uint32_t)w ^ (uint32_t)(w >> 32); }
            if (OP == 4) asm volatile("dp4a.u32.u32 %0, %0, %1, %2;" : "+r"(x[i]) : "r"(y), "r"(z));
            if (OP == 5) asm volatile("shf.r.wrap.b32 %0, %0, %1, %2;" : "+r"(x[i]) : "r"(y), "r"(z));
            if (OP == 6) asm volatile("lop3.b32 %0, %0, %1, %2, 0x96;" : "+r"(x[i]) : "r"(y), "r"(z));
            if (OP == 7) asm volatile("prmt.b32 %0, %0, %1, %2;" : "+r"(x[i]) : "r"(y), "r"(z));
            if (OP == 8) asm volatile("shr.u32 %0, %0, 5;" : "+r"(x[i]));
            if (OP == 9) asm volatile("bfe.u32 %0, %0, 7, 5;" : "+r"(x[i]));
            if (OP == 10) asm volatile("popc.b32 %0, %0;" : "+r"(x[i]));
            if (OP == 11) asm volatile("add.u32 %0, %0, %1;" : "+r"(x[i]) : "r"(y));
            if (OP == 12) asm volatile("mad.hi.u32 %0, %0, %1, %2;" : "+r"(x[i]) : "r"(y), "r"(z));
            if (OP == 13) { float f = __uint_as_float(x[i]); asm volatile("fma.rn.f32 %0, %0, %1, %2;" : "+f"(f) : "f"(__uint_as_float(y)), "f"(__uint_as_float(z))); x[i] = __float_as_uint(f); }
            if (OP == 14) asm volatile("mul24.lo.u32 %0, %0, %1;" : "+r"(x[i]) : "r"(y));
            if (OP == 15) asm volatile("mul.wide.u16 %0, %1, %2;" : "=r"(x[i]) : "h"((unsigned short)x[i]), "h"((unsigned short)y));
            if (OP == 16) asm volatile("shf.l.wrap.b32 %0, %0, %0, %1;" : "+r"(x[i]) : "r"(y));
            if (OP == 17) asm volatile("bfind.u32 %0, %0;" : "+r"(x[i]));
            if (OP == 18) asm volatile("vabsdiff4.u32.u32.u32.add %0, %0, %1, %2;" : "+r"(x[i]) : "r"(y), "r"(z));
            if (OP == 19) asm volatile("dp2a.lo.u32.u32 %0, %0, %1, %2;" : "+r"(x[i]) : "r"(y), "r"(z));
        }
    }
    unsigned long long t1 = clock64();
    uint32_t s = 0;
#pragma unroll
    for (int i = 0; i < CHAINS; i++) s ^= x[i];
    out[blockIdx.x * blockDim.x + threadIdx.x] = s;
    if (threadIdx.x == 0 && blockIdx.x == 0) *cyc = t1 - t0;
}
template <int OP> void run(const char *name, uint32_t *d, unsigned long long *dc) {
    const int threads = 1024;                       // 32 warps = 8 per sub-partition
    k<OP><<<132, threads>>>(d, 12345u, dc);
    cudaDeviceSynchronize();
    k<OP><<<132, threads>>>(d, 12345u, dc);
    cudaDeviceSynchronize();
    unsigned long long c = 0; cudaMemcpy(&c, dc, 8, cudaMemcpyDeviceToHost);
    double per = (double)c / ((double)ITERS * CHAINS * 8.0);      // 8 warps per sub-partition issue ITERS*CHAINS each
    printf("%-22s %8.2f cycles per warp-instruction per sub-partition (%s)\n", name, per, cudaGetErrorString(cudaGetLastError()));
}
int main() {
    uint32_t *d; unsigned long long *dc;
    cudaMalloc(&d, 132 * 1024 * 4); cudaMalloc(&dc, 8);
    run<0>("mul.lo.u32", d, dc); run<1>("mad.lo.u32", d, dc); run<2>("mul.hi.u32", d, dc); run<12>("mad.hi.u32", d, dc);
    run<3>("mul.wide.u32 (+xor)", d, dc); run<4>("dp4a.u32.u32", d, dc); run<19>("dp2a.lo.u32.u32", d, dc);
    run<5>("shf.r.wrap", d, dc); run<16>("shf.l.wrap (rot)", d, dc); run<6>("lop3", d, dc); run<7>("prmt", d, dc);
    run<8>("shr.u32 imm", d, dc); run<9>("bfe.u32", d, dc); run<10>("popc", d, dc); run<11>("add.u32", d, dc);
    run<13>("fma.rn.f32", d, dc); run<14>("mul24.lo.u32", d, dc); run<15>("mul.wide.u16", d, dc); run<17>("bfind", d, dc); run<18>("vabsdiff4.add", d, dc);
    return 0;
}
