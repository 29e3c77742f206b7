// Second pipe-rate microbenchmark: mixes of the instructions of the v3 Viterbi step, to learn which share an issue pipe on sm_90a.
// Every kernel interleaves up to three instruction kinds over independent register chains; the number printed is warp-instructions per
// cycle per SM sub-partition (all kinds together).  Check the SASS of this file (cuobjdump -sass) before trusting a line: ptxas is free
// to pick another opcode for an add.   nvcc -arch=sm_90a -O3 -o pipes2 pipes2.cu && ./pipes2
#include <cuda_runtime.h>
#include <stdint.h>
#include <stdio.h>
#define ITER 2048
enum { ADDMIN, VADD2, VMIN2, IADD_RR, IADD_IMM, IADD3_, IMAD_RR, IMAD_IMM, PRMT_, LOP3_, SHFL_, IDP_, NONE_ };
template <int OP> __device__ __forceinline__ uint32_t op(uint32_t a, uint32_t b, uint32_t c) {
    uint32_t r = a;
    if (OP == ADDMIN) asm volatile("{.reg .b32 t; add.u16x2 t, %1, %2; min.u16x2 %0, t, %3;}" : "=r"(r) : "r"(a), "r"(b), "r"(c));
    else if (OP == VADD2) asm volatile("add.u16x2 %0, %1, %2;" : "=r"(r) : "r"(a), "r"(b));
    else if (OP == VMIN2) asm volatile("min.u16x2 %0, %1, %2;" : "=r"(r) : "r"(a), "r"(b));
    else if (OP == IADD_RR) asm volatile("add.u32 %0, %1, %2;" : "=r"(r) : "r"(a), "r"(b));
    else if (OP == IADD_IMM) asm volatile("add.u32 %0, %1, 0x00040004;" : "=r"(r) : "r"(a));
    else if (OP == IADD3_) asm volatile("{.reg .b32 t; add.u32 t, %1, %2; add.u32 %0, t, %3;}" : "=r"(r) : "r"(a), "r"(b), "r"(c));
    else if (OP == IMAD_RR) asm volatile("mad.lo.u32 %0, %1, %2, %3;" : "=r"(r) : "r"(a), "r"(b), "r"(c));
    else if (OP == IMAD_IMM) asm volatile("mad.lo.u32 %0, %1, 0x0101, %2;" : "=r"(r) : "r"(a), "r"(b));
    else if (OP == PRMT_) asm volatile("prmt.b32 %0, %1, %2, 0x7531;" : "=r"(r) : "r"(a), "r"(b));
    else if (OP == LOP3_) asm volatile("lop3.b32 %0, %1, %2, %3, 0xE8;" : "=r"(r) : "r"(a), "r"(b), "r"(c));
    else if (OP == SHFL_) asm volatile("shfl.sync.bfly.b32 %0, %1, 2, 0x1f, 0xffffffff;" : "=r"(r) : "r"(a));
    else if (OP == IDP_) asm volatile("dp4a.u32.s32 %0, %1, %2, %3;" : "=r"(r) : "r"(a), "r"(b), "r"(c));
    return r;
}
template <int A, int NA, int B, int NB, int C, int NC>
__global__ void k(uint32_t* out, uint32_t s, long long* cyc) {
    uint32_t v[12];
#pragma unroll
    for (int i = 0; i < 12; i++) v[i] = s * (i + 1) + threadIdx.x;
    uint32_t b = s ^ 0x01000100u, c = s + 77u;
    __syncthreads();
    long long t0 = clock64();
    for (int it = 0; it < ITER; it++) {
#pragma unroll
        for (int i = 0; i < 4; i++) {
#pragma unroll
            for (int j = 0; j < NA; j++) v[i] = op<A>(v[i], b, c);
#pragma unroll
            for (int j = 0; j < NB; j++) v[4 + i] = op<B>(v[4 + i], c, b);
#pragma unroll
            for (int j = 0; j < NC; j++) v[8 + i] = op<C>(v[8 + i], b, c);
        }
    }
    long long t1 = clock64();
    uint32_t acc = 0;
#pragma unroll
    for (int i = 0; i < 12; i++) acc ^= v[i];
    out[blockIdx.x * blockDim.x + threadIdx.x] = acc;
    if (threadIdx.x == 0 && blockIdx.x == 0) *cyc = t1 - t0;
}
template <int A, int NA, int B, int NB, int C, int NC> void run(const char* name, int wps = 4) {
    uint32_t* d; long long* dc; cudaMalloc(&d, 1 << 22); cudaMalloc(&dc, 8);
    int nsm; cudaDeviceGetAttribute(&nsm, cudaDevAttrMultiProcessorCount, 0);     // one CTA per SM
    for (int r = 0; r < 2; r++) { k<A, NA, B, NB, C, NC><<<nsm, 128 * wps>>>(d, 12345u, dc); cudaDeviceSynchronize(); }
    long long c; cudaMemcpy(&c, dc, 8, cudaMemcpyDeviceToHost);
    printf("%-52s warps/SMSP %d  warp-inst/cycle/SMSP %.3f\n", name, wps, (double)ITER * 4 * (NA + NB + NC) * wps / (double)c);
    cudaFree(d); cudaFree(dc);
}
int main() {
    run<IADD_RR, 1, NONE_, 0, NONE_, 0>("add r,r");
    run<IADD_IMM, 1, NONE_, 0, NONE_, 0>("add r,imm");
    run<IADD3_, 1, NONE_, 0, NONE_, 0>("add r,r,r (2 adds in PTX)");
    run<IMAD_RR, 1, NONE_, 0, NONE_, 0>("mad.lo r,r,r");
    run<IMAD_IMM, 1, NONE_, 0, NONE_, 0>("mad.lo r,imm,r");
    run<SHFL_, 1, NONE_, 0, NONE_, 0>("shfl.bfly");
    run<ADDMIN, 1, VADD2, 1, NONE_, 0>("addmin + vadd2");
    run<ADDMIN, 1, VADD2, 1, IADD_RR, 1>("addmin + vadd2 + add r,r");
    run<ADDMIN, 1, VADD2, 1, IADD_IMM, 1>("addmin + vadd2 + add r,imm");
    run<ADDMIN, 1, VADD2, 1, IMAD_RR, 1>("addmin + vadd2 + mad r,r,r");
    run<ADDMIN, 1, VADD2, 1, IMAD_IMM, 1>("addmin + vadd2 + mad r,imm,r");
    run<ADDMIN, 1, VADD2, 1, PRMT_, 1>("addmin + vadd2 + prmt");
    run<ADDMIN, 2, VADD2, 2, PRMT_, 1>("2 addmin + 2 vadd2 + prmt");
    run<ADDMIN, 2, VADD2, 2, IADD_RR, 1>("2 addmin + 2 vadd2 + add r,r");
    run<ADDMIN, 2, VADD2, 2, SHFL_, 1>("2 addmin + 2 vadd2 + shfl");
    run<VADD2, 1, IADD_RR, 1, NONE_, 0>("vadd2 + add r,r");
    run<VADD2, 1, IMAD_RR, 1, NONE_, 0>("vadd2 + mad r,r,r");
    run<VADD2, 1, IMAD_IMM, 1, NONE_, 0>("vadd2 + mad r,imm,r");
    run<VADD2, 1, IDP_, 1, NONE_, 0>("vadd2 + dp4a");
    run<VADD2, 1, PRMT_, 1, NONE_, 0>("vadd2 + prmt");
    run<ADDMIN, 1, IADD_RR, 1, NONE_, 0>("addmin + add r,r");
    run<ADDMIN, 1, IADD_IMM, 1, NONE_, 0>("addmin + add r,imm");
    run<ADDMIN, 1, IMAD_RR, 1, NONE_, 0>("addmin + mad r,r,r");
    run<VMIN2, 1, VADD2, 2, NONE_, 0>("vmin2 + 2 vadd2");
    run<VMIN2, 1, IADD_RR, 2, NONE_, 0>("vmin2 + 2 add r,r");
    run<PRMT_, 1, IADD_RR, 1, NONE_, 0>("prmt + add r,r");
    run<PRMT_, 1, IMAD_RR, 1, NONE_, 0>("prmt + mad r,r,r");
    run<ADDMIN, 1, VADD2, 1, NONE_, 0>("addmin + vadd2 (2 warps)", 2);
    run<ADDMIN, 1, VADD2, 1, NONE_, 0>("addmin + vadd2 (1 warp)", 1);
    return 0;
}
