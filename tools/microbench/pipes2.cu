// Second pipe-rate microbenchmark: the opcodes of the four-lane Viterbi's 24-step stream, alone and mixed 1:1 with the fused add-min
// (VIADDMNMX.U16x2) and with the 16x2 add (VIADD.16x2), to learn which issue pipe each one takes on sm_90a.  Every kernel interleaves up to
// three instruction kinds over independent register chains; the number printed is warp-instructions per cycle per SM sub-partition (all
// kinds together).  Reading it: an opcode alone at 0.5 sits on a half-rate pipe; a 1:1 mix at ~1.0 means the two kinds issue on different
// pipes, at ~0.5 that they share one.  Check the SASS of this file (cuobjdump -sass) before trusting a line: ptxas is free to pick another
// opcode for an add.  "unif" marks a uniform-register operand (URx), as ptxas places the history marks in the Viterbi kernel.
//   nvcc -gencode arch=compute_90a,code=sm_90a -O3 -o pipes2 pipes2.cu && ./pipes2
#include <cuda_runtime.h>
#include <stdint.h>
#include <stdio.h>
#define ITER 2048
enum { ADDMIN, VADD2, VMIN2, IADD_RR, IADD_RU, IADD3_, RSUB, IMAD_RR, IMAD_IMM, PRMT_, PRMT_R, LOP3_, SHFL_, IDP_, NONE_ };
// a: the chain's value; x, y: two other chains of the same kind (so that ptxas can neither fold nor reassociate a chain); u: a uniform value
// that changes every iteration (a uniform-register operand, URx); sel: a PRMT selector in a vector register
template <int OP> __device__ __forceinline__ uint32_t op(uint32_t a, uint32_t x, uint32_t y, uint32_t u, uint32_t sel) {
    uint32_t r = a;
    if (OP == ADDMIN) asm volatile("{.reg .b32 t; add.u16x2 t, %1, %2; min.u16x2 %0, t, %3;}" : "=r"(r) : "r"(a), "r"(x), "r"(y));
    else if (OP == VADD2) asm volatile("add.u16x2 %0, %1, %2;" : "=r"(r) : "r"(a), "r"(x));
    else if (OP == VMIN2) asm volatile("min.u16x2 %0, %1, %2;" : "=r"(r) : "r"(a), "r"(x));
    else if (OP == IADD_RR) asm volatile("add.u32 %0, %1, %2;" : "=r"(r) : "r"(a), "r"(x));
    else if (OP == IADD_RU) asm volatile("add.u32 %0, %1, %2;" : "=r"(r) : "r"(a), "r"(u));
    else if (OP == IADD3_) asm volatile("{.reg .b32 t; add.u32 t, %1, %2; add.u32 %0, t, %3;}" : "=r"(r) : "r"(a), "r"(x), "r"(y));
    else if (OP == RSUB) asm volatile("sub.u32 %0, %2, %1;" : "=r"(r) : "r"(a), "r"(x));
    else if (OP == IMAD_RR) asm volatile("mad.lo.u32 %0, %1, %2, %3;" : "=r"(r) : "r"(a), "r"(x), "r"(y));
    else if (OP == IMAD_IMM) asm volatile("mad.lo.u32 %0, %1, 0x0101, %2;" : "=r"(r) : "r"(a), "r"(x));
    else if (OP == PRMT_) asm volatile("prmt.b32 %0, %1, %2, 0x7531;" : "=r"(r) : "r"(a), "r"(x));
    else if (OP == PRMT_R) asm volatile("prmt.b32 %0, %1, %2, %3;" : "=r"(r) : "r"(a), "r"(x), "r"(sel));
    else if (OP == LOP3_) asm volatile("lop3.b32 %0, %1, %2, %3, 0xE8;" : "=r"(r) : "r"(a), "r"(x), "r"(y));
    else if (OP == SHFL_) asm volatile("shfl.sync.bfly.b32 %0, %1, 2, 0x1f, 0xffffffff;" : "=r"(r) : "r"(a));
    else if (OP == IDP_) asm volatile("dp4a.u32.s32 %0, %1, %2, %3;" : "=r"(r) : "r"(a), "r"(u), "r"(x));
    return r;
}
template <int A, int NA, int B, int NB, int C, int NC>
__global__ void k(uint32_t* out, uint32_t s, long long* cyc) {
    uint32_t v[12];
#pragma unroll
    for (int i = 0; i < 12; i++) v[i] = s * (i + 1) + threadIdx.x;
    const uint32_t sel = __shfl_sync(0xFFFFFFFFu, (s & 0x3u) | 0x7100u, 0);
    __syncthreads();
    long long t0 = clock64();
    for (int it = 0; it < ITER; it++) {
        const uint32_t u = s ^ ((uint32_t)it << 8);
#pragma unroll
        for (int i = 0; i < 4; i++) {
#pragma unroll
            for (int j = 0; j < NA; j++) v[i] = op<A>(v[i], v[(i + 1) & 3], v[(i + 2) & 3], u, sel);
#pragma unroll
            for (int j = 0; j < NB; j++) v[4 + i] = op<B>(v[4 + i], v[4 + ((i + 1) & 3)], v[4 + ((i + 2) & 3)], u, sel);
#pragma unroll
            for (int j = 0; j < NC; j++) v[8 + i] = op<C>(v[8 + i], v[8 + ((i + 1) & 3)], v[8 + ((i + 2) & 3)], u, sel);
        }
    }
    long long t1 = clock64();
    uint32_t acc = 0;
#pragma unroll
    for (int i = 0; i < 12; i++) acc ^= v[i];
    out[blockIdx.x * blockDim.x + threadIdx.x] = acc;
    if (threadIdx.x == 0 && blockIdx.x == 0) *cyc = t1 - t0;
}
template <int A, int NA, int B, int NB, int C, int NC> void run(const char* name, int wps = 8) {
    uint32_t* d; long long* dc; cudaMalloc(&d, 1 << 22); cudaMalloc(&dc, 8);
    int nsm; cudaDeviceGetAttribute(&nsm, cudaDevAttrMultiProcessorCount, 0);     // one CTA per SM
    for (int r = 0; r < 2; r++) { k<A, NA, B, NB, C, NC><<<nsm, 128 * wps>>>(d, 12345u, dc); cudaDeviceSynchronize(); }
    long long c; cudaMemcpy(&c, dc, 8, cudaMemcpyDeviceToHost);
    printf("%-44s warps/SMSP %d  warp-inst/cycle/SMSP %.3f\n", name, wps, (double)ITER * 4 * (NA + NB + NC) * wps / (double)c);
    cudaFree(d); cudaFree(dc);
}
// one opcode alone, then 1:1 with the add-min, then 1:1 with the 16x2 add
#define ROW(OP, NAME) run<OP, 1, NONE_, 0, NONE_, 0>(NAME); run<ADDMIN, 1, OP, 1, NONE_, 0>("addmin + " NAME); run<VADD2, 1, OP, 1, NONE_, 0>("vadd2 + " NAME);
int main() {
    run<ADDMIN, 1, NONE_, 0, NONE_, 0>("VIADDMNMX.U16x2");
    run<VADD2, 1, NONE_, 0, NONE_, 0>("VIADD.16x2");
    run<ADDMIN, 1, VADD2, 1, NONE_, 0>("addmin + vadd2");
    ROW(VMIN2, "VIMNMX.U16x2")
    ROW(IADD_RR, "add r,r")
    ROW(IADD_RU, "add r,r(unif)")
    ROW(IADD3_, "add r,r,r")
    ROW(RSUB, "sub r - r")
    ROW(IMAD_RR, "mad.lo r,r,r")
    ROW(IMAD_IMM, "mad.lo r,imm,r")
    ROW(PRMT_, "prmt imm selector")
    ROW(PRMT_R, "prmt register selector")
    ROW(LOP3_, "lop3")
    ROW(SHFL_, "shfl.bfly")
    ROW(IDP_, "dp4a")
    // the stream's own mix per trellis step, rounded: 8 add-min, 8 16x2 adds, 4 scalar adds (the marks)
    run<ADDMIN, 2, VADD2, 2, IADD_RU, 1>("2 addmin + 2 vadd2 + add r,r(unif)");
    run<ADDMIN, 2, VADD2, 2, PRMT_R, 1>("2 addmin + 2 vadd2 + prmt");
    run<ADDMIN, 2, VADD2, 2, SHFL_, 1>("2 addmin + 2 vadd2 + shfl");
    run<ADDMIN, 1, VADD2, 1, NONE_, 0>("addmin + vadd2 (4 warps)", 4);
    run<ADDMIN, 1, VADD2, 1, NONE_, 0>("addmin + vadd2 (2 warps)", 2);
    run<ADDMIN, 1, VADD2, 1, NONE_, 0>("addmin + vadd2 (1 warp)", 1);
    return 0;
}
