// Pipe-rate microbenchmark for the integer SIMD instructions the Viterbi kernel is built from (sm_90a).
// Each kernel runs a dependent-free stream of one instruction kind (8 independent chains per thread) so the number reported is
// issue throughput: warp-instructions per cycle per SM sub-partition.   nvcc -arch=sm_90a -O3 -o pipes pipes.cu && ./pipes
#include <cuda_runtime.h>
#include <stdint.h>
#include <stdio.h>
#define ITER 4096
template <int OP> __device__ __forceinline__ uint32_t op(uint32_t a, uint32_t b, uint32_t c) {
    uint32_t r;
    if (OP == 0) asm volatile("min.u16x2 %0, %1, %2;" : "=r"(r) : "r"(a), "r"(b));                                       // VIMNMX.U16x2
    else if (OP == 1) asm volatile("{.reg .b32 t; add.u16x2 t, %1, %2; min.u16x2 %0, t, %3;}" : "=r"(r) : "r"(a), "r"(b), "r"(c)); // VIADDMNMX.U16x2
    else if (OP == 2) asm volatile("add.u16x2 %0, %1, %2;" : "=r"(r) : "r"(a), "r"(b));                                   // VIADD.16x2
    else if (OP == 3) asm volatile("mad.lo.u32 %0, %1, 1, %2;" : "=r"(r) : "r"(a), "r"(b));                               // IMAD.IADD
    else if (OP == 4) asm volatile("lop3.b32 %0, %1, %2, %3, 0xE8;" : "=r"(r) : "r"(a), "r"(b), "r"(c));                  // LOP3
    else if (OP == 5) asm volatile("prmt.b32 %0, %1, %2, 0x7531;" : "=r"(r) : "r"(a), "r"(b));                            // PRMT
    else if (OP == 6) asm volatile("mul.hi.u32 %0, %1, 0x80000000;" : "=r"(r) : "r"(a));                                  // IMAD.HI
    else if (OP == 7) asm volatile("dp4a.u32.s32 %0, %1, %2, %3;" : "=r"(r) : "r"(a), "r"(b), "r"(c));                    // IDP.4A
    else if (OP == 8) asm volatile("shr.u32 %0, %1, 1;" : "=r"(r) : "r"(a));                                              // SHF
    else if (OP == 9) asm volatile("add.u32 %0, %1, %2;" : "=r"(r) : "r"(a), "r"(b));                                     // IADD3 / VIADD (compiler's choice)
    else if (OP == 10) asm volatile("{.reg .b32 t; min.u16x2 t, %1, %2; min.u16x2 %0, t, %3;}" : "=r"(r) : "r"(a), "r"(b), "r"(c)); // VIMNMX3.U16x2
    else r = a;
    return r;
}
// MIX: alternate OPA (ALU) and OPB (FMA-pipe) instructions
template <int OPA, int OPB, int NA, int NB>
__global__ void k(uint32_t* out, uint32_t s, long long* cyc) {
    uint32_t v[8];
#pragma unroll
    for (int i = 0; i < 8; i++) v[i] = s * (i + 1) + threadIdx.x;
    uint32_t b = s ^ 0x01000100u, c = s + 77u;
    __syncthreads();
    long long t0 = clock64();
    for (int it = 0; it < ITER; it++) {
#pragma unroll
        for (int i = 0; i < 8; i++) {
#pragma unroll
            for (int j = 0; j < NA; j++) v[i] = op<OPA>(v[i], b, c);
#pragma unroll
            for (int j = 0; j < NB; j++) v[(i + 3) & 7] = op<OPB>(v[(i + 3) & 7], c, b);
        }
    }
    long long t1 = clock64();
    uint32_t acc = 0;
#pragma unroll
    for (int i = 0; i < 8; i++) acc ^= v[i];
    out[blockIdx.x * blockDim.x + threadIdx.x] = acc;
    if (threadIdx.x == 0 && blockIdx.x == 0) *cyc = t1 - t0;
}
template <int OPA, int OPB, int NA, int NB> void run(const char* name, int warps_per_smsp) {
    uint32_t* d; long long* dc; cudaMalloc(&d, 1 << 22); cudaMalloc(&dc, 8);
    int nsm; cudaDeviceGetAttribute(&nsm, cudaDevAttrMultiProcessorCount, 0);     // one CTA per SM
    int threads = 32 * 4 * warps_per_smsp;
    k<OPA, OPB, NA, NB><<<nsm, threads>>>(d, 12345u, dc); cudaDeviceSynchronize();
    k<OPA, OPB, NA, NB><<<nsm, threads>>>(d, 12345u, dc); cudaDeviceSynchronize();
    long long c; cudaMemcpy(&c, dc, 8, cudaMemcpyDeviceToHost);
    double ninst = (double)ITER * 8 * (NA + NB) * warps_per_smsp;      // warp-instructions per SMSP
    printf("%-34s warps/SMSP %d  cycles %9lld  warp-inst/cycle/SMSP %.3f\n", name, warps_per_smsp, c, ninst / (double)c);
    cudaFree(d); cudaFree(dc);
}
#define R1(OP, NAME) run<OP, 11, 1, 0>(NAME, 1); run<OP, 11, 1, 0>(NAME, 4); run<OP, 11, 1, 0>(NAME, 8);
int main() {
    R1(0, "VIMNMX.U16x2") R1(1, "VIADDMNMX.U16x2") R1(2, "VIADD.16x2") R1(3, "IMAD.IADD") R1(4, "LOP3") R1(5, "PRMT")
    R1(6, "IMAD.HI") R1(7, "IDP.4A") R1(8, "SHF") R1(9, "add.u32") R1(10, "VIMNMX3.U16x2")
    run<1, 3, 1, 1>("VIADDMNMX + IMAD.IADD 1:1", 4); run<1, 3, 1, 1>("VIADDMNMX + IMAD.IADD 1:1", 8);
    run<0, 3, 1, 2>("VIMNMX + 2 IMAD.IADD", 4);
    run<4, 3, 1, 1>("LOP3 + IMAD.IADD 1:1", 4);
    run<1, 2, 1, 1>("VIADDMNMX + VIADD.16x2 1:1", 4);
    run<1, 5, 1, 1>("VIADDMNMX + PRMT 1:1", 4);
    run<1, 6, 1, 1>("VIADDMNMX + IMAD.HI 1:1", 4);
    run<1, 7, 1, 1>("VIADDMNMX + IDP.4A 1:1", 4);
    return 0;
}
