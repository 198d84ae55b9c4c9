// Pipe-rate microbenchmark for the decode-attention design space (sm_90a): legacy mma.sync fp16 vs u8 vs e4m3,
// fp8 conversions, LOP3 / PRMT.  One CTA per SM, W warps per CTA; cycles per warp instruction per sub-partition.
//   nvcc -O3 -gencode arch=compute_90a,code=sm_90a -o tools/ubench/pipes tools/ubench/pipes.cu && tools/ubench/pipes
#include <cstdio>
#include <cstdint>
#include <cuda_fp16.h>
#include <cuda_runtime.h>

#define ITERS 2048

template <int OP>
__global__ void k(uint32_t *out, long long *cyc, uint32_t seed) {
    uint32_t a0 = seed + threadIdx.x, a1 = a0 * 3, a2 = a0 * 5, a3 = a0 * 7, b0 = a0 ^ 0x3c003c00u, b1 = a1 ^ 0x38383838u;
    float c[8][4];
    int ci[8][4];
#pragma unroll
    for (int i = 0; i < 8; ++i) { c[i][0] = c[i][1] = c[i][2] = c[i][3] = 0.f; ci[i][0] = ci[i][1] = ci[i][2] = ci[i][3] = 0; }
    uint32_t r[8];
#pragma unroll
    for (int i = 0; i < 8; ++i) r[i] = a0 + i * 0x01010101u;
    __syncthreads();
    long long t0 = clock64();
    for (int it = 0; it < ITERS; ++it) {
#pragma unroll
        for (int i = 0; i < 8; ++i) {
            if (OP == 0) {
                asm volatile("mma.sync.aligned.m16n8k16.row.col.f32.f16.f16.f32 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, {%0,%1,%2,%3};"
                             : "+f"(c[i][0]), "+f"(c[i][1]), "+f"(c[i][2]), "+f"(c[i][3])
                             : "r"(a0), "r"(a1), "r"(a2), "r"(a3), "r"(b0), "r"(b1));
            } else if (OP == 1) {
                asm volatile("mma.sync.aligned.m16n8k32.row.col.s32.u8.s8.s32 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, {%0,%1,%2,%3};"
                             : "+r"(ci[i][0]), "+r"(ci[i][1]), "+r"(ci[i][2]), "+r"(ci[i][3])
                             : "r"(a0), "r"(a1), "r"(a2), "r"(a3), "r"(b0), "r"(b1));
            } else if (OP == 11) {     // e4m3 mma.sync
                asm volatile("mma.sync.aligned.m16n8k32.row.col.f32.e4m3.e4m3.f32 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, {%0,%1,%2,%3};"
                             : "+f"(c[i][0]), "+f"(c[i][1]), "+f"(c[i][2]), "+f"(c[i][3])
                             : "r"(a0), "r"(a1), "r"(a2), "r"(a3), "r"(b0), "r"(b1));
            } else if (OP == 2) {      // f16x2 -> e4m3x2
                uint16_t o;
                asm volatile("cvt.rn.satfinite.e4m3x2.f16x2 %0, %1;" : "=h"(o) : "r"(r[i]));
                r[i] += o;
            } else if (OP == 3) {      // e4m3x2 -> f16x2
                uint32_t o;
                asm volatile("cvt.rn.f16x2.e4m3x2 %0, %1;" : "=r"(o) : "h"((uint16_t)r[i]));
                r[i] ^= o;
            } else if (OP == 4) {      // LOP3
                asm volatile("lop3.b32 %0, %0, %1, %2, 0xea;" : "+r"(r[i]) : "r"(a1), "r"(a2));
            } else if (OP == 5) {      // PRMT
                asm volatile("prmt.b32 %0, %0, %1, 0x5410;" : "+r"(r[i]) : "r"(a1));
            } else if (OP == 6) {      // HFMA2
                asm volatile("fma.rn.f16x2 %0, %0, %1, %2;" : "+r"(r[i]) : "r"(b0), "r"(b1));
            } else if (OP == 7) {      // f32 pair -> e4m3x2
                uint16_t o;
                asm volatile("cvt.rn.satfinite.e4m3x2.f32 %0, %1, %2;" : "=h"(o) : "f"(__uint_as_float(r[i])), "f"(__uint_as_float(a1)));
                r[i] += o;
            } else if (OP == 8) {      // SHF
                asm volatile("shf.r.wrap.b32 %0, %0, %1, 3;" : "+r"(r[i]) : "r"(a1));
            } else if (OP == 9) {      // mixed: 4 LOP3 per u8 MMA (16 two-bit codes of a word -> 4 A registers, no shift)
                uint32_t w = r[i];
                uint32_t x0, x1, x2, x3;
                asm volatile("lop3.b32 %0, %1, 0x03030303, 0, 0xc0;" : "=r"(x0) : "r"(w));
                asm volatile("lop3.b32 %0, %1, 0x0c0c0c0c, 0, 0xc0;" : "=r"(x1) : "r"(w));
                asm volatile("lop3.b32 %0, %1, 0x30303030, 0, 0xc0;" : "=r"(x2) : "r"(w));
                asm volatile("lop3.b32 %0, %1, 0xc0c0c0c0, 0, 0xc0;" : "=r"(x3) : "r"(w));
                asm volatile("mma.sync.aligned.m16n8k32.row.col.s32.u8.s8.s32 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, {%0,%1,%2,%3};"
                             : "+r"(ci[i][0]), "+r"(ci[i][1]), "+r"(ci[i][2]), "+r"(ci[i][3])
                             : "r"(x0), "r"(x1), "r"(x2), "r"(x3), "r"(b0), "r"(b1));
                r[i] = w + 0x11;
            } else if (OP == 10) {     // mixed fp16: 8 LOP3 + 1 SHF per 2 fp16 MMAs (today's ratio for 16 codes)
                uint32_t w = r[i], x[8], s;
                asm volatile("shf.r.wrap.b32 %0, %1, %1, 2;" : "=r"(s) : "r"(w));
#pragma unroll
                for (int j = 0; j < 4; ++j) {
                    asm volatile("lop3.b32 %0, %1, %2, 0, 0xc0;" : "=r"(x[j]) : "r"(w), "r"(0x00300030u << (2 * j)));
                    asm volatile("lop3.b32 %0, %1, %2, 0, 0xc0;" : "=r"(x[4 + j]) : "r"(s), "r"(0x00300030u << (2 * j)));
                }
                asm volatile("mma.sync.aligned.m16n8k16.row.col.f32.f16.f16.f32 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, {%0,%1,%2,%3};"
                             : "+f"(c[i][0]), "+f"(c[i][1]), "+f"(c[i][2]), "+f"(c[i][3])
                             : "r"(x[0]), "r"(x[1]), "r"(x[2]), "r"(x[3]), "r"(b0), "r"(b1));
                asm volatile("mma.sync.aligned.m16n8k16.row.col.f32.f16.f16.f32 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, {%0,%1,%2,%3};"
                             : "+f"(c[i][0]), "+f"(c[i][1]), "+f"(c[i][2]), "+f"(c[i][3])
                             : "r"(x[4]), "r"(x[5]), "r"(x[6]), "r"(x[7]), "r"(b0), "r"(b1));
                r[i] = w + 0x11;
            }
        }
    }
    long long t1 = clock64();
    uint32_t acc = 0;
#pragma unroll
    for (int i = 0; i < 8; ++i) acc += r[i] + __float_as_uint(c[i][0] + c[i][1] + c[i][2] + c[i][3]) + ci[i][0] + ci[i][1] + ci[i][2] + ci[i][3];
    out[blockIdx.x * blockDim.x + threadIdx.x] = acc;
    if (threadIdx.x == 0) cyc[blockIdx.x] = t1 - t0;
}

template <int OP>
void run(const char *name, int per_iter) {
    uint32_t *out; long long *cyc;
    cudaMalloc(&out, 148 * 1024 * 4); cudaMalloc(&cyc, 148 * 8);
    for (int warps : {4, 8, 16}) {
        k<OP><<<148, warps * 32>>>(out, cyc, 1);
        k<OP><<<148, warps * 32>>>(out, cyc, 1);
        cudaDeviceSynchronize();
        long long h[148]; cudaMemcpy(h, cyc, sizeof h, cudaMemcpyDeviceToHost);
        double avg = 0; for (int i = 0; i < 148; ++i) avg += h[i]; avg /= 148;
        double per = avg / (double(ITERS) * 8 * per_iter * (warps / 4.0));   // cycles per warp instruction per sub-partition
        printf("%-34s warps/SM %2d  cycles per warp-instr per SMSP %.3f\n", name, warps, per);
    }
    cudaError_t e = cudaGetLastError(); if (e) printf("  error %s\n", cudaGetErrorString(e));
    cudaFree(out); cudaFree(cyc);
}

int main() {
    run<0>("HMMA.16816.F32 (fp16)", 1);
    run<1>("IMMA.16832.U8.S8", 1);
    run<11>("mma.sync e4m3 (F2FP + 2 HMMA)", 1);
    run<2>("cvt f16x2->e4m3x2", 1);
    run<3>("cvt e4m3x2->f16x2", 1);
    run<7>("cvt f32,f32->e4m3x2", 1);
    run<4>("LOP3", 1);
    run<5>("PRMT", 1);
    run<8>("SHF", 1);
    run<6>("HFMA2", 1);
    run<9>("mix u8: 4 LOP3 + IMMA /16 codes", 1);
    run<10>("mix f16: 8 LOP3+SHF+2 HMMA /16 codes", 1);
    return 0;
}
