// Probe: accuracy of three ways of feeding 2-bit codes to mma.sync.m16n8k16 (fp16 in, fp32 accumulate):
//   exact  : A = ((w & mask_j) | 0x6400) - 1024            = c * 4^j                 (LOP3 + HADD2 per pair)
//   denorm : A = (w & mask_j)  (fp16 denormal)              = c * 4^j * 2^-24         (LOP3 per pair)
//   offset : A = (w & mask_j) | 0x6400                      = 1024 + c * 4^j          (LOP3 per pair; minus 1024*sum(B))
// B = hi/lo split of x*s (x, s random fp16), K = 128 (8 accumulating MMAs), compared with fp64.
// Build: nvcc -gencode arch=compute_90a,code=sm_90a -O3 -o mma_unpack_variants mma_unpack_variants.cu
#include <cstdio>
#include <cstdlib>
#include <cstdint>
#include <cmath>
#include <cuda_fp16.h>

__device__ __forceinline__ void mma(float (&c)[4], uint32_t a0, uint32_t a1, uint32_t a2, uint32_t a3, uint32_t b0, uint32_t b1) {
    asm volatile("mma.sync.aligned.m16n8k16.row.col.f32.f16.f16.f32 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, {%0,%1,%2,%3};"
                 : "+f"(c[0]), "+f"(c[1]), "+f"(c[2]), "+f"(c[3]) : "r"(a0), "r"(a1), "r"(a2), "r"(a3), "r"(b0), "r"(b1));
}

// codes[step][m][k] (2-bit), B[step][n][k] fp16 bits; out[variant][j][m][n]
__global__ void probe(const uint8_t* codes, const uint16_t* B, float* out, float bscale_log2) {
    const int lane = threadIdx.x, g = lane >> 2, t = lane & 3;
    for (int variant = 0; variant < 3; ++variant)
        for (int j = 0; j < 5; ++j) {
            float c[4] = {0, 0, 0, 0}, ones[4] = {0, 0, 0, 0};
            for (int st = 0; st < 8; ++st) {
                auto A2 = [&](int m, int k) -> uint32_t {
                    const uint32_t lo = codes[(st * 16 + m) * 16 + k], hi = codes[(st * 16 + m) * 16 + k + 1];
                    uint32_t w = (lo << (2 * j)) | (hi << (16 + 2 * j));
                    if (variant == 0) { w |= 0x64006400u; __half2 h = __hsub2(*(__half2*)&w, __float2half2_rn(1024.f)); return *(uint32_t*)&h; }
                    if (variant == 1) return w;
                    return w | 0x64006400u;
                };
                auto B2 = [&](int n, int k) -> uint32_t {
                    return (uint32_t)B[(st * 8 + n) * 16 + k] | ((uint32_t)B[(st * 8 + n) * 16 + k + 1] << 16);
                };
                const uint32_t a0 = A2(g, 2 * t), a1 = A2(g + 8, 2 * t), a2 = A2(g, 2 * t + 8), a3 = A2(g + 8, 2 * t + 8);
                const uint32_t b0 = B2(g, 2 * t), b1 = B2(g, 2 * t + 8);
                mma(c, a0, a1, a2, a3, b0, b1);
                if (variant == 2) mma(ones, 0x64006400u, 0x64006400u, 0x64006400u, 0x64006400u, b0, b1);
            }
            float sc = 1.f / (float)(1 << (2 * j));
            if (variant == 1) sc *= 16777216.f;
            float* o = out + ((variant * 5 + j) * 16) * 8;
            o[g * 8 + 2 * t] = (c[0] - ones[0]) * sc; o[g * 8 + 2 * t + 1] = (c[1] - ones[1]) * sc;
            o[(g + 8) * 8 + 2 * t] = (c[2] - ones[2]) * sc; o[(g + 8) * 8 + 2 * t + 1] = (c[3] - ones[3]) * sc;
        }
}

int main() {
    const int trials = 200;
    uint8_t* hc = (uint8_t*)malloc(8 * 16 * 16); uint16_t* hb = (uint16_t*)malloc(8 * 8 * 16 * 2);
    uint8_t* dc; uint16_t* db; float* dout; float hout[3 * 5 * 16 * 8];
    cudaMalloc(&dc, 8 * 16 * 16); cudaMalloc(&db, 8 * 8 * 16 * 2); cudaMalloc(&dout, sizeof(hout));
    for (int bs = 0; bs <= 12; bs += 6) {                      // B pre-scaled by 2^bs
        double worst_w[3][5] = {}, worst_l1[3][5] = {}, rms_w[3][5] = {};
        srand(1234);
        for (int tr = 0; tr < trials; ++tr) {
            for (int i = 0; i < 8 * 16 * 16; ++i) hc[i] = rand() & 3;
            // columns n even = hi, n odd = lo of the same x*s; x ~ N(0,1)-ish, s ~ U(0.5, 2)
            for (int st = 0; st < 8; ++st)
                for (int n = 0; n < 8; n += 2)
                    for (int k = 0; k < 16; ++k) {
                        float x = 0; for (int r = 0; r < 6; ++r) x += rand() / (float)RAND_MAX - 0.5f; x *= 1.41f;
                        if (tr % 4 == 1) x = fabsf(x);                               // biased sign: large sum(B)
                        float s = 0.5f + 1.5f * rand() / (float)RAND_MAX;
                        __half xh = __float2half(x * ldexpf(1.f, bs)), sh = __float2half(s);
                        float a = __half2float(xh) * __half2float(sh);
                        __half hi = __float2half(a); __half lo = __float2half(a - __half2float(hi));
                        hb[(st * 8 + n) * 16 + k] = *(uint16_t*)&hi; hb[(st * 8 + n + 1) * 16 + k] = *(uint16_t*)&lo;
                    }
            cudaMemcpy(dc, hc, 8 * 16 * 16, cudaMemcpyHostToDevice); cudaMemcpy(db, hb, 8 * 8 * 16 * 2, cudaMemcpyHostToDevice);
            probe<<<1, 32>>>(dc, db, dout, (float)bs); cudaMemcpy(hout, dout, sizeof(hout), cudaMemcpyDeviceToHost);
            for (int v = 0; v < 3; ++v) for (int j = 0; j < 5; ++j)
                for (int m = 0; m < 16; ++m) for (int n = 0; n < 8; n += 2) {
                    double ref = 0, l1 = 0;
                    for (int st = 0; st < 8; ++st) for (int k = 0; k < 16; ++k) {
                        double b = (double)__half2float(*(__half*)&hb[(st * 8 + n) * 16 + k]) + (double)__half2float(*(__half*)&hb[(st * 8 + n + 1) * 16 + k]);
                        double term = hc[(st * 16 + m) * 16 + k] * b; ref += term; l1 += fabs(term);
                    }
                    const float* o = hout + ((v * 5 + j) * 16) * 8;
                    double got = (double)o[m * 8 + n] + (double)o[m * 8 + n + 1];
                    double e = fabs(got - ref);
                    worst_w[v][j] = fmax(worst_w[v][j], e / (fabs(ref) + 1e-300 + 1e-3 * l1));
                    worst_l1[v][j] = fmax(worst_l1[v][j], e / l1);
                    rms_w[v][j] += (e / l1) * (e / l1);
                }
        }
        const char* names[3] = {"exact ", "denorm", "offset"};
        for (int v = 0; v < 3; ++v) for (int j = 0; j < 5; ++j)
            printf("Bscale 2^%-2d %s j=%d  worst err/L1 = %.3e (2^%.1f)  rms err/L1 = %.3e  worst err/(|W|+1e-3 L1) = %.3e\n", bs, names[v], j,
                   worst_l1[v][j], log2(worst_l1[v][j] + 1e-300), sqrt(rms_w[v][j] / (trials * 16 * 4)), worst_w[v][j]);
    }
    return 0;
}
