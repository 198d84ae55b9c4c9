// kivi_bgemv.cu -- batched "outer-dim" dequant-GEMV on caller-supplied (reference) layouts, sm_90a.
//
//   C[u_q, n] = sum_k A[u_q, k] * (scale[u_kv, k, n/g] * code[u_kv, k, n] + zero[u_kv, k, n/g])
//
// Replaces kivi_gemv.gemv_forward_cuda_outer_dim (quant/csrc/gemv_cuda.cu:511-557, kernels
// :265-427) and, on KIVI_LAYOUT_REFERENCE, the whole of cuda_bmm_fA_qB_outer
// (quant/matmul.py:178-219) without its three transpose().contiguous() copies.
//
// Design (KIVI_LAYOUT_REFERENCE, the layout the models hold their cache in):
//   * the packed axis n is the contiguous one, so a lane owns one 32-element CELL of a row
//     (8 B of 2-bit codes / 16 B of 4-bit codes -> one 64/128-bit load) and, for g % 32 == 0,
//     exactly one (scale, zero) pair per row: no cross-lane traffic in the k loop;
//   * sum_k x*(s*c+z) is evaluated as sum_k (x*s)*c + sum_k x*z: x*s is exact in fp32 (two fp16
//     factors), the code is consumed as an in-place denormal (kivi_common.cuh) -> 1 LOP3 + 1 FFMA
//     per element instead of the reference's shift/and/I2F/FFMA/FFMA, fp32 accumulation kept;
//   * GQA: the G query heads of a KV head are processed by the same lane, so packed bytes are
//     read once per KV head (the reference re-reads them per query head, gemv_cuda.cu:361-365);
//   * "wide" shape (q.K^T: K = head_dim rows, N = tokens): a warp sweeps 1024 tokens over all rows;
//     "tall" shape (p.V: K = tokens, N = head_dim): lanes tile (rows x cells), 8 warps split the
//     rows, one shuffle + shared-memory reduction at the end.
#include "kivi_common.cuh"

namespace kivi {

// kivi_bgemv_mma.cu: tensor-core path for the two hot shapes on the reference layout (KIVI_ERR_UNSUPPORTED = not eligible)
int bgemv_ref_mma(const __half* A, long long a_stride, const uint32_t* qB, long long qb_us, long long qb_rs,
                  const __half* S, const __half* Z, long long sz_us, long long sz_rs, __half* C,
                  int B, int nh, int nh_kv, int K, int N, int bits, int g, cudaStream_t st);

template <int BITS> struct CellWords;                       // 32 elements of BITS bits
template <> struct CellWords<2> { using vec_t = uint2; static constexpr int kWords = 2; };
template <> struct CellWords<4> { using vec_t = uint4; static constexpr int kWords = 4; };

template <int BITS>
__device__ __forceinline__ void fma_cell(float (&acc)[32], const typename CellWords<BITS>::vec_t& cw, float a2) {
    constexpr int FPI = 32 / BITS;
    const uint32_t* w = reinterpret_cast<const uint32_t*>(&cw);
    #pragma unroll
    for (int j = 0; j < CellWords<BITS>::kWords; ++j) {
        float (&sub)[FPI] = *reinterpret_cast<float (*)[FPI]>(&acc[j * FPI]);
        fma_word<BITS>(sub, w[j], a2);
    }
}

template <int BITS>
__device__ __forceinline__ float cell_rescale(int e) { return field_rescale<BITS>(e % (32 / BITS)); }

// ------------------------------------------------------------------------------------------------
// wide: one warp = 1024 consecutive n, loops over all K rows.  grid = (U_kv, n-tiles/4, ratio/G)
// ------------------------------------------------------------------------------------------------
constexpr int kWideKTile = 128;

template <int BITS, int G>
__global__ void __launch_bounds__(128)
bgemv_ref_wide_kernel(const __half* __restrict__ A, int64_t a_stride,
                      const uint32_t* __restrict__ qB, int64_t qb_us, int64_t qb_rs,
                      const __half* __restrict__ S, const __half* __restrict__ Z, int64_t sz_us, int64_t sz_rs,
                      __half* __restrict__ C, int ratio, int K, int N, int g)
{
    using CW = CellWords<BITS>;
    using vec_t = typename CW::vec_t;
    __shared__ float xs[G][kWideKTile];

    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int ukv = blockIdx.x;
    const int h0 = blockIdx.z * G;                               // first query head of this chunk
    const int cell = (blockIdx.y * 4 + warp) * 32 + lane;
    const int n0 = cell * 32;
    const bool valid = n0 < N;

    const vec_t* cp = reinterpret_cast<const vec_t*>(qB + ukv * qb_us) + cell;
    const int64_t cp_rs = qb_rs / CW::kWords;                    // row stride in vec_t
    const __half* sp = S + ukv * sz_us + n0 / g;
    const __half* zp = Z + ukv * sz_us + n0 / g;

    float acc[G][32];
    float zs[G];
    #pragma unroll
    for (int h = 0; h < G; ++h) {
        zs[h] = 0.f;
        #pragma unroll
        for (int e = 0; e < 32; ++e) acc[h][e] = 0.f;
    }

    for (int k0 = 0; k0 < K; k0 += kWideKTile) {
        const int kt = min(kWideKTile, K - k0);
        __syncthreads();
        for (int i = threadIdx.x; i < G * kWideKTile; i += blockDim.x) {
            const int h = i / kWideKTile, k = i % kWideKTile;
            float v = 0.f;
            if (k < kt) v = __half2float(A[((int64_t)ukv * ratio + h0 + h) * a_stride + k0 + k]) * kPreScale;
            xs[h][k] = v;
        }
        __syncthreads();
        if (valid) {
            #pragma unroll 4
            for (int k = 0; k < kt; ++k) {
                const int64_t kk = k0 + k;
                const vec_t cw = __ldg(cp + kk * cp_rs);
                const float sf = __half2float(__ldg(sp + kk * sz_rs));
                const float zf = __half2float(__ldg(zp + kk * sz_rs));
                #pragma unroll
                for (int h = 0; h < G; ++h) {
                    const float x2 = xs[h][k];
                    zs[h] = fmaf(x2, zf, zs[h]);
                    fma_cell<BITS>(acc[h], cw, x2 * sf);
                }
            }
        }
    }
    if (!valid) return;
    #pragma unroll
    for (int h = 0; h < G; ++h) {
        __half* out = C + ((int64_t)ukv * ratio + h0 + h) * N + n0;
        const float zt = zs[h] * kPreScaleInv;
        #pragma unroll
        for (int v = 0; v < 4; ++v) {
            __align__(16) __half2 o[4];
            #pragma unroll
            for (int e = 0; e < 4; ++e) {
                const int i0 = v * 8 + 2 * e;
                o[e] = __floats2half2_rn(fmaf(acc[h][i0], cell_rescale<BITS>(i0), zt),
                                         fmaf(acc[h][i0 + 1], cell_rescale<BITS>(i0 + 1), zt));
            }
            *reinterpret_cast<uint4*>(out + v * 8) = *reinterpret_cast<const uint4*>(o);
        }
    }
}

// ------------------------------------------------------------------------------------------------
// tall: N <= 256.  lanes = (row class rc, cell ng); 8 warps split the rows.
// grid = (U_kv, 1, ratio/G), block = 256
// ------------------------------------------------------------------------------------------------
template <int BITS, int G>
__global__ void __launch_bounds__(256)
bgemv_ref_tall_kernel(const __half* __restrict__ A, int64_t a_stride,
                      const uint32_t* __restrict__ qB, int64_t qb_us, int64_t qb_rs,
                      const __half* __restrict__ S, const __half* __restrict__ Z, int64_t sz_us, int64_t sz_rs,
                      __half* __restrict__ C, int ratio, int K, int N, int g, int ng_log2)
{
    using CW = CellWords<BITS>;
    using vec_t = typename CW::vec_t;
    extern __shared__ float red[];                               // [8][NGp][G][33]

    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int ngp = 1 << ng_log2;
    const int ng = lane & (ngp - 1), rc = lane >> ng_log2;
    const int rpw = 32 >> ng_log2;                               // rows per warp step
    const int ukv = blockIdx.x;
    const int h0 = blockIdx.z * G;
    const int n0 = ng * 32;
    const bool cell_ok = n0 < N;

    const vec_t* cp = reinterpret_cast<const vec_t*>(qB + ukv * qb_us) + ng;
    const int64_t cp_rs = qb_rs / CW::kWords;
    const __half* sp = S + ukv * sz_us + n0 / g;
    const __half* zp = Z + ukv * sz_us + n0 / g;
    const __half* ap = A + ((int64_t)ukv * ratio + h0) * a_stride;

    float acc[G][32];
    float zs[G];
    #pragma unroll
    for (int h = 0; h < G; ++h) {
        zs[h] = 0.f;
        #pragma unroll
        for (int e = 0; e < 32; ++e) acc[h][e] = 0.f;
    }
    if (cell_ok) {
        #pragma unroll 2
        for (int k = warp * rpw + rc; k < K; k += 8 * rpw) {
            const vec_t cw = __ldg(cp + (int64_t)k * cp_rs);
            const float sf = __half2float(__ldg(sp + (int64_t)k * sz_rs));
            const float zf = __half2float(__ldg(zp + (int64_t)k * sz_rs));
            #pragma unroll
            for (int h = 0; h < G; ++h) {
                const float x2 = __half2float(__ldg(ap + h * a_stride + k)) * kPreScale;
                zs[h] = fmaf(x2, zf, zs[h]);
                fma_cell<BITS>(acc[h], cw, x2 * sf);
            }
        }
    }
    // reduce over the row classes held by different lanes of the warp
    for (int o = ngp; o < 32; o <<= 1) {
        #pragma unroll
        for (int h = 0; h < G; ++h) {
            zs[h] += __shfl_xor_sync(0xffffffffu, zs[h], o);
            #pragma unroll
            for (int e = 0; e < 32; ++e) acc[h][e] += __shfl_xor_sync(0xffffffffu, acc[h][e], o);
        }
    }
    if (rc == 0) {
        #pragma unroll
        for (int h = 0; h < G; ++h) {
            float* r = red + (((warp * ngp + ng) * G + h) * 33);
            #pragma unroll
            for (int e = 0; e < 32; ++e) r[e] = acc[h][e];
            r[32] = zs[h];
        }
    }
    __syncthreads();
    for (int o = threadIdx.x; o < ngp * G * 32; o += blockDim.x) {
        const int e = o & 31, h = (o >> 5) % G, c = (o >> 5) / G;
        const int n = c * 32 + e;
        if (n >= N) continue;
        float s = 0.f, zt = 0.f;
        #pragma unroll
        for (int w = 0; w < 8; ++w) {
            const float* r = red + (((w * ngp + c) * G + h) * 33);
            s += r[e];
            zt += r[32];
        }
        C[((int64_t)ukv * ratio + h0 + h) * N + n] =
            __float2half_rn(fmaf(s, cell_rescale<BITS>(e), zt * kPreScaleInv));
    }
}

// ------------------------------------------------------------------------------------------------
// any group size / alignment the reference accepts (g % fpi == 0): one thread per output element,
// per-element fma(fma(s,c,z), x, acc) exactly like the reference.  Slow path, never used by decode.
// ------------------------------------------------------------------------------------------------
template <int BITS>
__global__ void __launch_bounds__(128)
bgemv_ref_generic_kernel(const __half* __restrict__ A, int64_t a_stride,
                         const uint32_t* __restrict__ qB, int64_t qb_us, int64_t qb_rs,
                         const __half* __restrict__ S, const __half* __restrict__ Z, int64_t sz_us, int64_t sz_rs,
                         __half* __restrict__ C, int ratio, int K, int N, int g)
{
    constexpr int FPI = 32 / BITS;
    const int n = blockIdx.y * blockDim.x + threadIdx.x;
    const int uq = blockIdx.x;
    if (n >= N) return;
    const int ukv = uq / ratio;
    const uint32_t* wp = qB + ukv * qb_us + n / FPI;
    const int sh = BITS * (n % FPI);
    const __half* sp = S + ukv * sz_us + n / g;
    const __half* zp = Z + ukv * sz_us + n / g;
    const __half* ap = A + (int64_t)uq * a_stride;
    float acc = 0.f;
    for (int k = 0; k < K; ++k) {
        const float c = (float)((__ldg(wp + (int64_t)k * qb_rs) >> sh) & ((1u << BITS) - 1u));
        const float dq = fmaf(__half2float(__ldg(sp + (int64_t)k * sz_rs)), c, __half2float(__ldg(zp + (int64_t)k * sz_rs)));
        acc = fmaf(dq, __half2float(__ldg(ap + k)), acc);
    }
    C[(int64_t)uq * N + n] = __float2half_rn(acc);
}

// ------------------------------------------------------------------------------------------------
// KIVI_LAYOUT_KERNEL (the reference extension's own operand layout: reduction axis contiguous).
// One warp per packed row (fpi outputs); lanes stride over ic; reduce-scatter butterfly at the end
// (fpi + 1 shuffles instead of the reference's 5 * fpi).
// ------------------------------------------------------------------------------------------------
template <int BITS>
__global__ void __launch_bounds__(128)
bgemv_kernel_layout_kernel(const __half* __restrict__ A, int64_t a_stride,
                           const uint32_t* __restrict__ qB, int64_t qb_us, int64_t qb_rs,
                           const __half* __restrict__ S, const __half* __restrict__ Z, int64_t sz_us, int64_t sz_rs,
                           __half* __restrict__ C, int ratio, int IC, int OC, int g)
{
    constexpr int FPI = 32 / BITS;
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int p = blockIdx.y * 4 + warp;                         // packed row
    const int uq = blockIdx.x;
    if (p >= OC / FPI) return;
    const int ukv = uq / ratio;
    const int grp = (p * FPI) / g;
    const uint32_t* wp = qB + ukv * qb_us + (int64_t)p * qb_rs;
    const __half* sp = S + ukv * sz_us + (int64_t)grp * sz_rs;
    const __half* zp = Z + ukv * sz_us + (int64_t)grp * sz_rs;
    const __half* ap = A + (int64_t)uq * a_stride;

    float acc[FPI];
    #pragma unroll
    for (int i = 0; i < FPI; ++i) acc[i] = 0.f;
    float zs = 0.f;
    #pragma unroll 4
    for (int ic = lane; ic < IC; ic += 32) {
        const uint32_t w = __ldg(wp + ic);
        const float x2 = __half2float(__ldg(ap + ic)) * kPreScale;
        zs = fmaf(x2, __half2float(__ldg(zp + ic)), zs);
        fma_word<BITS>(acc, w, x2 * __half2float(__ldg(sp + ic)));
    }
    zs = warp_sum(zs) * kPreScaleInv;
    #pragma unroll
    for (int i = 0; i < FPI; ++i) acc[i] *= field_rescale<BITS>(i);
    // reduce-scatter: after the step with offset o, a lane keeps the half of its values selected by
    // its bit o; lane bits (16,8,4[,2]) end up encoding the output index.
    int width = FPI;
    #pragma unroll
    for (int o = 16; width > 1; o >>= 1) {
        width >>= 1;
        const bool upper = (lane & o) != 0;
        #pragma unroll
        for (int j = 0; j < FPI / 2; ++j) {
            if (j < width) {
                const float send = upper ? acc[j] : acc[j + width];
                const float keep = upper ? acc[j + width] : acc[j];
                acc[j] = keep + __shfl_xor_sync(0xffffffffu, send, o);
            }
        }
    }
    constexpr int kSteps = (FPI == 16) ? 4 : 3;                  // log2(FPI)
    #pragma unroll
    for (int o = 16 >> kSteps; o >= 1; o >>= 1) acc[0] += __shfl_xor_sync(0xffffffffu, acc[0], o);
    if ((lane & ((32 >> kSteps) - 1)) == 0) {
        const int j = lane >> (5 - kSteps);                      // bits 16,8,4(,2) -> output index, MSB first
        C[(int64_t)uq * OC + p * FPI + j] = __float2half_rn(acc[0] + zs);
    }
}

// ------------------------------------------------------------------------------------------------
// inner-dim AWQ-style 4-bit GEMV (tests-only surface of the reference, gemv_cuda.cu:60-246)
// ------------------------------------------------------------------------------------------------
template <int BITS>
__global__ void __launch_bounds__(128)
gemv_inner_kernel(const __half* __restrict__ in, const uint32_t* __restrict__ kernel,
                  const __half* __restrict__ S, const __half* __restrict__ Z, __half* __restrict__ out,
                  int IC, int OC, int g, int64_t sf_w)
{
    constexpr int FPI = 32 / BITS;
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int oc = blockIdx.y * 4 + warp;
    const int b = blockIdx.x;
    if (oc >= OC) return;
    const int nw = IC / FPI;
    float acc = 0.f;
    for (int wi = lane; wi < nw; wi += 32) {
        uint32_t w = __ldg(kernel + (int64_t)oc * nw + wi);
        const int grp = (wi * FPI) / g;
        const float sf = __half2float(__ldg(S + (int64_t)oc * sf_w + grp));
        const float zf = __half2float(__ldg(Z + (int64_t)oc * sf_w + grp));
        const __half* xp = in + (int64_t)b * IC + wi * FPI;
        #pragma unroll
        for (int j = 0; j < FPI; ++j) {
            const float dq = fmaf(sf, (float)(w & ((1u << BITS) - 1u)), zf);
            acc = fmaf(dq, __half2float(__ldg(xp + j)), acc);
            w >>= BITS;
        }
    }
    acc = warp_sum(acc);
    if (lane == 0) out[(int64_t)b * OC + oc] = __float2half_rn(acc);
}

// ------------------------------------------------------------------------------------------------
// host dispatch
// ------------------------------------------------------------------------------------------------
struct GemvArgs {
    const __half* A; int64_t a_stride;
    const uint32_t* qB; int64_t qb_us, qb_rs;
    const __half *S, *Z; int64_t sz_us, sz_rs;
    __half* C; int B, nh, nh_kv, K, N, g;
    cudaStream_t st;
};

template <int BITS, int G>
static int launch_ref_fast(const GemvArgs& a) {
    const int ratio = a.nh / a.nh_kv;
    const int ukv = a.B * a.nh_kv;
    if (a.N > 256) {
        dim3 grid(ukv, cdiv(cdiv(a.N, 1024), 4), ratio / G);
        bgemv_ref_wide_kernel<BITS, G><<<grid, 128, 0, a.st>>>(a.A, a.a_stride, a.qB, a.qb_us, a.qb_rs, a.S, a.Z,
                                                               a.sz_us, a.sz_rs, a.C, ratio, a.K, a.N, a.g);
    } else {
        int lg = 0;
        while ((32 << lg) < a.N) ++lg;
        const size_t smem = (size_t)8 * (1 << lg) * G * 33 * sizeof(float);
        if (smem > 48 * 1024)
            cudaFuncSetAttribute(bgemv_ref_tall_kernel<BITS, G>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
        dim3 grid(ukv, 1, ratio / G);
        bgemv_ref_tall_kernel<BITS, G><<<grid, 256, smem, a.st>>>(a.A, a.a_stride, a.qB, a.qb_us, a.qb_rs, a.S, a.Z,
                                                                  a.sz_us, a.sz_rs, a.C, ratio, a.K, a.N, a.g, lg);
    }
    return post_launch();
}

template <int BITS>
static int launch_bgemv(const GemvArgs& a, int layout) {
    constexpr int FPI = 32 / BITS;
    const int ratio = a.nh / a.nh_kv;
    const int uq = a.B * a.nh;
    if (layout == KIVI_LAYOUT_KERNEL) {
        dim3 grid(uq, cdiv(a.N / FPI, 4));
        bgemv_kernel_layout_kernel<BITS><<<grid, 128, 0, a.st>>>(a.A, a.a_stride, a.qB, a.qb_us, a.qb_rs, a.S, a.Z,
                                                                  a.sz_us, a.sz_rs, a.C, ratio, a.K, a.N, a.g);
        return post_launch();
    }
    if (!tuning().no_mma_gemv) {
        const int rc = bgemv_ref_mma(a.A, a.a_stride, a.qB, a.qb_us, a.qb_rs, a.S, a.Z, a.sz_us, a.sz_rs, a.C,
                                     a.B, a.nh, a.nh_kv, a.K, a.N, BITS, a.g, a.st);
        if (rc != KIVI_ERR_UNSUPPORTED) return rc;
    }
    constexpr int kCellBytes = 4 * BITS;                          // 32 elements
    const bool fast = (a.g % 32 == 0) &&
                      (reinterpret_cast<uintptr_t>(a.qB) % kCellBytes == 0) &&
                      ((a.qb_us * 4) % kCellBytes == 0) && ((a.qb_rs * 4) % kCellBytes == 0) &&
                      (reinterpret_cast<uintptr_t>(a.C) % 16 == 0);
    if (fast) {
        if (ratio % 4 == 0) return launch_ref_fast<BITS, 4>(a);
        if (ratio % 2 == 0) return launch_ref_fast<BITS, 2>(a);
        return launch_ref_fast<BITS, 1>(a);
    }
    dim3 grid(uq, cdiv(a.N, 128));
    bgemv_ref_generic_kernel<BITS><<<grid, 128, 0, a.st>>>(a.A, a.a_stride, a.qB, a.qb_us, a.qb_rs, a.S, a.Z,
                                                            a.sz_us, a.sz_rs, a.C, ratio, a.K, a.N, a.g);
    return post_launch();
}

}  // namespace kivi

extern "C" int kivi_bgemv_outer_f16(const void* A, int64_t a_stride,
                                    const void* qB, int64_t qb_unit_stride, int64_t qb_row_stride,
                                    const void* scales, const void* zeros, int64_t sz_unit_stride, int64_t sz_row_stride,
                                    void* C, int B, int nh, int nh_kv, int K, int N,
                                    int bits, int group_size, int layout, void* stream)
{
    if (!(bits == 2 || bits == 4 || (bits == 8 && layout == KIVI_LAYOUT_REFERENCE)))
        return KIVI_ERR_BITS;                                                      // quant/matmul.py:215
    if (nh_kv <= 0 || nh <= 0 || nh % nh_kv != 0) return KIVI_ERR_GQA;             // quant/matmul.py:216
    if (layout != KIVI_LAYOUT_REFERENCE && layout != KIVI_LAYOUT_KERNEL) return KIVI_ERR_LAYOUT;
    const int fpi = 32 / bits;
    if (B < 0 || K < 0 || N < 0) return KIVI_ERR_SHAPE;
    if (group_size <= 0 || group_size % fpi != 0) return KIVI_ERR_GROUP;
    if (N % group_size != 0) return KIVI_ERR_SHAPE;
    if (B == 0 || N == 0) return KIVI_OK;
    if (!A || !qB || !scales || !zeros || !C) return KIVI_ERR_NULL;
    if ((int64_t)B * nh > 0x7fffffff || (int64_t)N / 128 > 65535 * 4) return KIVI_ERR_UNSUPPORTED;   // grid.x = units, grid.y = column tiles
    kivi::GemvArgs a{(const __half*)A, a_stride, (const uint32_t*)qB, qb_unit_stride, qb_row_stride,
                     (const __half*)scales, (const __half*)zeros, sz_unit_stride, sz_row_stride,
                     (__half*)C, B, nh, nh_kv, K, N, group_size, (cudaStream_t)stream};
    if (bits == 8) {   // Triton-surface only (quant/matmul.py:112-175 accepts 8-bit): slow exact path
        dim3 grid(B * nh, kivi::cdiv(N, 128));
        kivi::bgemv_ref_generic_kernel<8><<<grid, 128, 0, a.st>>>(a.A, a.a_stride, a.qB, a.qb_us, a.qb_rs, a.S, a.Z,
                                                               a.sz_us, a.sz_rs, a.C, nh / nh_kv, K, N, group_size);
        return kivi::post_launch();
    }
    return bits == 2 ? kivi::launch_bgemv<2>(a, layout) : kivi::launch_bgemv<4>(a, layout);
}

extern "C" int kivi_gemv_inner_f16(const void* in, const void* kernel, const void* scales, const void* zeros,
                                   void* out, int Bn, int IC, int OC, int bits, int group_size, int64_t sf_w,
                                   void* stream)
{
    if (!(bits == 2 || bits == 4 || bits == 8)) return KIVI_ERR_BITS;
    const int fpi = 32 / bits;
    if (group_size <= 0 || group_size % fpi != 0) return KIVI_ERR_GROUP;
    if (Bn < 0 || IC < 0 || OC < 0 || IC % fpi != 0) return KIVI_ERR_SHAPE;
    if (sf_w < kivi::cdiv(IC, group_size)) return KIVI_ERR_SHAPE;
    if (Bn == 0 || OC == 0) return KIVI_OK;
    if (!in || !kernel || !scales || !zeros || !out) return KIVI_ERR_NULL;
    dim3 grid(Bn, kivi::cdiv(OC, 4));
    cudaStream_t st = (cudaStream_t)stream;
    #define KIVI_INNER(BITS_) kivi::gemv_inner_kernel<BITS_><<<grid, 128, 0, st>>>( \
        (const __half*)in, (const uint32_t*)kernel, (const __half*)scales, (const __half*)zeros, (__half*)out, \
        IC, OC, group_size, sf_w)
    if (bits == 2) KIVI_INNER(2); else if (bits == 4) KIVI_INNER(4); else KIVI_INNER(8);
    #undef KIVI_INNER
    return kivi::post_launch();
}
