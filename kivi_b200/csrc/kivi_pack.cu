// kivi_pack.cu -- fused asymmetric min/max quantise + bit-pack along the last dim (sm_90a).
//
// Replaces triton_quantize_and_pack_along_last_dim (quant/new_pack.py:217-252): Triton min/max
// kernel (:158-177) + 6 ATen elementwise kernels (:238-242, incl. an int32 temp 16x the packed
// size) + zeros + Triton OR-pack kernel (:132-154) become ONE kernel that reads x once
// (128-bit loads) and writes code/scale/mn once.  Bit-exact against the reference chain (quant_scale / quant_code):
//   d = fp16(mx - mn); scale = fp16(d / (2^b - 1)); t1 = fp16(x - mn); t2 = fp16(t1 / scale);
//   q = int(rint(clamp(t2, 0, 2^b - 1)))   (NaN from 0/0 -> 0, the CUDA cvt result)
#include "kivi_common.cuh"

namespace kivi {

// One thread = one output word (fpi = 32/BITS consecutive elements).  LPG = lanes per group =
// group_size / fpi, a power of two <= 32, so a group never straddles a warp.
template <int BITS, bool VEC>
__global__ void __launch_bounds__(256)
pack_lastdim_kernel(const __half* __restrict__ x, int64_t n_words, int lpg_log2,
                    int32_t* __restrict__ code, __half* __restrict__ scale, __half* __restrict__ mn_out)
{
    constexpr int FPI = 32 / BITS;
    const int64_t wid = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    const bool active = wid < n_words;
    const float maxq = (float)((1 << BITS) - 1);

    float v[FPI];
    if (active) {
        const __half* src = x + wid * FPI;
        if constexpr (VEC) {
            constexpr int NV = (FPI * 2 + 15) / 16;                 // uint4 loads per word
            if constexpr (FPI * 2 >= 16) {
                #pragma unroll
                for (int j = 0; j < NV; ++j) {
                    const uint4 u = __ldg(reinterpret_cast<const uint4*>(src) + j);
                    const __half2* h = reinterpret_cast<const __half2*>(&u);
                    #pragma unroll
                    for (int e = 0; e < 4; ++e) {
                        v[j * 8 + 2 * e] = __low2float(h[e]);
                        v[j * 8 + 2 * e + 1] = __high2float(h[e]);
                    }
                }
            } else {                                                // 8-bit: 4 halfs = 8 B
                const uint2 u = __ldg(reinterpret_cast<const uint2*>(src));
                const __half2* h = reinterpret_cast<const __half2*>(&u);
                v[0] = __low2float(h[0]); v[1] = __high2float(h[0]);
                v[2] = __low2float(h[1]); v[3] = __high2float(h[1]);
            }
        } else {
            #pragma unroll
            for (int j = 0; j < FPI; ++j) v[j] = __half2float(src[j]);
        }
    } else {
        #pragma unroll
        for (int j = 0; j < FPI; ++j) v[j] = 0.f;
    }
    float mnf = v[0], mxf = v[0];
    #pragma unroll
    for (int j = 1; j < FPI; ++j) { mnf = fminf(mnf, v[j]); mxf = fmaxf(mxf, v[j]); }
    // group-wide min/max across the LPG lanes that share the group (exact: values are fp16)
    for (int o = 1; o < (1 << lpg_log2); o <<= 1) {
        mnf = fminf(mnf, __shfl_xor_sync(0xffffffffu, mnf, o));
        mxf = fmaxf(mxf, __shfl_xor_sync(0xffffffffu, mxf, o));
    }
    if (!active) return;
    const __half sc = quant_scale(mnf, mxf, BITS);
    const float scf = __half2float(sc), rcp = __frcp_rn(scf);
    uint32_t word = 0;
    #pragma unroll
    for (int j = 0; j < FPI; ++j) word |= quant_code(v[j], mnf, scf, rcp, maxq) << (BITS * j);
    code[wid] = (int32_t)word;
    if ((wid & ((1 << lpg_log2) - 1)) == 0) {
        const int64_t gid = wid >> lpg_log2;
        scale[gid] = sc;
        mn_out[gid] = __float2half_rn(mnf);
    }
}

// Fallback for group sizes whose lanes-per-group is not a power of two <= 32 (or g % fpi != 0):
// one thread per word, each element rescans its own group.  Correct for every (g, bits) the
// reference accepts; never on the decode path.
template <int BITS>
__global__ void __launch_bounds__(256)
pack_lastdim_generic_kernel(const __half* __restrict__ x, int64_t n_words, int g,
                            int32_t* __restrict__ code, __half* __restrict__ scale, __half* __restrict__ mn_out)
{
    constexpr int FPI = 32 / BITS;
    const int64_t wid = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (wid >= n_words) return;
    const float maxq = (float)((1 << BITS) - 1);
    uint32_t word = 0;
    int64_t last_gid = -1;
    float mnf = 0.f, scf = 0.f, rcp = 0.f;
    for (int j = 0; j < FPI; ++j) {
        const int64_t e = wid * FPI + j;
        const int64_t gid = e / g;
        if (gid != last_gid) {
            const __half* gp = x + gid * g;
            float mxf;
            mnf = mxf = __half2float(gp[0]);
            for (int i = 1; i < g; ++i) { const float t = __half2float(gp[i]); mnf = fminf(mnf, t); mxf = fmaxf(mxf, t); }
            const __half sc = quant_scale(mnf, mxf, BITS);
            scf = __half2float(sc);
            rcp = __frcp_rn(scf);
            if (e == gid * g) { scale[gid] = sc; mn_out[gid] = __float2half_rn(mnf); }
            last_gid = gid;
        }
        word |= quant_code(__half2float(x[e]), mnf, scf, rcp, maxq) << (BITS * j);
    }
    code[wid] = (int32_t)word;
}

template <int BITS>
static int launch_pack(const void* x, int64_t rows, int64_t T, int g, void* code, void* scale, void* mn,
                       cudaStream_t st)
{
    constexpr int FPI = 32 / BITS;
    const int64_t n_words = rows * (T / FPI);
    if (n_words == 0) return KIVI_OK;
    const int64_t blocks = cdiv64(n_words, 256);
    if (blocks > 0x7fffffffLL) return KIVI_ERR_SHAPE;
    const int lpg = g / FPI;
    const bool pow2 = (g % FPI == 0) && lpg >= 1 && lpg <= 32 && (lpg & (lpg - 1)) == 0;
    if (pow2) {
        int lg = 0;
        while ((1 << lg) < lpg) ++lg;
        const bool vec = (reinterpret_cast<uintptr_t>(x) % 16) == 0;
        if (vec)
            pack_lastdim_kernel<BITS, true><<<(unsigned)blocks, 256, 0, st>>>(
                (const __half*)x, n_words, lg, (int32_t*)code, (__half*)scale, (__half*)mn);
        else
            pack_lastdim_kernel<BITS, false><<<(unsigned)blocks, 256, 0, st>>>(
                (const __half*)x, n_words, lg, (int32_t*)code, (__half*)scale, (__half*)mn);
    } else {
        pack_lastdim_generic_kernel<BITS><<<(unsigned)blocks, 256, 0, st>>>(
            (const __half*)x, n_words, g, (int32_t*)code, (__half*)scale, (__half*)mn);
    }
    return post_launch();
}

// Unpack + dequantise along the last dim in fp16 (data.to(fp16) * scale + mn, each op rounded to
// fp16), quant/new_pack.py:69-83 (V) and :51-66 (K, after a transpose).  One thread per word.
template <int BITS>
__global__ void __launch_bounds__(256)
unpack_dequant_lastdim_kernel(const uint32_t* __restrict__ code, const __half* __restrict__ scale,
                              const __half* __restrict__ mn, int64_t n_words, int g, __half* __restrict__ out)
{
    constexpr int FPI = 32 / BITS;
    const int64_t wid = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (wid >= n_words) return;
    const uint32_t w = code[wid];
    #pragma unroll
    for (int j = 0; j < FPI; ++j) {
        const int64_t e = wid * FPI + j;
        const int64_t gid = e / g;
        const __half c = __float2half_rn((float)((w >> (BITS * j)) & ((1u << BITS) - 1u)));
        out[e] = __hadd_rn(__hmul_rn(c, scale[gid]), mn[gid]);   // two roundings: no HFMA contraction
    }
}

}  // namespace kivi

extern "C" int kivi_unpack_dequant_lastdim_f16(const void* code, const void* scale, const void* mn,
                                               int64_t rows, int64_t T, int group_size, int bits,
                                               void* out, void* stream)
{
    if (!(bits == 2 || bits == 4 || bits == 8)) return KIVI_ERR_BITS;
    if (rows < 0 || T < 0 || group_size <= 0 || T % group_size != 0 || T % (32 / bits) != 0) return KIVI_ERR_SHAPE;
    if (rows == 0 || T == 0) return KIVI_OK;
    if (!code || !scale || !mn || !out) return KIVI_ERR_NULL;
    const int64_t n_words = rows * (T / (32 / bits));
    const int64_t blocks = kivi::cdiv64(n_words, 256);
    if (blocks > 0x7fffffffLL) return KIVI_ERR_SHAPE;
    cudaStream_t st = (cudaStream_t)stream;
    if (bits == 2)
        kivi::unpack_dequant_lastdim_kernel<2><<<(unsigned)blocks, 256, 0, st>>>((const uint32_t*)code, (const __half*)scale, (const __half*)mn, n_words, group_size, (__half*)out);
    else if (bits == 4)
        kivi::unpack_dequant_lastdim_kernel<4><<<(unsigned)blocks, 256, 0, st>>>((const uint32_t*)code, (const __half*)scale, (const __half*)mn, n_words, group_size, (__half*)out);
    else
        kivi::unpack_dequant_lastdim_kernel<8><<<(unsigned)blocks, 256, 0, st>>>((const uint32_t*)code, (const __half*)scale, (const __half*)mn, n_words, group_size, (__half*)out);
    return kivi::post_launch();
}

extern "C" int kivi_pack_lastdim_f16(const void* x, int64_t rows, int64_t T, int group_size, int bits,
                                     void* code, void* scale, void* mn, void* stream)
{
    if (!(bits == 2 || bits == 4 || bits == 8)) return KIVI_ERR_BITS;
    if (rows < 0 || T < 0 || group_size <= 0) return KIVI_ERR_SHAPE;
    if (T % group_size != 0 || T % (32 / bits) != 0) return KIVI_ERR_SHAPE;       // quant/new_pack.py:222
    if (rows == 0 || T == 0) return KIVI_OK;
    if (!x || !code || !scale || !mn) return KIVI_ERR_NULL;
    cudaStream_t st = (cudaStream_t)stream;
    switch (bits) {
        case 2: return kivi::launch_pack<2>(x, rows, T, group_size, code, scale, mn, st);
        case 4: return kivi::launch_pack<4>(x, rows, T, group_size, code, scale, mn, st);
        default: return kivi::launch_pack<8>(x, rows, T, group_size, code, scale, mn, st);
    }
}
