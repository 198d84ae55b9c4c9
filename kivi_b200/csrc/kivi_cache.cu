// kivi_cache.cu -- pre-allocated, blocked KIVI cache: sizing, prefill pack, state advance, export to
// the reference's 9-tuple layout (sm_90a).  Layout: kivi_decode.cuh.
//
// Replaces the cache handling of LlamaFlashAttention_KIVI.forward (models/llama_kivi.py):
//   prefill split + pack  :425-452   -> kivi_cache_prefill_f16 (fused transpose + quantise + fragment pack of
//                                       K, no .transpose(2,3).contiguous() temp; same kernel for V)
//   torch.cat growth      :350-352, :393-395, :391 -> nothing: blocks / ring slots are written in place
//   9-tuple               :454-455   -> kivi_cache_export_f16 (tests / interop only)
// Continuous batching (no counterpart in the reference): kivi_cache_refill_f16 re-runs the prefill kernels for one sequence
// of a live cache, kivi_cache_shift_f16 / kivi_cache_shift_state drop the oldest blocks of the shared timeline.
// Beam search (the reference's _reorder_cache, :950-957, without the 9-tuples): kivi_cache_reorder_f16 makes batch rows
// copies of other rows on the device.
#include "kivi_decode.cuh"

namespace kivi {

// ------------------------------------------------------------------------------------------------
// Where the prefill kernels write.  A prefill fills every unit from its own prompt: FillDesc{} (all zero).  A refill
// (kivi_cache_refill_f16) fills the units u0 .. u0 + Hkv - 1 of one sequence of a live cache with a T-token sequence x
// whose first s positions repeat the first real token, x[p] = src[max(p - s, 0)]; window token i of V lands in ring slot
// (ring + i) % v_res_cap; `state` is read, not written, and must hold the lengths the host passed (tk, tv; T = n + s).
// ------------------------------------------------------------------------------------------------
struct FillDesc { int u0, s, ring, refill, tk, tv; };

// a refill whose lengths differ from the device's `state` writes nothing (residual_prefill_kernel flags it)
__device__ __forceinline__ bool fill_refused(const CacheDesc& c, const FillDesc& f, int T) {
    if (!f.refill) return false;
    const int* st = c.state;
    return st[ST_TK] != f.tk || st[ST_R] != T - f.tk || st[ST_TV] != f.tv || st[ST_L] != T - f.tv ||
           st[ST_VHEAD] != f.ring || st[ST_KVLEN] != T;
}

// ------------------------------------------------------------------------------------------------
// Prefill: one CTA per (unit, block of 128 tokens).  The [128 tokens][128 channels] fp16 tile is staged in
// shared memory; quantisation runs along the OUTER dim of the block in groups of g (K: tokens of a channel,
// V: channels of a token); the codes are then gathered into the A-fragment words of the block.
//   IS_K = true : inner = channel, outer = token     IS_K = false: inner = token, outer = channel
// x holds n rows per unit (grid.y indexes the units of x; the cache unit is f.u0 + grid.y).
// ------------------------------------------------------------------------------------------------
template <int BITS, bool IS_K>
__global__ void __launch_bounds__(256)
block_prefill_kernel(CacheDesc c, const __half* __restrict__ x, int n, int nq, FillDesc f)
{
    extern __shared__ __align__(16) uint8_t sm[];
    __half (*tile)[kD + 8] = reinterpret_cast<__half (*)[kD + 8]>(sm);               // [token][channel]
    uint8_t (*codes)[kD + 4] = reinterpret_cast<uint8_t (*)[kD + 4]>(sm + kBlockTokens * (kD + 8) * 2);  // [inner][outer]
    if (fill_refused(c, f, n + f.s)) return;
    const int u = f.u0 + blockIdx.y, blk = blockIdx.x;
    const int t0 = blk * kBlockTokens;
    const int nt = min(kBlockTokens, nq - t0);
    const __half* src = x + (int64_t)blockIdx.y * n * kD;
    for (int i = threadIdx.x; i < nt * (kD / 8); i += blockDim.x) {
        const int t = i / (kD / 8), p = i % (kD / 8);
        const int row = max(t0 + t - f.s, 0);                                      // pad positions repeat source row 0
        *reinterpret_cast<uint4*>(&tile[t][p * 8]) = __ldg(reinterpret_cast<const uint4*>(src + (int64_t)row * kD) + p);
    }
    for (int i = threadIdx.x; i < kD * (kD + 4); i += blockDim.x) (&codes[0][0])[i] = 0;
    __syncthreads();
    const int g = c.g;
    const float maxq = (float)((1 << BITS) - 1);
    const int bb = lay_block_bytes(BITS, g);
    const int cap = IS_K ? c.k_cap_blocks : c.v_cap_blocks;
    uint8_t* blkp = (IS_K ? c.k_store : c.v_store) + ((int64_t)u * cap + blk) * bb;
    auto val = [&](int inner, int outer) -> float {
        return __half2float(IS_K ? tile[outer][inner] : tile[inner][outer]);
    };
    const int n_inner = IS_K ? kD : nt;                  // valid inner indices
    const int n_outer = IS_K ? nt : kD;                  // valid outer indices (multiple of g)
    for (int w = threadIdx.x; w < n_inner * (n_outer / g); w += blockDim.x) {
        const int inner = w % n_inner, G = w / n_inner;
        float mnf = val(inner, G * g), mxf = mnf;
        for (int i = 1; i < g; ++i) { const float v = val(inner, G * g + i); mnf = fminf(mnf, v); mxf = fmaxf(mxf, v); }
        const __half sc = quant_scale(mnf, mxf, BITS);
        const float scf = __half2float(sc), rcp = __frcp_rn(scf);
        for (int i = 0; i < g; ++i) codes[inner][G * g + i] = (uint8_t)quant_code(val(inner, G * g + i), mnf, scf, rcp, maxq);
        *reinterpret_cast<__half*>(blkp + lay_scale_off(BITS, g, inner, G)) = sc;
        *reinterpret_cast<__half*>(blkp + lay_zero_off(BITS, g, inner, G)) = __float2half_rn(mnf);
    }
    __syncthreads();
    // gather: one thread per word
    for (int w = threadIdx.x; w < Lay<BITS>::kCodeBytes / 4; w += blockDim.x)
        reinterpret_cast<uint32_t*>(blkp)[w] = lay_word(BITS, w, [&](int inner, int outer) -> uint32_t { return codes[inner][outer]; });
}

// residual windows of the prompt + state (a refill leaves `state` alone, or flags lengths that differ from it)
__global__ void __launch_bounds__(256)
residual_prefill_kernel(CacheDesc c, const __half* __restrict__ k, const __half* __restrict__ v, int n,
                        int nqk, int nqv, FillDesc f)
{
    const int T = n + f.s;
    if (fill_refused(c, f, T)) {
        if (blockIdx.x == 0 && threadIdx.x == 0) atomicOr(&c.state[6], KIVI_STATE_ERR_LENGTHS);
        return;
    }
    const int u = f.u0 + blockIdx.x;
    const int r = T - nqk, L = T - nqv;
    const uint4* ks = reinterpret_cast<const uint4*>(k + (int64_t)blockIdx.x * n * kD);
    const uint4* vs = reinterpret_cast<const uint4*>(v + (int64_t)blockIdx.x * n * kD);
    for (int i = threadIdx.x; i < r * (kD / 8); i += blockDim.x)                 // window rows are unit-swizzled (win_unit)
        reinterpret_cast<uint4*>(c.k_res + (int64_t)u * c.R * kD)[win_unit(i / 16, i % 16)] =
            __ldg(ks + (int64_t)max(nqk + i / 16 - f.s, 0) * 16 + i % 16);
    for (int i = threadIdx.x; i < L * (kD / 8); i += blockDim.x)
        reinterpret_cast<uint4*>(c.v_res + (int64_t)u * c.v_res_cap * kD)[win_unit((f.ring + i / 16) % c.v_res_cap, i % 16)] =
            __ldg(vs + (int64_t)max(nqv + i / 16 - f.s, 0) * 16 + i % 16);
    if (!f.refill && u == 0 && threadIdx.x == 0) {
        c.state[ST_TK] = nqk; c.state[ST_R] = r; c.state[ST_TV] = nqv; c.state[ST_L] = L;
        c.state[ST_VHEAD] = 0; c.state[ST_KVLEN] = n; c.state[6] = 0; c.state[7] = 0;
    }
}

// ------------------------------------------------------------------------------------------------
// Timeline shift: drop the first d blocks of every unit's K and V store (block j -> j - d) so that the shared length can
// shrink.  One CTA per (unit, store) moves the bytes of blocks [d, nblk) down by d blocks, D = d blocks at a time: chunk
// i reads [(i+1)D, (i+2)D) and writes [iD, (i+1)D), which chunk i - 1 read; a CTA barrier per chunk orders the overlap.
// The windows do not move; the vacated last d blocks are zeroed.  The device lengths must be those the host passed (else: nothing moves, state[6] flagged).
// ------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256)
shift_blocks_kernel(CacheDesc c, int d, int tk, int tv)
{
    if (c.state[ST_TK] != tk || c.state[ST_TV] != tv) {
        if (blockIdx.x == 0 && blockIdx.y == 0 && threadIdx.x == 0) atomicOr(&c.state[6], KIVI_STATE_ERR_LENGTHS);
        return;
    }
    const int u = blockIdx.x, isv = blockIdx.y;
    const int bb = lay_block_bytes(isv ? c.v_bits : c.k_bits, c.g);
    const int nblk = cdiv(isv ? tv : tk, kBlockTokens);                          // blocks holding tokens before the shift
    uint4* base = reinterpret_cast<uint4*>((isv ? c.v_store : c.k_store) + (int64_t)u * (isv ? c.v_cap_blocks : c.k_cap_blocks) * bb);
    const int64_t D = (int64_t)d * bb / 16, total = (int64_t)(nblk - d) * bb / 16;
    constexpr int kUnroll = 4;                                                   // loads in flight per thread before its stores
    for (int64_t c0 = 0; c0 < total; c0 += D) {
        const int64_t cnt = min(D, total - c0);
        for (int64_t i = threadIdx.x; i < cnt; i += kUnroll * blockDim.x) {
            uint4 t[kUnroll];
            #pragma unroll
            for (int e = 0; e < kUnroll; ++e)
                if (i + e * blockDim.x < cnt) t[e] = base[c0 + D + i + e * blockDim.x];
            #pragma unroll
            for (int e = 0; e < kUnroll; ++e)
                if (i + e * blockDim.x < cnt) base[c0 + i + e * blockDim.x] = t[e];
        }
        __syncthreads();
    }
    // the d blocks that held tokens and now lie past the end are cleared, as a prefill or an import leaves them
    for (int64_t i = threadIdx.x; i < D; i += blockDim.x) base[total + i] = make_uint4(0u, 0u, 0u, 0u);
}

// the lengths after a shift (once per model, after every layer's shift_blocks_kernel); kv_start: NULL or [B]
__global__ void shift_state_kernel(int* state, int shift, int32_t* kv_start, int B)
{
    const bool ok = state[ST_TK] >= shift && state[ST_TV] >= shift;
    __syncthreads();
    if (!ok) {
        if (threadIdx.x == 0) atomicOr(&state[6], KIVI_STATE_ERR_LENGTHS);
        return;
    }
    if (kv_start)
        for (int b = threadIdx.x; b < B; b += blockDim.x) kv_start[b] -= shift;
    if (threadIdx.x == 0) {
        state[ST_TK] -= shift; state[ST_TV] -= shift; state[ST_KVLEN] -= shift;
    }
}

// One decode step's bookkeeping (models/llama_kivi.py:343-356, :386-399): the data movement is done by
// the decode kernels per unit; the lengths advance here, once per step for all layers.
__global__ void advance_kernel(int* state, int R, int v_res_cap)
{
    int tk = state[ST_TK], r = state[ST_R], tv = state[ST_TV], L = state[ST_L], vh = state[ST_VHEAD];
    r += 1;
    if (r == R) { tk += R; r = 0; }
    L += 1;
    if (L > R) { tv += 1; vh = (vh + 1) % v_res_cap; L = R; }
    state[ST_TK] = tk; state[ST_R] = r; state[ST_TV] = tv; state[ST_L] = L; state[ST_VHEAD] = vh;
    state[ST_KVLEN] += 1;
}

// ------------------------------------------------------------------------------------------------
// export to the reference layouts (the 9-tuple of models/llama_kivi.py:454-455)
//   K: code [U][128][tk/fpi] words, scale/mn [U][128][tk/g]       (packed along tokens per channel)
//   V: code [U][tv][128/fpi] words, scale/mn [U][tv][128/g]       (packed along channels per token)
// ------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256)
export_kv_kernel(CacheDesc c, int tk, int tv, int L, int vhead, int r,
                 uint32_t* __restrict__ k_code, __half* __restrict__ k_scale, __half* __restrict__ k_mn,
                 uint32_t* __restrict__ v_code, __half* __restrict__ v_scale, __half* __restrict__ v_mn,
                 __half* __restrict__ k_full, __half* __restrict__ v_full)
{
    const int u = blockIdx.y, g = c.g;
    const int stride = gridDim.x * blockDim.x, tid = blockIdx.x * blockDim.x + threadIdx.x;
    {   // K
        const int bits = c.k_bits, fpi = 32 / bits, wpr = tk / fpi, gpr = tk / g;
        const int bb = lay_block_bytes(bits, g);
        const uint8_t* ub = c.k_store + (int64_t)u * c.k_cap_blocks * bb;
        for (int i = tid; i < kD * wpr; i += stride) {
            const int d = i / wpr, w = i % wpr;
            uint32_t word = 0;
            for (int e = 0; e < fpi; ++e) {
                const int tok = w * fpi + e, blk = tok / kBlockTokens, o = tok % kBlockTokens;
                const uint32_t src = *reinterpret_cast<const uint32_t*>(ub + (int64_t)blk * bb + lay_word_off(bits, d, o));
                word |= ((src >> lay_bit_pos(bits, d, o)) & ((1u << bits) - 1u)) << (bits * e);
            }
            k_code[((int64_t)u * kD + d) * wpr + w] = word;
        }
        for (int i = tid; i < kD * gpr; i += stride) {
            const int d = i / gpr, gi = i % gpr;
            const int tok = gi * g, blk = tok / kBlockTokens, G = (tok % kBlockTokens) / g;
            k_scale[((int64_t)u * kD + d) * gpr + gi] = *reinterpret_cast<const __half*>(ub + (int64_t)blk * bb + lay_scale_off(bits, g, d, G));
            k_mn[((int64_t)u * kD + d) * gpr + gi] = *reinterpret_cast<const __half*>(ub + (int64_t)blk * bb + lay_zero_off(bits, g, d, G));
        }
    }
    {   // V
        const int bits = c.v_bits, fpi = 32 / bits, wpt = kD / fpi, gpt = kD / g;
        const int bb = lay_block_bytes(bits, g);
        const uint8_t* ub = c.v_store + (int64_t)u * c.v_cap_blocks * bb;
        for (int i = tid; i < tv * wpt; i += stride) {
            const int t = i / wpt, w = i % wpt;
            const int blk = t / kBlockTokens, inner = t % kBlockTokens;
            uint32_t word = 0;
            for (int e = 0; e < fpi; ++e) {
                const int o = w * fpi + e;
                const uint32_t src = *reinterpret_cast<const uint32_t*>(ub + (int64_t)blk * bb + lay_word_off(bits, inner, o));
                word |= ((src >> lay_bit_pos(bits, inner, o)) & ((1u << bits) - 1u)) << (bits * e);
            }
            v_code[(int64_t)u * tv * wpt + i] = word;
        }
        for (int i = tid; i < tv * gpt; i += stride) {
            const int t = i / gpt, G = i % gpt;
            const int blk = t / kBlockTokens, inner = t % kBlockTokens;
            v_scale[(int64_t)u * tv * gpt + i] = *reinterpret_cast<const __half*>(ub + (int64_t)blk * bb + lay_scale_off(bits, g, inner, G));
            v_mn[(int64_t)u * tv * gpt + i] = *reinterpret_cast<const __half*>(ub + (int64_t)blk * bb + lay_zero_off(bits, g, inner, G));
        }
    }
    for (int i = tid; i < r * kD; i += stride)
        k_full[(int64_t)u * r * kD + i] = c.k_res[(int64_t)u * c.R * kD + win_off(i / kD, i % kD)];
    for (int i = tid; i < L * kD; i += stride) {
        const int t = i / kD, d = i % kD;
        v_full[(int64_t)u * L * kD + i] = c.v_res[(int64_t)u * c.v_res_cap * kD + win_off((vhead + t) % c.v_res_cap, d)];
    }
}

// ------------------------------------------------------------------------------------------------
// import from the reference layouts: the inverse of export_kv_kernel.  One thread per destination word / meta half / window
// element; every byte of the blocks that hold imported tokens is written (codes of tokens past the end are zero).
// ------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256)
import_kv_kernel(CacheDesc c, int tk, int tv, int L, int r,
                 const uint32_t* __restrict__ k_code, const __half* __restrict__ k_scale, const __half* __restrict__ k_mn,
                 const uint32_t* __restrict__ v_code, const __half* __restrict__ v_scale, const __half* __restrict__ v_mn,
                 const __half* __restrict__ k_full, const __half* __restrict__ v_full)
{
    const int u = blockIdx.y, g = c.g, ngrp = 128 / g;
    const int stride = gridDim.x * blockDim.x, tid = blockIdx.x * blockDim.x + threadIdx.x;
    for (int isv = 0; isv < 2; ++isv) {                    // 0: K store (inner = channel, outer = token), 1: V store
        const int bits = isv ? c.v_bits : c.k_bits, fpi = 32 / bits, n_tok = isv ? tv : tk;
        const int wpb = lay_code_bytes(bits) / 4;          // words per block
        const int bb = lay_block_bytes(bits, g), nblk = cdiv(n_tok, kBlockTokens);
        uint8_t* ub = (isv ? c.v_store : c.k_store) + (int64_t)u * (isv ? c.v_cap_blocks : c.k_cap_blocks) * bb;
        const uint32_t* code = isv ? v_code : k_code;
        const __half* sc = isv ? v_scale : k_scale;
        const __half* mn = isv ? v_mn : k_mn;
        const int wpr_k = tk / fpi, gpr_k = tk / g;        // K: words / groups per channel row
        const int wpt_v = kD / fpi, gpt_v = kD / g;        // V: words / groups per token row
        for (int i = tid; i < nblk * wpb; i += stride) {
            const int blk = i / wpb, w = i % wpb;
            reinterpret_cast<uint32_t*>(ub + (int64_t)blk * bb)[w] = lay_word(bits, w, [&](int inner, int o) -> uint32_t {
                if (!isv) {
                    const int tok = blk * kBlockTokens + o;
                    return tok < tk ? (code[((int64_t)u * kD + inner) * wpr_k + tok / fpi] >> (bits * (tok % fpi))) & ((1u << bits) - 1u) : 0u;
                }
                const int tok = blk * kBlockTokens + inner;
                return tok < tv ? (code[((int64_t)u * tv + tok) * wpt_v + o / fpi] >> (bits * (o % fpi))) & ((1u << bits) - 1u) : 0u;
            });
        }
        for (int i = tid; i < nblk * 128 * ngrp; i += stride) {
            const int blk = i / (128 * ngrp), inner = (i / ngrp) % 128, G = i % ngrp;
            __half s = __float2half_rn(0.f), z = s;
            if (!isv) {
                const int tok = blk * kBlockTokens + G * g;
                if (tok < tk) { s = sc[((int64_t)u * kD + inner) * gpr_k + tok / g]; z = mn[((int64_t)u * kD + inner) * gpr_k + tok / g]; }
            } else {
                const int tok = blk * kBlockTokens + inner;
                if (tok < tv) { s = sc[((int64_t)u * tv + tok) * gpt_v + G]; z = mn[((int64_t)u * tv + tok) * gpt_v + G]; }
            }
            *reinterpret_cast<__half*>(ub + (int64_t)blk * bb + lay_scale_off(bits, g, inner, G)) = s;
            *reinterpret_cast<__half*>(ub + (int64_t)blk * bb + lay_zero_off(bits, g, inner, G)) = z;
        }
    }
    for (int i = tid; i < r * kD; i += stride)
        c.k_res[(int64_t)u * c.R * kD + win_off(i / kD, i % kD)] = k_full[(int64_t)u * r * kD + i];
    for (int i = tid; i < L * kD; i += stride)
        c.v_res[(int64_t)u * c.v_res_cap * kD + win_off(i / kD, i % kD)] = v_full[(int64_t)u * L * kD + i];
    if (u == 0 && tid == 0) {
        c.state[ST_TK] = tk; c.state[ST_R] = r; c.state[ST_TV] = tv; c.state[ST_L] = L;
        c.state[ST_VHEAD] = 0; c.state[ST_KVLEN] = tk + r; c.state[6] = 0; c.state[7] = 0;
    }
}

// ------------------------------------------------------------------------------------------------
// Row reorder (beam search): sequence b's units become a copy of sequence src[b]'s units as they were before the call.
// A unit's bytes are four regions: the live packed K blocks, the live packed V blocks (lengths from `state`), the whole
// fp16 K window and the whole V ring.  The scratch holds one full-capacity slot per (row, unit), regions at the same
// offsets, so the staging and the copy address source and destination alike.
//   launch 1 (STAGE): row s is staged when it is rewritten (src[s] != s) and another rewritten row reads it;
//   launch 2        : every rewritten row b copies from row s = src[b]: from the scratch if s was staged, else from the
//                     cache, whose row s this call does not write.
// One CTA per (unit of a row, chunk); grid.y = rows.  Any src outside [0, B) stops every CTA before it writes.
// ------------------------------------------------------------------------------------------------
constexpr int kReorderChunks = 4;                                                // CTAs per unit

struct ReorderDesc { int64_t kb, vb, kw, vw; };                                  // bytes of the four full-capacity regions

__device__ __forceinline__ void copy16(uint4* __restrict__ dst, const uint4* __restrict__ src, int64_t n, int lane, int stride)
{
    constexpr int kUnroll = 4;                                                   // loads in flight per thread before its stores
    for (int64_t i = lane; i < n; i += (int64_t)kUnroll * stride) {
        uint4 t[kUnroll];
        #pragma unroll
        for (int e = 0; e < kUnroll; ++e)
            if (i + (int64_t)e * stride < n) t[e] = src[i + (int64_t)e * stride];
        #pragma unroll
        for (int e = 0; e < kUnroll; ++e)
            if (i + (int64_t)e * stride < n) dst[i + (int64_t)e * stride] = t[e];
    }
}

template <bool STAGE>
__global__ void __launch_bounds__(256)
reorder_rows_kernel(CacheDesc c, const int32_t* __restrict__ src, uint8_t* __restrict__ scratch, ReorderDesc r)
{
    const int row = blockIdx.y, h = blockIdx.x / kReorderChunks, chunk = blockIdx.x % kReorderChunks;
    bool bad = false, read_by_other = false;
    for (int b = threadIdx.x; b < c.B; b += blockDim.x) {
        const int s = src[b];
        bad |= s < 0 || s >= c.B;
        read_by_other |= s == row && b != row;
    }
    bad = __syncthreads_or(bad);
    read_by_other = __syncthreads_or(read_by_other);
    if (bad) {
        if (!STAGE && blockIdx.x == 0 && row == 0 && threadIdx.x == 0) atomicOr(&c.state[6], KIVI_STATE_ERR_ROWS);
        return;
    }
    const int s = src[row];
    if (s == row || (STAGE && !read_by_other)) return;                          // nothing to stage / row kept
    const int64_t slot = r.kb + r.vb + r.kw + r.vw;                              // scratch bytes of one unit
    const int64_t kbb = lay_block_bytes(c.k_bits, c.g), vbb = lay_block_bytes(c.v_bits, c.g);
    const int64_t nk = (int64_t)min(cdiv(c.state[ST_TK], kBlockTokens), c.k_cap_blocks) * kbb;
    const int64_t nv = (int64_t)min(cdiv(c.state[ST_TV], kBlockTokens), c.v_cap_blocks) * vbb;
    // the unit's four regions in the cache (STAGE: the row itself; else: row s) and in the scratch
    const int64_t us = (int64_t)(STAGE ? row : s) * c.Hkv + h, ud = (int64_t)row * c.Hkv + h;
    const bool from_scratch = !STAGE && src[s] != s;                             // s is rewritten too: it was staged
    const uint8_t* in[4]; uint8_t* out[4];
    const uint8_t* cache_in[4] = {c.k_store + us * r.kb, c.v_store + us * r.vb,
                                  reinterpret_cast<const uint8_t*>(c.k_res) + us * r.kw,
                                  reinterpret_cast<const uint8_t*>(c.v_res) + us * r.vw};
    uint8_t* sc = scratch + us * slot;
    uint8_t* sc_regions[4] = {sc, sc + r.kb, sc + r.kb + r.vb, sc + r.kb + r.vb + r.kw};
    uint8_t* cache_out[4] = {c.k_store + ud * r.kb, c.v_store + ud * r.vb,
                             reinterpret_cast<uint8_t*>(c.k_res) + ud * r.kw, reinterpret_cast<uint8_t*>(c.v_res) + ud * r.vw};
    const int64_t bytes[4] = {nk, nv, r.kw, r.vw};
    #pragma unroll
    for (int i = 0; i < 4; ++i) {
        in[i] = STAGE ? cache_in[i] : (from_scratch ? sc_regions[i] : cache_in[i]);
        out[i] = STAGE ? sc_regions[i] : cache_out[i];
    }
    const int lane = chunk * blockDim.x + threadIdx.x, stride = kReorderChunks * blockDim.x;
    #pragma unroll
    for (int i = 0; i < 4; ++i)
        copy16(reinterpret_cast<uint4*>(out[i]), reinterpret_cast<const uint4*>(in[i]), bytes[i] / 16, lane, stride);
}

int make_desc(const kivi_cache_t* k, CacheDesc* d)
{
    if (!k) return KIVI_ERR_NULL;
    if (!(k->k_bits == 2 || k->k_bits == 4) || !(k->v_bits == 2 || k->v_bits == 4)) return KIVI_ERR_BITS;
    if (k->head_dim != kD) return KIVI_ERR_SHAPE;
    if (!(k->group_size == 32 || k->group_size == 64 || k->group_size == 128)) return KIVI_ERR_GROUP;
    if (k->residual_length <= 0 || k->residual_length % k->group_size != 0) return KIVI_ERR_SHAPE;   // llama_kivi.py:344
    if (!(k->residual_length == 32 || k->residual_length == 64 || k->residual_length == 128 || k->residual_length == 256))
        return KIVI_ERR_UNSUPPORTED;                  // a K flush must tile the 128-token blocks
    if (k->batch <= 0 || k->num_kv_heads <= 0 || k->num_heads % k->num_kv_heads != 0) return KIVI_ERR_GQA;
    if (k->k_cap_blocks <= 0 || k->v_cap_blocks <= 0) return KIVI_ERR_SHAPE;
    if (k->v_res_cap < k->residual_length + 1) return KIVI_ERR_SHAPE;
    if (!k->k_store || !k->v_store || !k->k_res || !k->v_res || !k->state) return KIVI_ERR_NULL;
    d->B = k->batch; d->Hkv = k->num_kv_heads; d->H = k->num_heads; d->k_bits = k->k_bits; d->v_bits = k->v_bits;
    d->g = k->group_size; d->R = k->residual_length; d->k_cap_blocks = k->k_cap_blocks; d->v_cap_blocks = k->v_cap_blocks;
    d->v_res_cap = k->v_res_cap;
    d->k_store = (uint8_t*)k->k_store; d->v_store = (uint8_t*)k->v_store;
    d->k_res = (__half*)k->k_res; d->v_res = (__half*)k->v_res; d->state = (int*)k->state;
    return KIVI_OK;
}

// host-passed lengths of a cache of tk + r == tv + L tokens: K flushed in whole windows, both windows within R
static bool lengths_ok(const CacheDesc& c, int tk, int r, int tv, int L)
{
    if (tk < 0 || r < 0 || tv < 0 || L < 0 || tk % c.R != 0 || r >= c.R || L > c.R || tk + r != tv + L) return false;
    return !(tv > 0 && L != c.R);                                   // the V store fills only once the window is full (:442-452)
}

// the launches of a prefill (f = FillDesc{}: n_units = B * Hkv) or of a refill of one sequence (n_units = Hkv):
// K store, V store, windows (+ state)
int launch_fill(const CacheDesc& c, const void* k, const void* v, int n, int nqk, int nqv, int n_units, FillDesc f,
                cudaStream_t st)
{
    const size_t smem = (size_t)kBlockTokens * (kD + 8) * 2 + (size_t)kD * (kD + 4);
    DeviceInfo di;
    int rc = device_info(&di);
    if (rc) return rc;
    static std::atomic<unsigned long long> optin[4];                 // 51.7 KB of dynamic shared memory: opt-in per device
    rc = ensure_dynamic_smem(block_prefill_kernel<2, true>, (int)smem, di.ordinal, optin[0]); if (rc) return rc;
    rc = ensure_dynamic_smem(block_prefill_kernel<4, true>, (int)smem, di.ordinal, optin[1]); if (rc) return rc;
    rc = ensure_dynamic_smem(block_prefill_kernel<2, false>, (int)smem, di.ordinal, optin[2]); if (rc) return rc;
    rc = ensure_dynamic_smem(block_prefill_kernel<4, false>, (int)smem, di.ordinal, optin[3]); if (rc) return rc;
    if (nqk > 0) {
        dim3 grid(cdiv(nqk, kBlockTokens), n_units);
        if (c.k_bits == 2) block_prefill_kernel<2, true><<<grid, 256, smem, st>>>(c, (const __half*)k, n, nqk, f);
        else               block_prefill_kernel<4, true><<<grid, 256, smem, st>>>(c, (const __half*)k, n, nqk, f);
        rc = post_launch(); if (rc) return rc;
    }
    if (nqv > 0) {
        dim3 grid(cdiv(nqv, kBlockTokens), n_units);
        if (c.v_bits == 2) block_prefill_kernel<2, false><<<grid, 256, smem, st>>>(c, (const __half*)v, n, nqv, f);
        else               block_prefill_kernel<4, false><<<grid, 256, smem, st>>>(c, (const __half*)v, n, nqv, f);
        rc = post_launch(); if (rc) return rc;
    }
    residual_prefill_kernel<<<n_units, 256, 0, st>>>(c, (const __half*)k, (const __half*)v, n, nqk, nqv, f);
    return post_launch();
}

}  // namespace kivi

using namespace kivi;

extern "C" int kivi_cache_sizes(int batch, int num_kv_heads, int k_bits, int v_bits, int group_size,
                                int residual_length, int max_tokens, int64_t* out /* [8] */)
{
    if (!out) return KIVI_ERR_NULL;
    if (!(k_bits == 2 || k_bits == 4) || !(v_bits == 2 || v_bits == 4)) return KIVI_ERR_BITS;
    if (!(group_size == 32 || group_size == 64 || group_size == 128)) return KIVI_ERR_GROUP;
    if (residual_length <= 0 || residual_length % group_size != 0 || batch <= 0 || num_kv_heads <= 0 || max_tokens <= 0)
        return KIVI_ERR_SHAPE;
    const int64_t U = (int64_t)batch * num_kv_heads;
    const int64_t capb = cdiv(max_tokens, kBlockTokens) + 1;
    const int64_t vres = residual_length + 1;
    out[0] = capb;                                                // k_cap_blocks
    out[1] = capb;                                                // v_cap_blocks
    out[2] = vres;                                                // v_res_cap
    out[3] = U * capb * lay_block_bytes(k_bits, group_size);      // bytes: k_store
    out[4] = U * capb * lay_block_bytes(v_bits, group_size);      // bytes: v_store
    out[5] = U * residual_length * kD * 2;                        // bytes: k_res
    out[6] = U * vres * kD * 2;                                   // bytes: v_res
    out[7] = 0;
    return KIVI_OK;
}

extern "C" int kivi_cache_prefill_f16(const kivi_cache_t* cache, const void* k, const void* v, int n, void* stream)
{
    CacheDesc c;
    int rc = make_desc(cache, &c);
    if (rc) return rc;
    if (n < 0) return KIVI_ERR_SHAPE;
    if (n > 0 && (!k || !v)) return KIVI_ERR_NULL;
    const int R = c.R;
    // models/llama_kivi.py:425-434 (K) and :442-449 (V)
    const int nqk = (n % R != 0) ? (n < R ? 0 : n - n % R) : n;
    const int nqv = (n <= R) ? 0 : n - R;
    if (cdiv(nqk, kBlockTokens) > c.k_cap_blocks || cdiv(nqv, kBlockTokens) > c.v_cap_blocks) return KIVI_ERR_CAPACITY;
    const int U = c.B * c.Hkv;
    if (U > 65535) return KIVI_ERR_UNSUPPORTED;                     // grid.y
    return launch_fill(c, k, v, n, nqk, nqv, U, FillDesc{0, 0, 0, 0, 0, 0}, (cudaStream_t)stream);
}

extern "C" int kivi_cache_refill_f16(const kivi_cache_t* cache, int seq, const void* k, const void* v, int n,
                                     int tk, int r, int tv, int L, int vhead, void* stream)
{
    CacheDesc c;
    int rc = make_desc(cache, &c);
    if (rc) return rc;
    if (seq < 0 || seq >= c.B) return KIVI_ERR_SHAPE;
    if (!lengths_ok(c, tk, r, tv, L)) return KIVI_ERR_SHAPE;
    if (vhead < 0 || vhead >= c.v_res_cap) return KIVI_ERR_SHAPE;
    const int T = tk + r;
    if (n < 1 || n > T) return KIVI_ERR_SHAPE;
    if (cdiv(tk, kBlockTokens) > c.k_cap_blocks || cdiv(tv, kBlockTokens) > c.v_cap_blocks) return KIVI_ERR_CAPACITY;
    if (!k || !v) return KIVI_ERR_NULL;
    return launch_fill(c, k, v, n, tk, tv, c.Hkv, FillDesc{seq * c.Hkv, T - n, vhead, 1, tk, tv}, (cudaStream_t)stream);
}

extern "C" int kivi_cache_shift_f16(const kivi_cache_t* cache, int shift, int tk, int tv, void* stream)
{
    CacheDesc c;
    int rc = make_desc(cache, &c);
    if (rc) return rc;
    if (shift <= 0 || shift % max(kBlockTokens, c.R) != 0 || shift > tk || shift > tv) return KIVI_ERR_SHAPE;
    if (cdiv(tk, kBlockTokens) > c.k_cap_blocks || cdiv(tv, kBlockTokens) > c.v_cap_blocks) return KIVI_ERR_CAPACITY;
    const int U = c.B * c.Hkv;
    shift_blocks_kernel<<<dim3(U, 2), 256, 0, (cudaStream_t)stream>>>(c, shift / kBlockTokens, tk, tv);
    return post_launch();
}

extern "C" int kivi_cache_shift_state(const kivi_cache_t* cache, int shift, int32_t* kv_start, void* stream)
{
    CacheDesc c;
    int rc = make_desc(cache, &c);
    if (rc) return rc;
    if (shift <= 0 || shift % max(kBlockTokens, c.R) != 0) return KIVI_ERR_SHAPE;
    shift_state_kernel<<<1, 256, 0, (cudaStream_t)stream>>>(c.state, shift, kv_start, c.B);
    return post_launch();
}

extern "C" int kivi_cache_advance(const kivi_cache_t* cache, void* stream)
{
    CacheDesc c;
    int rc = make_desc(cache, &c);
    if (rc) return rc;
    advance_kernel<<<1, 1, 0, (cudaStream_t)stream>>>(c.state, c.R, c.v_res_cap);
    return post_launch();
}

extern "C" int kivi_cache_export_f16(const kivi_cache_t* cache, int tk, int r, int tv, int L, int vhead,
                                     void* k_code, void* k_scale, void* k_mn, void* k_full,
                                     void* v_code, void* v_scale, void* v_mn, void* v_full, void* stream)
{
    CacheDesc c;
    int rc = make_desc(cache, &c);
    if (rc) return rc;
    if (tk > 0 && (!k_code || !k_scale || !k_mn)) return KIVI_ERR_NULL;
    if (tv > 0 && (!v_code || !v_scale || !v_mn)) return KIVI_ERR_NULL;
    const int U = c.B * c.Hkv;
    export_kv_kernel<<<dim3(8, U), 256, 0, (cudaStream_t)stream>>>(c, tk, tv, L, vhead, r,
        (uint32_t*)k_code, (__half*)k_scale, (__half*)k_mn, (uint32_t*)v_code, (__half*)v_scale, (__half*)v_mn,
        (__half*)k_full, (__half*)v_full);
    return post_launch();
}

extern "C" int kivi_cache_import_f16(const kivi_cache_t* cache, int tk, int r, int tv, int L,
                                     const void* k_code, const void* k_scale, const void* k_mn, const void* k_full,
                                     const void* v_code, const void* v_scale, const void* v_mn, const void* v_full, void* stream)
{
    CacheDesc c;
    int rc = make_desc(cache, &c);
    if (rc) return rc;
    if (!lengths_ok(c, tk, r, tv, L)) return KIVI_ERR_SHAPE;
    if (cdiv(tk, kBlockTokens) > c.k_cap_blocks || cdiv(tv, kBlockTokens) > c.v_cap_blocks) return KIVI_ERR_CAPACITY;
    if (tk > 0 && (!k_code || !k_scale || !k_mn)) return KIVI_ERR_NULL;
    if (tv > 0 && (!v_code || !v_scale || !v_mn)) return KIVI_ERR_NULL;
    if ((r > 0 && !k_full) || (L > 0 && !v_full)) return KIVI_ERR_NULL;
    const int U = c.B * c.Hkv;
    if (U > 65535) return KIVI_ERR_UNSUPPORTED;
    import_kv_kernel<<<dim3(8, U), 256, 0, (cudaStream_t)stream>>>(c, tk, tv, L, r,
        (const uint32_t*)k_code, (const __half*)k_scale, (const __half*)k_mn,
        (const uint32_t*)v_code, (const __half*)v_scale, (const __half*)v_mn, (const __half*)k_full, (const __half*)v_full);
    return post_launch();
}

extern "C" int kivi_cache_read_state(const kivi_cache_t* cache, int32_t* host_state8, void* stream)
{
    CacheDesc c;
    int rc = make_desc(cache, &c);
    if (rc) return rc;
    if (!host_state8) return KIVI_ERR_NULL;
    cudaError_t e = cudaMemcpyAsync(host_state8, c.state, 8 * sizeof(int32_t), cudaMemcpyDeviceToHost, (cudaStream_t)stream);
    if (e == cudaSuccess) e = cudaStreamSynchronize((cudaStream_t)stream);
    return e == cudaSuccess ? KIVI_OK : (int)e;
}

static ReorderDesc reorder_desc(const CacheDesc& c)
{
    return ReorderDesc{(int64_t)c.k_cap_blocks * lay_block_bytes(c.k_bits, c.g), (int64_t)c.v_cap_blocks * lay_block_bytes(c.v_bits, c.g),
                       (int64_t)c.R * kD * 2, (int64_t)c.v_res_cap * kD * 2};
}

extern "C" int64_t kivi_cache_reorder_scratch_bytes(const kivi_cache_t* cache)
{
    CacheDesc c;
    int rc = make_desc(cache, &c);
    if (rc) return rc;
    const ReorderDesc r = reorder_desc(c);
    return (int64_t)c.B * c.Hkv * (r.kb + r.vb + r.kw + r.vw);
}

extern "C" int kivi_cache_reorder_f16(const kivi_cache_t* cache, const int32_t* src, void* scratch, int64_t scratch_bytes,
                                      void* stream)
{
    CacheDesc c;
    int rc = make_desc(cache, &c);
    if (rc) return rc;
    if (!src || !scratch) return KIVI_ERR_NULL;
    if (scratch_bytes < kivi_cache_reorder_scratch_bytes(cache)) return KIVI_ERR_SHAPE;
    if (c.B > 65535) return KIVI_ERR_UNSUPPORTED;                                   // grid.y
    const ReorderDesc r = reorder_desc(c);
    const dim3 grid(c.Hkv * kReorderChunks, c.B);
    reorder_rows_kernel<true><<<grid, 256, 0, (cudaStream_t)stream>>>(c, src, (uint8_t*)scratch, r);
    rc = post_launch();
    if (rc) return rc;
    reorder_rows_kernel<false><<<grid, 256, 0, (cudaStream_t)stream>>>(c, src, (uint8_t*)scratch, r);
    return post_launch();
}
