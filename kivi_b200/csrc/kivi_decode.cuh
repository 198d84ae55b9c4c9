// kivi_decode.cuh -- KIVI cache layout in HBM (tensor-core friendly blocks) + mbarrier / bulk-copy (TMA)
// PTX helpers (sm_90a).
//
// Every packed store is a sequence of 128 x 128 BLOCKS "inner x outer":
//     K store: inner = channel d (the reduction index of q.K^T), outer = token   -> one block = 128 tokens
//     V store: inner = token t  (the reduction index of p.V),   outer = channel  -> one block = 128 tokens
// Quantisation groups run along the OUTER dim (g tokens per channel for K, g channels per token for V --
// exactly the reference's per-channel K / per-token V scheme), so a block is the same object for both.
//
//   block = [ codes: 8 chunks x kChunkBytes ][ meta: 8 chunks x (128/g) groups x 4 x 16 bytes ]
//   chunk c = inner indices 16c .. 16c+15.  Its codes are stored as the A-operand fragments of
//   mma.sync.m16n8k16 (row = outer, col = inner), so that a lane's 128-bit shared-memory load yields its four
//   A registers for F = 16/bits consecutive MMAs at once:
//       word(lane = 4*g8 + t, r), r = 0..3:   inner pair 16c + 2t + 8*(r >> 1) + {0, 1},  row = g8 + 8*(r & 1)
//       low  16 bits: field j (bits [bits*j, bits*j + bits)) = code[inner even][outer 16*j + row]
//       high 16 bits: field j                                = code[inner odd ][outer 16*j + row]
//   (a "slab" = the 16*F outer rows covered by one word set: 128 rows at 2 bits, 64 rows at 4 bits.)
//   A code becomes an fp16 MMA operand with ONE LOP3 per PAIR of codes (see Lay<>::shr below).
//   meta entry (c, G, t) = 8 halfs { z[i0], z[i0+1], s[i0], s[i0+1], z[i0+8], z[i0+9], s[i0+8], s[i0+9] },
//   i0 = 16c + 2t, of outer group G: ONE 128-bit load gives a lane the two half2 of scales it multiplies with
//   its half2 of x (q or p) to build its B fragment, and its four registers ARE the A operand of the zero-term
//   MMA (rows 0..7 = zeros of group G; rows 8..15 = the scales, whose products are ignored).
//
//   K window [U][R][128] fp16, V window [U][R+1][128] fp16 ring (head = state.vhead).  Inside a 256-byte row the eight-
//   channel (16-byte) units are XOR-swizzled with the row's slot index: unit' = unit ^ (slot & 7)  (win_off below), so that
//   the MMA fragment loads of 8 consecutive rows at one channel offset hit 8 different bank groups of shared memory.
//   state    int32[8] on the device, shared by the layers of a model: {tk, r, tv, L, vhead, kv_len}
//
// Policy restated from models/llama_kivi.py:343-356 (K: the fp16 window is quantised per channel in
// groups of g tokens as soon as it holds R tokens) and :386-399 (V: the window holds the newest R
// tokens; each step the oldest one is quantised per token in groups of g channels).
#pragma once
#include "kivi_common.cuh"

namespace kivi {

constexpr int kD = 128;            // head_dim of every model the reference ships (Llama / Mistral)
constexpr int kBlockTokens = 128;  // tokens per block (K: outer rows, V: inner rows)

struct CacheDesc {
    int B, Hkv, H, k_bits, v_bits, g, R;
    int k_cap_blocks, v_cap_blocks, v_res_cap;
    uint8_t* k_store;
    uint8_t* v_store;
    __half* k_res;
    __half* v_res;
    int* state;
};

enum { ST_TK = 0, ST_R = 1, ST_TV = 2, ST_L = 3, ST_VHEAD = 4, ST_KVLEN = 5 };

// ---- bit helpers of the packed-block contraction (decode attention, reference-layout GEMV) ------
__device__ __forceinline__ uint32_t h2_as_u32(const __half2 h) { return *reinterpret_cast<const uint32_t*>(&h); }
__device__ __forceinline__ __half2 u32_as_h2(const uint32_t u) { return *reinterpret_cast<const __half2*>(&u); }
// 2^e as an fp32 built from its exponent bits (-126 <= e <= 127)
__device__ __forceinline__ float pow2f(int e) { return __uint_as_float((uint32_t)(127 + e) << 23); }
// floor(log2 |x|) of a normal fp32 x from its exponent bits (-127 for 0); every fp16 is a normal fp32
__device__ __forceinline__ int floor_log2f(float x) { return (int)((__float_as_uint(x) >> 23) & 0xff) - 127; }

template <int BITS>
struct Lay {
    static constexpr int F = 16 / BITS;                  // fields per 16-bit half = MMAs per slab
    static constexpr int kSlabRows = 16 * F;             // outer rows per slab (128 / 64)
    static constexpr int kSlabs = 128 / kSlabRows;       // slabs per block (1 / 2)
    static constexpr int kChunkBytes = 512 * kSlabs;     // 128 words per slab
    static constexpr int kCodeBytes = 8 * kChunkBytes;   // 4096 / 8192
    // Unpack: field j of a 16-bit half is brought to bit offset P(j) in [4, 10) by an optional shift of the whole
    // word, isolated with one AND, and consumed AS IS: the fp16 denormal  code * 2^(P - 24).  mma.sync handles
    // denormal inputs exactly when their set bits sit at offset >= 4 (tools/probes/mma_unpack_variants.cu probes it; fields
    // at lower offsets can lose bits, and the GPU tests hold every kernel to the oracle), so no magic-number subtraction
    // is needed: ONE LOP3 per pair of codes.
    //   2-bit: fields 0,1 <- (w << 4);  fields 2,3,4 in place;  fields 5,6,7 <- (w >> 6)
    //   4-bit: field 0 <- (w << 4);  field 1 in place;  field 2 <- (w >> 4);  field 3 <- (w >> 8)
    __host__ __device__ static constexpr int shr(int j) {            // > 0: right shift, < 0: left shift
        return BITS == 2 ? (j < 2 ? -4 : (j < 5 ? 0 : 6)) : (j == 0 ? -4 : (j == 1 ? 0 : (j == 2 ? 4 : 8)));
    }
    __host__ __device__ static constexpr int bitpos(int j) { return BITS * j - shr(j); }
    // exact power of two 2^(24 - P) that undoes the denormal scaling of field j
    __device__ __forceinline__ static float field_scale(int j) { return pow2f(24 - bitpos(j)); }
};

__host__ __device__ inline int lay_code_bytes(int bits) { return bits == 2 ? 4096 : 8192; }
__host__ __device__ inline int lay_meta_bytes(int g) { return 8 * (128 / g) * 4 * 16; }
__host__ __device__ inline int lay_block_bytes(int bits, int g) { return lay_code_bytes(bits) + lay_meta_bytes(g); }

// The word index (inside a block) of element (inner i, outer o) is the sum of two independent parts:
//   lay_word_inner(bits, i): chunk c = i >> 4 and the lane / register bits that i selects (t = (i & 7) >> 1, r >> 1 = bit 3 of i);
//   lay_word_row(sl, row)  : slab sl = o / slab_rows and row = o % 16 in [0, 16) (g8 = row & 7, r & 1 = row >> 3).
__host__ __device__ inline int lay_word_inner(int bits, int i) {
    const int F = 16 / bits, slab_rows = 16 * F, slabs = 128 / slab_rows;
    return (i >> 4) * slabs * 128 + ((i & 7) >> 1) * 4 + ((i >> 3) & 1) * 2;
}
__host__ __device__ inline int lay_word_row(int sl, int row) { return sl * 128 + (row & 7) * 16 + (row >> 3); }

// byte offset (inside a block) of the word holding element (inner i, outer o), and its bit position
__host__ __device__ inline int lay_word_off(int bits, int i, int o) {
    const int F = 16 / bits, slab_rows = 16 * F;
    return 4 * (lay_word_inner(bits, i) + lay_word_row(o / slab_rows, o % 16));
}
__host__ __device__ inline int lay_bit_pos(int bits, int i, int o) {
    const int F = 16 / bits, slab_rows = 16 * F;
    return 16 * (i & 1) + bits * ((o % slab_rows) >> 4);
}

// The inverse of lay_word_off: word w of a block holds, in its low / high 16 bits, field j of the codes of
// (inner i0, outer o0 + 16 j) / (inner i0 + 1, outer o0 + 16 j), j = 0 .. F - 1.
struct WordPos { int i0, o0; };
__host__ __device__ inline WordPos lay_word_pos(int bits, int w) {
    const int F = 16 / bits, slab_rows = 16 * F, slabs = 128 / slab_rows;
    const int c = w / (slabs * 128), sl = (w / 128) % slabs, lw = w % 128;
    const int lane = lw >> 2, r = lw & 3;
    return {c * 16 + 2 * (lane & 3) + 8 * (r >> 1), sl * slab_rows + (lane >> 2) + 8 * (r & 1)};
}
// word w of a block, assembled from code(inner, outer), the b-bit code of one element
template <class Code>
__device__ __forceinline__ uint32_t lay_word(int bits, int w, Code&& code) {
    const WordPos p = lay_word_pos(bits, w);
    uint32_t word = 0;
    for (int par = 0; par < 2; ++par)
        for (int j = 0; j < 16 / bits; ++j) word |= code(p.i0 + par, p.o0 + 16 * j) << (16 * par + bits * j);
    return word;
}
// element offset (halfs, inside a unit's window) of (slot, channel): 16-byte units swizzled with the slot index
__host__ __device__ inline int win_off(int slot, int ch) { return slot * kD + ((((ch >> 3) ^ (slot & 7)) << 3) | (ch & 7)); }
// the same for a 16-byte unit index (0..15) of the row
__host__ __device__ inline int win_unit(int slot, int unit) { return slot * 16 + (unit ^ (slot & 7)); }

// byte offsets (inside a block) of the fp16 zero / scale of (inner i, outer group G)
__host__ __device__ inline int lay_zero_off(int bits, int g, int i, int G) {
    const int c = i >> 4, ii = i & 15;
    const int t = (ii & 7) >> 1;
    return lay_code_bytes(bits) + (((c * (128 / g)) + G) * 4 + t) * 16 + (ii >> 3) * 8 + (ii & 1) * 2;
}
__host__ __device__ inline int lay_scale_off(int bits, int g, int i, int G) { return lay_zero_off(bits, g, i, G) + 4; }
// byte offset of the 8-byte meta half { z[i0], z[i0 + 1], s[i0], s[i0 + 1] } of an inner pair (i0 even): the pair's two zeros
// and, 4 bytes on, its two scales are adjacent, so one 8-byte store writes all four
__host__ __device__ inline int lay_meta_pair_off(int bits, int g, int i0, int G) { return lay_zero_off(bits, g, i0, G); }

// ---- PTX helpers -------------------------------------------------------------------------------
__device__ __forceinline__ uint32_t smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }

__device__ __forceinline__ void mbar_init(uint64_t* bar, uint32_t count) {
    asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count));
}
__device__ __forceinline__ void mbar_fence_init() {
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
}
__device__ __forceinline__ void mbar_expect_tx(uint64_t* bar, uint32_t bytes) {
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes) : "memory");
}
__device__ __forceinline__ void mbar_arrive(uint64_t* bar) {
    asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(smem_u32(bar)) : "memory");
}
__device__ __forceinline__ void mbar_wait(uint64_t* bar, uint32_t parity) {
    asm volatile(
        "{\n\t.reg .pred p;\n\t"
        "WAIT_%=:\n\t"
        "mbarrier.try_wait.parity.shared::cta.b64 p, [%0], %1;\n\t"
        "@p bra DONE_%=;\n\t"
        "bra WAIT_%=;\n\t"
        "DONE_%=:\n\t}" ::"r"(smem_u32(bar)), "r"(parity) : "memory");
}
// 1-D bulk copy global -> shared through the TMA engine (SASS: UBLKCP), completion on an mbarrier.
// dst/src 16-B aligned, bytes % 16 == 0.  The packed cache is read exactly once per step: evict-first.
__device__ __forceinline__ void bulk_g2s(void* dst_smem, const void* src_gmem, uint32_t bytes, uint64_t* bar,
                                         uint64_t policy) {
    asm volatile(
        "cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes.L2::cache_hint [%0], [%1], %2, [%3], %4;"
        ::"r"(smem_u32(dst_smem)), "l"(src_gmem), "r"(bytes), "r"(smem_u32(bar)), "l"(policy) : "memory");
}
// L2 prefetch of a contiguous piece of global memory (a hint: no completion, no destination); src 16-B aligned, bytes % 16 == 0
__device__ __forceinline__ void bulk_prefetch_l2(const void* src_gmem, uint32_t bytes) {
    asm volatile("cp.async.bulk.prefetch.L2.global [%0], %1;" ::"l"(src_gmem), "r"(bytes) : "memory");
}
// the same copy without a cache hint (data other warps read too)
__device__ __forceinline__ void bulk_g2s_plain(void* dst_smem, const void* src_gmem, uint32_t bytes, uint64_t* bar) {
    asm volatile(
        "cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];"
        ::"r"(smem_u32(dst_smem)), "l"(src_gmem), "r"(bytes), "r"(smem_u32(bar)) : "memory");
}
__device__ __forceinline__ uint64_t policy_evict_first() {
    uint64_t p;
    asm volatile("createpolicy.fractional.L2::evict_first.b64 %0, 1.0;" : "=l"(p));
    return p;
}
__device__ __forceinline__ uint64_t policy_evict_last() {
    uint64_t p;
    asm volatile("createpolicy.fractional.L2::evict_last.b64 %0, 1.0;" : "=l"(p));
    return p;
}
__device__ __forceinline__ void named_bar_sync(int id, int nthreads) {
    asm volatile("bar.sync %0, %1;" ::"r"(id), "r"(nthreads) : "memory");
}

// D(16x8, f32) += A(16x16, f16, row) * B(16x8, f16, col)      (SASS: HMMA.16816.F32)
__device__ __forceinline__ void mma_16816(float (&c)[4], uint32_t a0, uint32_t a1, uint32_t a2, uint32_t a3,
                                          uint32_t b0, uint32_t b1) {
    asm volatile("mma.sync.aligned.m16n8k16.row.col.f32.f16.f16.f32 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, {%0,%1,%2,%3};"
                 : "+f"(c[0]), "+f"(c[1]), "+f"(c[2]), "+f"(c[3])
                 : "r"(a0), "r"(a1), "r"(a2), "r"(a3), "r"(b0), "r"(b1));
}

// D = A * B (no accumulator input: the zero registers are free, and no instruction is spent clearing D beforehand)
__device__ __forceinline__ void mma_16816_init(float (&c)[4], uint32_t a0, uint32_t a1, uint32_t a2, uint32_t a3,
                                               uint32_t b0, uint32_t b1) {
    asm volatile("mma.sync.aligned.m16n8k16.row.col.f32.f16.f16.f32 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, {%10,%10,%10,%10};"
                 : "=f"(c[0]), "=f"(c[1]), "=f"(c[2]), "=f"(c[3])
                 : "r"(a0), "r"(a1), "r"(a2), "r"(a3), "r"(b0), "r"(b1), "f"(0.f));
}

// ---- the packed-block contraction shared by the decode attention and the reference-layout GEMV ---
// Build switches (A/B builds; they apply to both kernels):
//   KIVI_BPREP2      1: b_prep is hi, then a PREDICATED fma(x, s, -hi) in the lo lanes (2 instructions); 0: branch-free 3
//   KIVI_SHIFT_IMAD  1: slab_mma's right shifts as IMAD.HI (the FMA pipe has room, the ALU pipe (LOP3) does not); 0: SHF
#ifndef KIVI_BPREP2
#define KIVI_BPREP2 1
#endif
#ifndef KIVI_SHIFT_IMAD
#define KIVI_SHIFT_IMAD 0
#endif

// One B-fragment register: a column with mask 0 gets hi = fp16(x*s), one with mask -1 (b_mask) gets lo = x*s - hi, exact
// while it is not below fp16's smallest step (the callers prescale x where it would be).
__device__ __forceinline__ uint32_t b_prep(uint32_t x2, uint32_t s2, __half2 msel) {
    const __half2 x = u32_as_h2(x2), s = u32_as_h2(s2);
#if KIVI_BPREP2
    __half2 b = __hmul2(x, s);
    if (h2_as_u32(msel) != 0u) b = __hfma2(x, s, __hneg2(b));   // lane-invariant predicate, negation folds into the HFMA2 operand
    return h2_as_u32(b);
#else
    const __half2 nh = __hmul2(__hmul2(x, s), msel);         // nh = hi * (part ? -1 : 0);  b = fma(x, s, nh)
    return h2_as_u32(__hfma2(x, s, nh));
#endif
}
// the b_prep mask of the lane's B column: hi in the even columns (g8 = lane >> 2), lo in the odd ones.  {-1, -1} / {0, 0}
// as bit constants, so that b_prep's test folds to g8 & 1.
__device__ __forceinline__ __half2 b_mask(int g8) { return u32_as_h2((g8 & 1) ? 0xbc00bc00u : 0u); }

// One slab on the tensor cores: w = the lane's four blocked A words of slab sl.  Its F fields are isolated as Lay<BITS>
// prescribes and MMA j = sl * F + j accumulates into acc[mm] with the B registers bpair(mm) returns (uint2 {b0, b1}).
// INIT: D = A * B instead of D += A * B.
template <int BITS, bool INIT, class BF>
__device__ __forceinline__ void slab_mma(const uint32_t (&w)[4], int sl, float (&acc)[8][4], BF&& bpair)
{
    using L = Lay<BITS>;
    constexpr uint32_t kField = ((1u << BITS) - 1u) * 0x00010001u;
    uint32_t wl4[4], wr4[4], wr6[4], wr8[4];    // the shifted copies a bit width needs (the others fold away)
    #pragma unroll
    for (int r = 0; r < 4; ++r) {
#if KIVI_SHIFT_IMAD
        wl4[r] = w[r] << 4; wr4[r] = __umulhi(w[r], 1u << 28); wr6[r] = __umulhi(w[r], 1u << 26); wr8[r] = __umulhi(w[r], 1u << 24);
#else
        wl4[r] = w[r] << 4; wr4[r] = w[r] >> 4; wr6[r] = w[r] >> 6; wr8[r] = w[r] >> 8;
#endif
    }
    #pragma unroll
    for (int j = 0; j < L::F; ++j) {
        uint32_t a[4];
        #pragma unroll
        for (int r = 0; r < 4; ++r) {
            const int sh = L::shr(j);
            const uint32_t src = sh == -4 ? wl4[r] : sh == 0 ? w[r] : sh == 4 ? wr4[r] : sh == 6 ? wr6[r] : wr8[r];
            a[r] = src & (kField << L::bitpos(j));
        }
        const int mm = sl * L::F + j;
        const uint2 b = bpair(mm);
        if (INIT) mma_16816_init(acc[mm], a[0], a[1], a[2], a[3], b.x, b.y);
        else mma_16816(acc[mm], a[0], a[1], a[2], a[3], b.x, b.y);
    }
}

// four 8x8 b16 matrices from shared memory, each delivered TRANSPOSED: lane (g8, t) receives, of matrix i, the elements
// (memory row 2t, column g8) and (memory row 2t+1, column g8); lanes 8i .. 8i+7 supply the row addresses of matrix i
__device__ __forceinline__ void ldmatrix_x4_trans(uint32_t (&r)[4], const void* row_ptr) {
    asm volatile("ldmatrix.sync.aligned.m8n8.x4.trans.shared.b16 {%0,%1,%2,%3}, [%4];"
                 : "=r"(r[0]), "=r"(r[1]), "=r"(r[2]), "=r"(r[3]) : "r"(smem_u32(row_ptr)));
}

}  // namespace kivi
