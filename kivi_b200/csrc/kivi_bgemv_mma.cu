// kivi_bgemv_mma.cu -- the "outer-dim" dequant-GEMV on the REFERENCE layouts with the tensor cores as unpack amortiser (sm_90a).
//
//   C[u_q, n] = sum_k A[u_q, k] * (scale[u_kv, k, n/g] * code[u_kv, k, n] + zero[u_kv, k, n/g])        (quant/matmul.py:178-219)
//
// The two shapes the attention hook produces (models/llama_kivi.py:324-325, :382-383):
//   wide  q.K^T : K = head_dim = 128 rows (inner), N = tokens (outer)        -> wide_kernel
//   tall  p.V   : K = tokens (inner),              N = head_dim = 128 (outer) -> tall_kernel
// kivi_bgemv.cu keeps the SIMT kernels (one LOP3 + one FFMA per code: bound by the 16-lane ALU pipe at ~0.4 of the HBM peak)
// for every other shape / alignment; this file serves the two hot shapes at g in {32, 64}.
//
// In the reference layout a 32-bit word holds 32/bits OUTER-consecutive codes of ONE inner index, while an mma.sync A register
// wants the codes of TWO inner-consecutive indices of one outer index.  One PRMT per pair of words fixes that:
//     lo = prmt(w[i], w[i'], 0x5410) = { low half of w[i] | low half of w[i'] },  hi = prmt(w[i], w[i'], 0x7632)
// and `lo` / `hi` are then words of exactly the blocked cache format of kivi_decode.cuh (field j of both halves = one MMA's
// operand pair), unpacked with ONE LOP3 per pair of codes as fp16 denormals (Lay<>::shr: exact for set bits at offset >= 4).
//   MMA (slab sl, field j), row rho < 8  : outer index (8 sl + rho) * 2F + j        (F = 16 / bits fields per half word)
//                           row 8 + rho  : outer index (8 sl + rho) * 2F + F + j
//   columns (B operand): (group gamma, head h, hi | lo) with hi = fp16(x*s), lo = x*s - hi (exact); a lane's two accumulator
//   columns are useful for the rows whose outer group is the lane's gamma; the other products are ignored cross terms.
//   The 16 k-indices of a chunk are mapped to inner rows (t, t+4 | t+8, t+12): the four t-lanes of a fragment load then hit
//   four different bank octets of the unpadded 32-byte rows (any k permutation is legal as long as B uses the same one).
// Data movement: every warp owns two private shared-memory stages and streams its own 128-outer x 128-inner (wide) /
// 128-inner x 128-outer (tall) tiles with cp.async (16-byte code units, 8/4-byte scale units; zero-fill past the ends), no CTA
// barrier in the loops.  tall: the CTAs of a thread-block CLUSTER split the tokens of a unit and reduce their fp32 partials
// through distributed shared memory, so few-long-unit shapes (B16 x 8 KV heads x 32k tokens) still fill the 132 SMs.
#include <cooperative_groups.h>

#include "kivi_decode.cuh"

namespace cg = cooperative_groups;

namespace kivi {
namespace bgm {

__device__ __forceinline__ uint32_t prmt(uint32_t a, uint32_t b, uint32_t sel) {
    uint32_t r;
    asm("prmt.b32 %0, %1, %2, %3;" : "=r"(r) : "r"(a), "r"(b), "r"(sel));
    return r;
}
__device__ __forceinline__ void cp_async16(void* dst, const void* src, int src_bytes) {   // bytes past src_bytes are zero-filled
    asm volatile("cp.async.cg.shared.global [%0], [%1], 16, %2;" ::"r"(smem_u32(dst)), "l"(src), "r"(src_bytes) : "memory");
}
__device__ __forceinline__ void cp_async8(void* dst, const void* src, int src_bytes) {
    asm volatile("cp.async.ca.shared.global [%0], [%1], 8, %2;" ::"r"(smem_u32(dst)), "l"(src), "r"(src_bytes) : "memory");
}
__device__ __forceinline__ void cp_async4(void* dst, const void* src, int src_bytes) {
    asm volatile("cp.async.ca.shared.global [%0], [%1], 4, %2;" ::"r"(smem_u32(dst)), "l"(src), "r"(src_bytes) : "memory");
}
__device__ __forceinline__ void cp_commit() { asm volatile("cp.async.commit_group;" ::: "memory"); }
template <int N_> __device__ __forceinline__ void cp_wait() { asm volatile("cp.async.wait_group %0;" ::"n"(N_) : "memory"); }

template <int BITS, int G, int GS>
struct Geo {
    static constexpr int kWords = 8 * Lay<BITS>::kSlabs;   // words per 128 outer indices: 8 / 16
    static constexpr int NG = 128 / GS;              // outer groups per tile: 4 / 2
    static constexpr int NP = NG * G;                // (group, head) column pairs of the one B fragment
    static_assert(NP <= 4, "one B fragment holds at most 4 (group, head) pairs");
    static constexpr int kRowBytes = kWords * 4;     // packed bytes of one inner index of a tile: 32 / 64
    static constexpr int kCodeBytes = 128 * kRowBytes;
    static constexpr int kMetaRow = NG * 2;          // scale (or zero) bytes of one inner index of a tile: 8 / 4
    static constexpr int kMetaBytes = 128 * kMetaRow;
    static constexpr int kStage = kCodeBytes + 2 * kMetaBytes;
};

// power of two that brings max|x| into [16, 32): keeps hi = fp16(x*s) clear of overflow and its residual clear of the
// fp16 denormal range (where the split would stop being exact); the result is rescaled by its exact inverse
__device__ __forceinline__ float pow2_prescale(float mx) {
    if (!(mx > 0.f) || !(mx < 3.0e38f)) return 1.f;
    const int k = max(-14, min(14, 4 - floor_log2f(mx)));
    return pow2f(k);
}

// Per-tile window of the split.  The row prescale alone does not bound x*s: a large scale overflows hi = fp16(x*s) (a zero
// code times inf is then NaN), and the tiles of a long softmax tail, or small scales, put the residual in the fp16
// denormals.  Each warp therefore checks its tile: the largest product x*s should lie in [2^kSplitMinE, 2^(kSplitMaxE+2))
// (wide: ex + es in [kSplitMinE, kSplitMaxE] with ex, es = floor(log2) of the largest |x| and largest finite |s| as they
// enter the split; tall: per-lane fp16 bounds of the products and warp votes).  Inside, the tile keeps the row prescale's
// arithmetic; outside, the largest finite |s| is brought into [2^9, 2^10) and (tall) max|x| into [16, 32) by exact powers of
// two, undone in the tile's fp32 fold.  wide keeps the row prescale of x, max|x| < 32 (below 16 only for a row whose max|q|
// is under 2^-10, which pow2_prescale cannot scale further), so there too every product stays below 2^15; the smaller ones
// remain exact down to 2^-17 of the largest.  A non-finite scale stays non-finite through any factor, and its outputs are
// non-finite in the reference as well; it does not set the factor of the tile's finite groups.
constexpr int kSplitMinE = -4, kSplitMaxE = 13;

// floor(log2) of a finite non-zero fp16 from its magnitude bits m (0 < m < 0x7c00)
__device__ __forceinline__ int h_ilogb(uint32_t m) { return m >= 0x400u ? (int)(m >> 10) - 15 : 31 - __clz(m) - 24; }
// per-half max of fp16 magnitude bits (NaN > inf > every finite value)
__device__ __forceinline__ uint32_t hmag_max(uint32_t acc, uint32_t w) { return __vmaxu2(acc, w & 0x7fff7fffu); }
// the same over the finite values only (inf and NaN count as 0)
__device__ __forceinline__ uint32_t hfin_max(uint32_t acc, uint32_t w) {
    const uint32_t m = w & 0x7fff7fffu;
    return __vmaxu2(acc, m & __vcmpltu2(m, 0x7c007c00u));
}
// the warp's max of both halves (one redux.sync)
__device__ __forceinline__ uint32_t warp_hmag_max(uint32_t v) { return __reduce_max_sync(0xffffffffu, max(v & 0xffffu, v >> 16)); }
// fp16 pair times a power of two, through fp32 (the factor need not be an fp16)
__device__ __forceinline__ uint32_t h2_scale(uint32_t w, float f) {
    const float2 v = __half22float2(u32_as_h2(w));
    return h2_as_u32(__floats2half2_rn(v.x * f, v.y * f));
}

// One chunk of 16 inner indices on the tensor cores.  W[sl][r]: the lane's raw words of inner rows (t, t+4, t+8, t+12)[r],
// word column 8 sl + g8.
template <int BITS, bool INIT>
__device__ __forceinline__ void chunk_mma(const uint32_t (&W)[Lay<BITS>::kSlabs][4], uint32_t b0, uint32_t b1, float (&acc)[8][4])
{
    #pragma unroll
    for (int sl = 0; sl < Lay<BITS>::kSlabs; ++sl) {
        uint32_t m[4];                                   // A registers before field isolation
        m[0] = prmt(W[sl][0], W[sl][1], 0x5410u);        // row g8,     k = 2t, 2t+1   (inner t, t+4):   low halves
        m[1] = prmt(W[sl][0], W[sl][1], 0x7632u);        // row g8 + 8, same k:                          high halves
        m[2] = prmt(W[sl][2], W[sl][3], 0x5410u);        // row g8,     k = 2t+8, 2t+9 (inner t+8, t+12)
        m[3] = prmt(W[sl][2], W[sl][3], 0x7632u);
        slab_mma<BITS, INIT>(m, sl, acc, [&](int) { return make_uint2(b0, b1); });
    }
}

struct Args {
    const __half* A; long long a_stride;
    const uint32_t* qB; long long qb_us, qb_rs;
    const __half *S, *Z; long long sz_us, sz_rs;
    __half* C;
    int ratio, K, N, meta_gran;
};

// ------------------------------------------------------------------------------------------------
// wide: K = 128 inner rows, N tokens.  grid = (U_kv * ratio / G, Y), block = 128 (4 warps).  The CTA streams 512-token tiles
// (full 128-byte line segments of every code row, one 32-byte sector of every scale / zero row) through two shared stages;
// warp w contracts tokens 128 w .. 128 w + 127 of the tile.  16-byte units of a code row are XOR-swizzled with
// 2 * (row & 3): the four t-lanes of a fragment load (rows r, r+1, r+2, r+3 of one word column) hit different bank octets.
// ------------------------------------------------------------------------------------------------
template <int BITS, int G, int GS>
struct WideGeo {
    static constexpr int kTileTok = 512;
    static constexpr int kRowBytes = kTileTok * BITS / 8;      // 128 / 256
    static constexpr int kUnits = kRowBytes / 16;              // 8 / 16
    static constexpr int kMetaRow = kTileTok / GS * 2;         // 32 / 16 bytes
    static constexpr int kCodeBytes = 128 * kRowBytes;
    static constexpr int kMetaBytes = 128 * kMetaRow;
    static constexpr int kStage = kCodeBytes + 2 * kMetaBytes; // 24 KB (2-bit g32) .. 36 KB (4-bit g64)
};

template <int BITS, int G, int GS>
__global__ void __launch_bounds__(128, 4)
wide_kernel(const Args a)
{
    using GE = Geo<BITS, G, GS>;
    using WG = WideGeo<BITS, G, GS>;
    constexpr int F = Lay<BITS>::F, SLABS = Lay<BITS>::kSlabs, NG = GE::NG, NP = GE::NP;
    constexpr int TG = WG::kMetaRow / 2;                                     // groups per tile row: 16 / 8
    extern __shared__ __align__(128) uint8_t smem[];
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int g8 = lane >> 2, t4 = lane & 3;
    uint2* q2 = reinterpret_cast<uint2*>(smem);                              // [G][8 chunks][4 t] half2 pairs (x[t], x[t+4] | x[t+8], x[t+12])
    float* qlin = reinterpret_cast<float*>(smem + G * 256);                  // [G][128] fp32 (prescaled)
    float* xsc = qlin + G * 128;                                             // [G] 1 / prescale
    int* xex = reinterpret_cast<int*>(xsc + G);                              // [G] floor(log2) of the prescaled max|x| (or a flag)
    float* wfac = xsc + 2 * G;                                               // [4] per warp: undoes the tile's scale factor (1 if none)
    constexpr int kZeroRow = -1000, kNonFinite = 1000;
    uint8_t* stage0 = smem + G * 768 + 64;

    const int zdim = a.ratio / G;                                           // head chunks of a unit sit in NEIGHBOURING CTAs: the second reader hits L2
    const int ukv = blockIdx.x / zdim, h0 = (blockIdx.x % zdim) * G;
    // ---- x rows of the G heads: prescale, the fragment pairs and an fp32 copy (zero term)
    if (warp < G) {
        const __half* ap = a.A + ((long long)ukv * a.ratio + h0 + warp) * a.a_stride;
        float xv[4], mx = 0.f;
        #pragma unroll
        for (int i = 0; i < 4; ++i) { xv[i] = __half2float(__ldg(ap + lane + 32 * i)); mx = fmaxf(mx, fabsf(xv[i])); }
        #pragma unroll
        for (int o = 16; o >= 1; o >>= 1) mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, o));
        const float ps = pow2_prescale(mx);
        #pragma unroll
        for (int i = 0; i < 4; ++i) qlin[warp * 128 + lane + 32 * i] = xv[i] * ps;
        if (lane == 0) {
            xsc[warp] = 1.f / ps;
            xex[warp] = !(mx < 3.0e38f) ? kNonFinite : mx == 0.f ? kZeroRow : floor_log2f(mx * ps);
        }
    }
    __syncthreads();
    if (warp < G) {                                                         // lane = (chunk c, t): rows 16c + t + {0, 4, 8, 12}
        const float* xl = qlin + warp * 128 + 16 * (lane >> 2) + (lane & 3);
        q2[warp * 32 + lane] = make_uint2(h2_as_u32(__floats2half2_rn(xl[0], xl[4])), h2_as_u32(__floats2half2_rn(xl[8], xl[12])));
    }

    const int n_tiles = cdiv(a.N, WG::kTileTok);
    const int row_bytes = a.N / (32 / BITS) * 4;                            // packed bytes of a full row
    const int meta_row_bytes = a.N / GS * 2;
    const uint8_t* code_u = reinterpret_cast<const uint8_t*>(a.qB + (long long)ukv * a.qb_us);
    const uint8_t* s_u = reinterpret_cast<const uint8_t*>(a.S + (long long)ukv * a.sz_us);
    const uint8_t* z_u = reinterpret_cast<const uint8_t*>(a.Z + (long long)ukv * a.sz_us);
    const long long code_rs = a.qb_rs * 4, meta_rs = a.sz_rs * 2;

    auto issue = [&](int tile, int st) {                                    // 512-token tile -> stage st, all 128 threads
        uint8_t* sc = stage0 + st * WG::kStage;
        uint8_t* ss = sc + WG::kCodeBytes;
        uint8_t* sz = ss + WG::kMetaBytes;
        const int off0 = tile * WG::kRowBytes;
        #pragma unroll
        for (int i = 0; i < 128 * WG::kUnits / 128; ++i) {
            const int idx = i * 128 + threadIdx.x, row = idx / WG::kUnits, un = idx % WG::kUnits;
            const int off = off0 + un * 16;
            const int nb = max(0, min(16, row_bytes - off));
            cp_async16(sc + row * WG::kRowBytes + ((un ^ ((row & 3) << 1)) << 4), nb ? code_u + row * code_rs + off : code_u, nb);
        }
        const int moff0 = tile * WG::kMetaRow;
        if (a.meta_gran >= 8) {
            constexpr int UPM = WG::kMetaRow / 8;                           // 4 / 2
            #pragma unroll
            for (int i = 0; i < 128 * UPM / 128; ++i) {
                const int idx = i * 128 + threadIdx.x, row = idx / UPM, un = idx % UPM;
                const int off = moff0 + un * 8;
                const int nb = max(0, min(8, meta_row_bytes - off));
                cp_async8(ss + row * WG::kMetaRow + un * 8, nb ? s_u + row * meta_rs + off : s_u, nb);
                cp_async8(sz + row * WG::kMetaRow + un * 8, nb ? z_u + row * meta_rs + off : z_u, nb);
            }
        } else {
            constexpr int UPM = WG::kMetaRow / 4;                           // 8 / 4
            #pragma unroll
            for (int i = 0; i < 128 * UPM / 128; ++i) {
                const int idx = i * 128 + threadIdx.x, row = idx / UPM, un = idx % UPM;
                const int off = moff0 + un * 4;
                const int nb = max(0, min(4, meta_row_bytes - off));
                cp_async4(ss + row * WG::kMetaRow + un * 4, nb ? s_u + row * meta_rs + off : s_u, nb);
                cp_async4(sz + row * WG::kMetaRow + un * 4, nb ? z_u + row * meta_rs + off : z_u, nb);
            }
        }
        cp_commit();
    };

    // this lane's B column: pair pi = g8 >> 1 = (group, head), hi | lo by the parity of g8
    const int pi_b = min(g8 >> 1, NP - 1), gam_b = pi_b / G, h_b = pi_b % G;
    const __half2 msel = b_mask(g8);
    // this lane's accumulator columns 2 t4, 2 t4 + 1 = pair t4
    const int gam_c = t4 / G, h_c = t4 % G;

    int tile = blockIdx.y, st = 0;
    if (tile < n_tiles) issue(tile, 0);
    for (; tile < n_tiles; tile += gridDim.y, st ^= 1) {
        const bool more = tile + (int)gridDim.y < n_tiles;
        if (more) { issue(tile + gridDim.y, st ^ 1); cp_wait<1>(); } else cp_wait<0>();
        __syncthreads();                                                    // the tile (and, first time, q2 / qlin) is visible to all warps
        const long long tokw = (long long)tile * WG::kTileTok + warp * 128; // first token of this warp
        if (tokw < a.N) {
            const uint8_t* sc = stage0 + st * WG::kStage;
            const __half* ss = reinterpret_cast<const __half*>(sc + WG::kCodeBytes);
            const __half* sz = reinterpret_cast<const __half*>(sc + WG::kCodeBytes + WG::kMetaBytes);
            // the tile's window (kSplitMinE): the warp's scale columns are its own, so it may rescale them in place
            {
                uint8_t* swarp = stage0 + st * WG::kStage + WG::kCodeBytes + warp * NG * 2;
                uint32_t sm = 0;
                #pragma unroll
                for (int i = 0; i < 4; ++i) {
                    const uint8_t* p = swarp + (lane + 32 * i) * WG::kMetaRow;
                    if constexpr (NG == 4) {
                        const uint2 w = *reinterpret_cast<const uint2*>(p);
                        sm = hfin_max(hfin_max(sm, w.x), w.y);
                    } else {
                        sm = hfin_max(sm, *reinterpret_cast<const uint32_t*>(p));
                    }
                }
                const uint32_t msb = warp_hmag_max(sm);                     // largest finite |s| of the tile
                bool trig = false;
                float rf = 1.f;
                if (msb != 0) {
                    const int es = h_ilogb(msb);
                    #pragma unroll
                    for (int h = 0; h < G; ++h) {                           // (a head with a non-finite q is non-finite anyway)
                        const int ex = xex[h];
                        if (ex != kZeroRow && ex != kNonFinite) trig |= ex + es > kSplitMaxE || ex + es < kSplitMinE;
                    }
                    if (trig) {
                        const int ks = kSplitMaxE - 4 - es;                 // max finite |s| into [2^9, 2^10): below 2^15 / 32
                        const float fs = pow2f(ks);
                        #pragma unroll
                        for (int i = 0; i < 4; ++i) {
                            uint8_t* p = swarp + (lane + 32 * i) * WG::kMetaRow;
                            if constexpr (NG == 4) {
                                uint2 w = *reinterpret_cast<const uint2*>(p);
                                w.x = h2_scale(w.x, fs); w.y = h2_scale(w.y, fs);
                                *reinterpret_cast<uint2*>(p) = w;
                            } else {
                                *reinterpret_cast<uint32_t*>(p) = h2_scale(*reinterpret_cast<const uint32_t*>(p), fs);
                            }
                        }
                        rf = pow2f(-ks);
                        __syncwarp();
                    }
                }
                if (lane == 0) wfac[warp] = rf;                             // read back in the epilogue: one register less in the MMAs
            }
            float acc[8][4];
            #pragma unroll
            for (int c = 0; c < 8; ++c) {
                const int r0 = 16 * c + t4;                                 // inner rows r0 + {0, 4, 8, 12}: all have (row & 3) == t4
                uint32_t W[SLABS][4];
                #pragma unroll
                for (int sl = 0; sl < SLABS; ++sl) {
                    const int wi = warp * GE::kWords + sl * 8 + g8;         // word column within the tile row
                    const int woff = ((((wi >> 2) ^ (t4 << 1)) << 2) | (wi & 3)) * 4;
                    #pragma unroll
                    for (int r = 0; r < 4; ++r)
                        W[sl][r] = *reinterpret_cast<const uint32_t*>(sc + (r0 + 4 * r) * WG::kRowBytes + woff);
                }
                const uint2 xq = q2[(h_b * 8 + c) * 4 + t4];
                const int gcol = warp * NG + gam_b;
                const uint32_t s01 = h2_as_u32(__halves2half2(ss[(r0) * TG + gcol], ss[(r0 + 4) * TG + gcol]));
                const uint32_t s23 = h2_as_u32(__halves2half2(ss[(r0 + 8) * TG + gcol], ss[(r0 + 12) * TG + gcol]));
                const uint32_t b0 = b_prep(xq.x, s01, msel), b1 = b_prep(xq.y, s23, msel);
                if (c == 0) chunk_mma<BITS, true>(W, b0, b1, acc);
                else chunk_mma<BITS, false>(W, b0, b1, acc);
            }
            // zero term of this lane's pair: sum_d x_h[d] * z[d][gamma]   (the g8 lanes split the rows, butterfly sum)
            float zt = 0.f;
            if (t4 < NP) {
                const int gcol = warp * NG + gam_c;
                #pragma unroll 4
                for (int i = 0; i < 16; ++i) {
                    const int d = g8 * 16 + i;
                    zt = fmaf(qlin[h_c * 128 + d], __half2float(sz[d * TG + gcol]), zt);
                }
            }
            zt += __shfl_xor_sync(0xffffffffu, zt, 4);
            zt += __shfl_xor_sync(0xffffffffu, zt, 8);
            zt += __shfl_xor_sync(0xffffffffu, zt, 16);
            // ---- epilogue: the lane owns, per slab, the 2F tokens of word column 8 sl + g8 if their group is its pair's group
            const float rs = xsc[h_c];
            __syncwarp();
            const float rfac = wfac[warp];
            #pragma unroll
            for (int sl = 0; sl < SLABS; ++sl) {
                const int o0 = (sl * 8 + g8) * 2 * F;                       // first of 2F consecutive tokens (within the warp's 128)
                if (t4 < NP && o0 / GS == gam_c) {
                    const long long tok0 = tokw + o0;
                    if (tok0 < a.N) {                                       // N % GS == 0 and 2F | GS: all 2F tokens or none
                        __align__(16) __half o[2 * F];
                        #pragma unroll
                        for (int j = 0; j < F; ++j) {
                            const float sc_j = Lay<BITS>::field_scale(j) * rfac;
                            o[j] = __float2half_rn(fmaf(acc[sl * F + j][0] + acc[sl * F + j][1], sc_j, zt) * rs);
                            o[F + j] = __float2half_rn(fmaf(acc[sl * F + j][2] + acc[sl * F + j][3], sc_j, zt) * rs);
                        }
                        __half* dst = a.C + ((long long)ukv * a.ratio + h0 + h_c) * a.N + tok0;
                        #pragma unroll
                        for (int v = 0; v < 2 * F / 8; ++v)
                            *reinterpret_cast<uint4*>(dst + 8 * v) = *reinterpret_cast<const uint4*>(o + 8 * v);
                    }
                }
            }
        }
        __syncthreads();                                                    // stage st is free for the copy issued next iteration
    }
}

// ------------------------------------------------------------------------------------------------
// tall: N = 128 outer, K tokens (inner).  grid = (U_kv * ratio / G, S) with cluster (1, S, 1); block = 256 (8 warps); the
// 8 S warps of a cluster take the 128-token tiles of the unit round-robin.
// ------------------------------------------------------------------------------------------------
template <int BITS, int G, int GS>
__global__ void __launch_bounds__(256, 2)
tall_kernel(const Args a)
{
    using GE = Geo<BITS, G, GS>;
    constexpr int F = Lay<BITS>::F, SLABS = Lay<BITS>::kSlabs, NG = GE::NG, NP = GE::NP;
    extern __shared__ __align__(128) uint8_t smem[];
    cg::cluster_group cluster = cg::this_cluster();
    const int S = (int)cluster.num_blocks(), crank = (int)cluster.block_rank();
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int g8 = lane >> 2, t4 = lane & 3;
    float* red = reinterpret_cast<float*>(smem);                             // [G][128] fp32 partial of this CTA (+ cluster reduce)
    float* xsc = red + G * 128;                                              // [G] prescale, [G] its inverse
    float* wmax = xsc + 2 * G;                                               // [8][G]
    uint8_t* wbase = smem + G * 512 + 256 + (size_t)warp * (2 * GE::kStage + 2 * G * 256);
    __half* xbuf = reinterpret_cast<__half*>(wbase + 2 * GE::kStage);        // [2 stages][G][128] prescaled x of the tile

    const int zdim = a.ratio / G;
    const int ukv = blockIdx.x / zdim, h0 = (blockIdx.x % zdim) * G;
    const __half* arow = a.A + ((long long)ukv * a.ratio + h0) * a.a_stride;
    // ---- prescale per head: max |x| over the whole row (every CTA of the cluster computes the same value)
    {
        float mx[G];
        #pragma unroll
        for (int h = 0; h < G; ++h) mx[h] = 0.f;
        for (int k = threadIdx.x; k < a.K; k += 256)
            #pragma unroll
            for (int h = 0; h < G; ++h) mx[h] = fmaxf(mx[h], fabsf(__half2float(__ldg(arow + h * a.a_stride + k))));
        #pragma unroll
        for (int h = 0; h < G; ++h) {
            #pragma unroll
            for (int o = 16; o >= 1; o >>= 1) mx[h] = fmaxf(mx[h], __shfl_xor_sync(0xffffffffu, mx[h], o));
            if (lane == 0) wmax[warp * G + h] = mx[h];
        }
        __syncthreads();
        if (threadIdx.x < G) {
            float m = 0.f;
            for (int w = 0; w < 8; ++w) m = fmaxf(m, wmax[w * G + threadIdx.x]);
            const float ps = pow2_prescale(m);
            xsc[threadIdx.x] = ps; xsc[G + threadIdx.x] = 1.f / ps;
        }
        __syncthreads();
    }

    const int n_tiles = cdiv(a.K, 128);
    const uint8_t* code_u = reinterpret_cast<const uint8_t*>(a.qB + (long long)ukv * a.qb_us);
    const uint8_t* s_u = reinterpret_cast<const uint8_t*>(a.S + (long long)ukv * a.sz_us);
    const uint8_t* z_u = reinterpret_cast<const uint8_t*>(a.Z + (long long)ukv * a.sz_us);

    auto issue = [&](int tile, int st) {                                    // tokens 128 tile .. +127 -> stage st
        uint8_t* sc = wbase + st * GE::kStage;
        uint8_t* ss = sc + GE::kCodeBytes;
        uint8_t* sz = ss + GE::kMetaBytes;
        const int t0 = tile * 128;
        constexpr int UPR = GE::kRowBytes / 16;
        #pragma unroll
        for (int i = 0; i < 128 * UPR / 32; ++i) {
            const int idx = i * 32 + lane, row = idx / UPR, un = idx % UPR;
            const bool in = t0 + row < a.K;
            cp_async16(sc + row * GE::kRowBytes + un * 16, in ? code_u + (long long)(t0 + row) * a.qb_rs * 4 + un * 16 : code_u,
                       in ? 16 : 0);
        }
        if (a.meta_gran >= 8 && GE::kMetaRow == 8) {
            #pragma unroll
            for (int i = 0; i < 4; ++i) {
                const int row = i * 32 + lane, nb = t0 + row < a.K ? 8 : 0;
                cp_async8(ss + row * 8, nb ? s_u + (long long)(t0 + row) * a.sz_rs * 2 : s_u, nb);
                cp_async8(sz + row * 8, nb ? z_u + (long long)(t0 + row) * a.sz_rs * 2 : z_u, nb);
            }
        } else {
            constexpr int UPM = GE::kMetaRow / 4;
            #pragma unroll
            for (int i = 0; i < 128 * UPM / 32; ++i) {
                const int idx = i * 32 + lane, row = idx / UPM, un = idx % UPM, nb = t0 + row < a.K ? 4 : 0;
                cp_async4(ss + row * GE::kMetaRow + un * 4, nb ? s_u + (long long)(t0 + row) * a.sz_rs * 2 + un * 4 : s_u, nb);
                cp_async4(sz + row * GE::kMetaRow + un * 4, nb ? z_u + (long long)(t0 + row) * a.sz_rs * 2 + un * 4 : z_u, nb);
            }
        }
        cp_commit();
        // the tile's x values (any alignment: A may be a strided slice of the probabilities, llama_kivi.py:382), prescaled
        __half* xb = xbuf + st * G * 128;
        #pragma unroll
        for (int h = 0; h < G; ++h)
            #pragma unroll
            for (int i = 0; i < 4; ++i) {
                const int k = t0 + lane + 32 * i;
                const float x = k < a.K ? __half2float(__ldg(arow + h * a.a_stride + k)) : 0.f;
                xb[h * 128 + lane + 32 * i] = __float2half_rn(x * xsc[h]);
            }
    };

    const int pi_b = min(g8 >> 1, NP - 1), gam_b = pi_b / G, h_b = pi_b % G;
    const __half2 msel = b_mask(g8);
    const int gam_c = t4 / G, h_c = t4 % G;
    float run[SLABS][2 * F];                                                // the lane's outputs (useful lanes only), summed over its tiles
    #pragma unroll
    for (int sl = 0; sl < SLABS; ++sl)
        #pragma unroll
        for (int j = 0; j < 2 * F; ++j) run[sl][j] = 0.f;
    float zrun = 0.f;                                                       // zero term of the lane's pair over the rows the lane handles

    const int gwarp = crank * 8 + warp, gstep = S * 8;
    int tile = gwarp, st = 0;
    if (tile < n_tiles) issue(tile, 0);
    for (; tile < n_tiles; tile += gstep, st ^= 1) {
        const bool more = tile + gstep < n_tiles;
        if (more) { issue(tile + gstep, st ^ 1); cp_wait<1>(); } else cp_wait<0>();
        __syncwarp();
        const uint8_t* sc = wbase + st * GE::kStage;
        const __half* ss = reinterpret_cast<const __half*>(sc + GE::kCodeBytes);
        const __half* sz = reinterpret_cast<const __half*>(sc + GE::kCodeBytes + GE::kMetaBytes);
        __half* xb = xbuf + st * G * 128;

        // the tile's window (kSplitMinE).  Each lane bounds the products x*s of the rows whose scales it reads by max|x| times
        // max s, in fp16 (inf where hi could overflow; raw bits, so a negative or non-finite scale also reads as >= 0x7c00).
        // Warp votes decide: any lane's bound overflows, or, for one head, every lane's bound is below 2^kSplitMinE.  A tile
        // outside the window (rare) gets x (per head) and s rescaled in place -- the stage is the warp's own -- from its exact
        // maxima (of the finite scales), and its fp32 fold and zero term take the exact inverse.
        uint4* sv = reinterpret_cast<uint4*>(wbase + st * GE::kStage + GE::kCodeBytes);
        bool trig;
        {
            uint32_t sm = 0;
            #pragma unroll
            for (int i = 0; i < GE::kMetaBytes / 512; ++i) {
                const uint4 w = sv[i * 32 + lane];
                sm = __vmaxu2(sm, __vmaxu2(__vmaxu2(w.x, w.y), __vmaxu2(w.z, w.w)));
            }
            sm = max(sm & 0xffffu, sm >> 16) * 0x10001u;
            uint32_t xq[G];
            #pragma unroll
            for (int h = 0; h < G; ++h) {                                   // x of the same rows: 8 / NG rows per 16-byte scale unit
                uint32_t m;
                if constexpr (NG == 4) {
                    const uint32_t* x2 = reinterpret_cast<const uint32_t*>(xb + h * 128);
                    m = __vmaxu2(x2[lane] & 0x7fff7fffu, x2[32 + lane] & 0x7fff7fffu);
                } else {
                    const uint2 x4 = reinterpret_cast<const uint2*>(xb + h * 128)[lane];
                    m = __vmaxu2(x4.x & 0x7fff7fffu, x4.y & 0x7fff7fffu);
                }
                xq[h] = max(m & 0xffffu, m >> 16);
            }
            const uint32_t q = h2_as_u32(__hmul2(u32_as_h2(xq[0] | (xq[G - 1] << 16)), u32_as_h2(sm)));
            const bool big = __vcmpgeu2(q, 0x7c007c00u) != 0;                // 2^(kSplitMaxE + 2) is past fp16's range
            const uint32_t small = __vcmpltu2(q, 0x2c002c00u);              // per head: below 2^kSplitMinE
            trig = __any_sync(0xffffffffu, big);
            if constexpr (G == 1) trig = trig || __all_sync(0xffffffffu, small != 0);
            else trig = trig || __all_sync(0xffffffffu, (small & 0xffffu) != 0) || __all_sync(0xffffffffu, (small >> 16) != 0);
        }
        float rf = 1.f, zf = 1.f;                                           // bring the lane's head's partials back to the row prescale
        if (trig) {                                                         // warp-uniform
            uint32_t sm = 0;
            #pragma unroll
            for (int i = 0; i < GE::kMetaBytes / 512; ++i) {
                const uint4 w = sv[i * 32 + lane];
                sm = hfin_max(hfin_max(hfin_max(hfin_max(sm, w.x), w.y), w.z), w.w);
            }
            const uint32_t msb = warp_hmag_max(sm);                         // largest finite |s| of the tile
            const int ks = msb == 0 ? 0 : kSplitMaxE - 4 - h_ilogb(msb);    // into [2^9, 2^10)
            const float fs = pow2f(ks);
            #pragma unroll
            for (int i = 0; i < GE::kMetaBytes / 512; ++i) {
                uint4 w = sv[i * 32 + lane];
                w.x = h2_scale(w.x, fs); w.y = h2_scale(w.y, fs); w.z = h2_scale(w.z, fs); w.w = h2_scale(w.w, fs);
                sv[i * 32 + lane] = w;
            }
            #pragma unroll
            for (int h = 0; h < G; ++h) {
                float x[4];
                uint32_t m = 0;
                #pragma unroll
                for (int i = 0; i < 4; ++i) {                               // the unscaled x again (the row prescale may have lost bits)
                    const int k = tile * 128 + lane + 32 * i;
                    const __half xh = k < a.K ? __ldg(arow + h * a.a_stride + k) : __float2half_rn(0.f);
                    m = max(m, (uint32_t)__half_as_ushort(xh) & 0x7fffu);
                    x[i] = __half2float(xh);
                }
                m = min(__reduce_max_sync(0xffffffffu, m), 0x7bffu);
                const int eps = floor_log2f(xsc[h]);                        // log2 of the row prescale
                const int ecx = m != 0 ? 4 - h_ilogb(m) : eps;              // max|x| into [16, 32)
                const float cx = pow2f(ecx);
                #pragma unroll
                for (int i = 0; i < 4; ++i) xb[h * 128 + lane + 32 * i] = __float2half_rn(x[i] * cx);
                if (h == h_c) { rf = pow2f(eps - ecx - ks); zf = pow2f(eps - ecx); }
            }
            __syncwarp();
        }

        float acc[8][4];
        #pragma unroll
        for (int c = 0; c < 8; ++c) {
            const int r0 = 16 * c + t4;
            uint32_t W[SLABS][4];
            #pragma unroll
            for (int sl = 0; sl < SLABS; ++sl)
                #pragma unroll
                for (int r = 0; r < 4; ++r)
                    W[sl][r] = *reinterpret_cast<const uint32_t*>(sc + (r0 + 4 * r) * GE::kRowBytes + (sl * 8 + g8) * 4);
            const __half* xh = xb + h_b * 128;
            const uint32_t x01 = h2_as_u32(__halves2half2(xh[r0], xh[r0 + 4])), x23 = h2_as_u32(__halves2half2(xh[r0 + 8], xh[r0 + 12]));
            const uint32_t s01 = h2_as_u32(__halves2half2(ss[(r0) * NG + gam_b], ss[(r0 + 4) * NG + gam_b]));
            const uint32_t s23 = h2_as_u32(__halves2half2(ss[(r0 + 8) * NG + gam_b], ss[(r0 + 12) * NG + gam_b]));
            const uint32_t b0 = b_prep(x01, s01, msel), b1 = b_prep(x23, s23, msel);
            if (c == 0) chunk_mma<BITS, true>(W, b0, b1, acc);
            else chunk_mma<BITS, false>(W, b0, b1, acc);
        }
        if (t4 < NP) {
            if (trig) {
                float zt = 0.f;
                #pragma unroll 4
                for (int i = 0; i < 16; ++i) {
                    const int d = g8 * 16 + i;
                    zt = fmaf(__half2float(xb[h_c * 128 + d]), __half2float(sz[d * NG + gam_c]), zt);
                }
                zrun = fmaf(zt, zf, zrun);
            } else {
                #pragma unroll 4
                for (int i = 0; i < 16; ++i) {
                    const int d = g8 * 16 + i;
                    zrun = fmaf(__half2float(xb[h_c * 128 + d]), __half2float(sz[d * NG + gam_c]), zrun);
                }
            }
        }
        // accumulator chains live for ONE tile (mma.sync accumulates with truncation); round-to-nearest adds across tiles
        auto fold = [&](float f) {
            #pragma unroll
            for (int sl = 0; sl < SLABS; ++sl)
                #pragma unroll
                for (int j = 0; j < F; ++j) {
                    const float sc_j = Lay<BITS>::field_scale(j) * f;
                    run[sl][j] = fmaf(acc[sl * F + j][0] + acc[sl * F + j][1], sc_j, run[sl][j]);
                    run[sl][F + j] = fmaf(acc[sl * F + j][2] + acc[sl * F + j][3], sc_j, run[sl][F + j]);
                }
        };
        if (trig) fold(rf);
        else fold(1.f);                                                     // (constant factor: the fold as it always was)
        __syncwarp();
    }
    // ---- reduce, in a fixed order (deterministic): lanes -> the warp's partial (its own stage memory, every output written
    // by exactly one lane) -> CTA partial -> rank 0 of the cluster through distributed shared memory
    zrun += __shfl_xor_sync(0xffffffffu, zrun, 4);
    zrun += __shfl_xor_sync(0xffffffffu, zrun, 8);
    zrun += __shfl_xor_sync(0xffffffffu, zrun, 16);                          // all lanes with the same t4 now hold the pair's zero term
    float* part = reinterpret_cast<float*>(wbase);                          // [G][128]
    #pragma unroll
    for (int sl = 0; sl < SLABS; ++sl) {
        const int o0 = (sl * 8 + g8) * 2 * F;
        if (t4 < NP && o0 / GS == gam_c) {
            #pragma unroll
            for (int j = 0; j < 2 * F; ++j) part[h_c * 128 + o0 + j] = run[sl][j] + zrun;
        }
    }
    __syncthreads();
    for (int i = threadIdx.x; i < G * 128; i += 256) {
        float v = 0.f;
        #pragma unroll
        for (int w = 0; w < 8; ++w)
            v += reinterpret_cast<const float*>(smem + G * 512 + 256 + (size_t)w * (2 * GE::kStage + 2 * G * 256))[i];
        red[i] = v;
    }
    __syncthreads();
    if (S > 1) {
        cluster.sync();                                                     // every CTA's partial is complete
        if (crank == 0) {
            for (int i = threadIdx.x; i < G * 128; i += 256) {
                float v = red[i];
                for (int r = 1; r < S; ++r) v += cluster.map_shared_rank(red, r)[i];
                red[i] = v;
            }
        }
        cluster.sync();                                                     // remote shared memory stays alive until rank 0 has read it
        if (crank != 0) return;
        __syncthreads();
    }
    for (int i = threadIdx.x; i < G * 128; i += 256) {
        const int h = i >> 7, n = i & 127;
        a.C[((long long)ukv * a.ratio + h0 + h) * 128 + n] = __float2half_rn(red[i] * xsc[G + h]);
    }
}

// ------------------------------------------------------------------------------------------------
// host
// ------------------------------------------------------------------------------------------------
template <int BITS, int G, int GS>
static int launch_wide(const Args& a, int U, cudaStream_t st)
{
    using WG = WideGeo<BITS, G, GS>;
    DeviceInfo di;
    int rc = device_info(&di);
    if (rc) return rc;
    const size_t smem = (size_t)G * 768 + 64 + 2 * WG::kStage;
    static std::atomic<unsigned long long> optin{0};
    rc = ensure_dynamic_smem(wide_kernel<BITS, G, GS>, (int)smem, di.ordinal, optin);
    if (rc) return rc;
    const int Z = a.ratio / G;
    const int n_tiles = cdiv(a.N, WG::kTileTok);
    // enough CTAs for ~3 per resident slot (4 CTAs per SM), never more than one per tile
    const long long slots = (long long)di.num_sms * 4;
    int Y = (int)min((long long)n_tiles, max(1ll, (3 * slots + (long long)U * Z - 1) / ((long long)U * Z)));
    if (Y > 65535) Y = 65535;
    wide_kernel<BITS, G, GS><<<dim3(U * Z, Y, 1), 128, smem, st>>>(a);
    return post_launch();
}

template <int BITS, int G, int GS>
static int launch_tall(const Args& a, int U, cudaStream_t st)
{
    using GE = Geo<BITS, G, GS>;
    DeviceInfo di;
    int rc = device_info(&di);
    if (rc) return rc;
    const size_t smem = (size_t)G * 512 + 256 + 8 * (2 * GE::kStage + 2 * G * 256);
    static std::atomic<unsigned long long> optin{0};
    rc = ensure_dynamic_smem(tall_kernel<BITS, G, GS>, (int)smem, di.ordinal, optin);
    if (rc) return rc;
    const int Z = a.ratio / G;
    const int n_tiles = cdiv(a.K, 128);
    int S = 1;                                                               // cluster size: split the tokens while the grid is short of 2 CTAs per SM
    while (S < 8 && (long long)U * Z * S < 2ll * di.num_sms && n_tiles >= 16 * S) S *= 2;
    cudaLaunchConfig_t cfg = {};
    cfg.gridDim = dim3(U * Z, S, 1); cfg.blockDim = dim3(256); cfg.dynamicSmemBytes = smem; cfg.stream = st;
    cudaLaunchAttribute attr[1];
    attr[0].id = cudaLaunchAttributeClusterDimension;
    attr[0].val.clusterDim.x = 1; attr[0].val.clusterDim.y = S; attr[0].val.clusterDim.z = 1;
    cfg.attrs = attr; cfg.numAttrs = 1;
    const cudaError_t e = cudaLaunchKernelEx(&cfg, tall_kernel<BITS, G, GS>, a);
    if (e != cudaSuccess) return (int)e;
    return post_launch();
}

}  // namespace bgm

// Try the tensor-core path for a KIVI_LAYOUT_REFERENCE call; returns KIVI_ERR_UNSUPPORTED when the shape / alignment is
// not one of the two hot ones (the caller then runs the SIMT kernels of kivi_bgemv.cu).
int bgemv_ref_mma(const __half* A, long long a_stride, const uint32_t* qB, long long qb_us, long long qb_rs,
                  const __half* S, const __half* Z, long long sz_us, long long sz_rs, __half* C,
                  int B, int nh, int nh_kv, int K, int N, int bits, int g, cudaStream_t st)
{
    if (!(bits == 2 || bits == 4) || !(g == 32 || g == 64)) return KIVI_ERR_UNSUPPORTED;
    const int ratio = nh / nh_kv, fpi = 32 / bits, NG = 128 / g;
    const long long U = (long long)B * nh_kv;
    if (U * ratio > 0x7fffffff) return KIVI_ERR_UNSUPPORTED;
    int G = 1;                                                               // heads per CTA: (128 / g) * G <= 4 column pairs
    if (NG == 2 && ratio % 2 == 0) G = 2;
    bgm::Args a{A, a_stride, qB, qb_us, qb_rs, S, Z, sz_us, sz_rs, C, ratio, K, N, 0};
    auto aligned = [](const void* p, long long us_bytes, long long rs_bytes, int gran) {
        return reinterpret_cast<uintptr_t>(p) % gran == 0 && us_bytes % gran == 0 && rs_bytes % gran == 0;
    };
    const bool wide = (K == 128 && N >= 64), tall = (N == 128 && K >= 1);
    if (!wide && !tall) return KIVI_ERR_UNSUPPORTED;
    if (!aligned(qB, qb_us * 4, qb_rs * 4, 16) || reinterpret_cast<uintptr_t>(C) % 16 != 0) return KIVI_ERR_UNSUPPORTED;
    if (aligned(S, sz_us * 2, sz_rs * 2, 8) && aligned(Z, sz_us * 2, sz_rs * 2, 8)) a.meta_gran = 8;
    else if (aligned(S, sz_us * 2, sz_rs * 2, 4) && aligned(Z, sz_us * 2, sz_rs * 2, 4)) a.meta_gran = 4;
    else return KIVI_ERR_UNSUPPORTED;
    #define KIVI_MMA_DISPATCH(FN)                                                                  \
        if (bits == 2 && g == 32) return bgm::FN<2, 1, 32>(a, (int)U, st);                         \
        if (bits == 4 && g == 32) return bgm::FN<4, 1, 32>(a, (int)U, st);                         \
        if (bits == 2 && g == 64) return G == 2 ? bgm::FN<2, 2, 64>(a, (int)U, st) : bgm::FN<2, 1, 64>(a, (int)U, st); \
        if (bits == 4 && g == 64) return G == 2 ? bgm::FN<4, 2, 64>(a, (int)U, st) : bgm::FN<4, 1, 64>(a, (int)U, st);
    (void)fpi;
    if (tall) {                                                              // (K = N = 128 is both shapes: either kernel computes it)
        KIVI_MMA_DISPATCH(launch_tall)
    }
    if (wide) {
        if (N % 64 != 0) return KIVI_ERR_UNSUPPORTED;                       // 16-byte code units must not straddle a row end mid-word pair
        // On THIS layout the merge (PRMT) and the scattered scale loads eat most of what the MMA saves: with one query head
        // per KV head the SIMT kernel (one LOP3 + one FFMA per code on two different pipes) is used, with shared KV heads (one
        // FFMA per code AND head) the MMA kernel (tools/microbench.py compares them).
        if (ratio < 2 || ratio / G > 2) return KIVI_ERR_UNSUPPORTED;
        KIVI_MMA_DISPATCH(launch_wide)
    }
    #undef KIVI_MMA_DISPATCH
    return KIVI_ERR_UNSUPPORTED;
}

}  // namespace kivi
