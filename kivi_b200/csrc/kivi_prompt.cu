// kivi_prompt.cu -- attention of a prompt over itself (sm_90a): causal, with a first visible key per sequence (left
// padding) and an optional sliding window, without an n x n mask and without expanding K / V to the query heads.
//
// A CTA owns 64 query ROWS of one KV head: a row is a (token, query head) pair, token-major, so the K / V tiles it
// stages serve every query head of the KV head it reads (GQA).  With hc = min(G, 64) query heads per CTA it holds
// 64 / hc tokens.  4 warps of 16 rows; per 64-key tile, S = Q.K^T and O += P.V on mma.sync m16n8k16 (fp16 operands, fp32
// accumulators), with an online (running) maximum and sum in fp32.  K / V tiles are staged by cp.async into two stages
// while the previous tile is contracted.  Tiles with no visible key for any row of the CTA -- after its last token, below
// the sequence's first real token, below the window of its first token -- are never loaded.
#include "kivi_decode.cuh"

namespace kivi {

// kD = 128 (kivi_decode.cuh): head_dim, contiguous
constexpr int kRows = 64;                 // query rows per CTA (4 warps x 16)
constexpr int kKeys = 64;                 // keys per K / V tile
constexpr int kThreads = 128;
constexpr int kTileBytes = 64 * kD * 2;   // one [64][128] fp16 tile (Q, K or V): 16 KB
constexpr int kSmemBytes = 5 * kTileBytes;  // Q + two stages of (K, V)

// Byte offset of 16-byte chunk c (0..15) of row r in a [64][128] fp16 tile.  Rows are 256 B, so every row starts on the
// same bank; XOR-ing the chunk with r & 7 puts the 8 rows one ldmatrix phase reads on 8 different 16-byte bank groups.
__device__ __forceinline__ uint32_t prompt_swz(int r, int c) { return (uint32_t)(r * 256 + ((c ^ (r & 7)) << 4)); }

// 16-byte global -> shared copy; valid == false fills the 16 bytes with zeros and reads nothing.
__device__ __forceinline__ void cp16(uint32_t dst, const void* src, bool valid) {
    asm volatile("cp.async.cg.shared.global [%0], [%1], 16, %2;" ::"r"(dst), "l"(src), "r"(valid ? 16 : 0) : "memory");
}
__device__ __forceinline__ void cp_commit() { asm volatile("cp.async.commit_group;" ::: "memory"); }
__device__ __forceinline__ void cp_wait_all_but_one() { asm volatile("cp.async.wait_group 1;" ::: "memory"); }

__device__ __forceinline__ void ldsm_x4(uint32_t (&r)[4], uint32_t addr) {
    asm volatile("ldmatrix.sync.aligned.m8n8.x4.shared.b16 {%0,%1,%2,%3}, [%4];"
                 : "=r"(r[0]), "=r"(r[1]), "=r"(r[2]), "=r"(r[3]) : "r"(addr));
}
__device__ __forceinline__ void ldsm_x4_t(uint32_t (&r)[4], uint32_t addr) {
    asm volatile("ldmatrix.sync.aligned.m8n8.x4.trans.shared.b16 {%0,%1,%2,%3}, [%4];"
                 : "=r"(r[0]), "=r"(r[1]), "=r"(r[2]), "=r"(r[3]) : "r"(addr));
}

struct PromptArgs {
    const __half* q;
    const __half* k;
    const __half* v;
    __half* out;                          // [B, n, H, 128]
    int64_t q_sb, q_sh, q_st, kv_sb, kv_sh, kv_st;
    const int32_t* kv_start;              // NULL or [B]
    int H, G, n, window;
    int hc;                               // query heads per CTA, min(G, 64)
    int mt;                               // tokens per CTA, 64 / hc
    int chunks;                           // CTAs per KV head and token tile, ceil(G / hc)
};

__global__ void __launch_bounds__(kThreads, 2) prompt_attention_kernel(const PromptArgs a)
{
    extern __shared__ __align__(128) uint8_t smem[];
    const uint32_t sQ = smem_u32(smem);
    const uint32_t sKV = sQ + kTileBytes;             // stage s: K at sKV + 2 s kTileBytes, V kTileBytes further
    const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
    const int b = blockIdx.z;
    const int kvh = blockIdx.y / a.chunks;
    const int h0 = (blockIdx.y % a.chunks) * a.hc;    // this CTA's first query head within the group
    const int nh = min(a.hc, a.G - h0);
    const int t0 = (gridDim.x - 1 - blockIdx.x) * a.mt;   // the tiles with the most keys start first
    const int t1 = min(t0 + a.mt, a.n) - 1;
    const int s_b = a.kv_start ? min(max(__ldg(a.kv_start + b), 0), a.n) : 0;
    auto lo_of = [&](int i) { return max(s_b, a.window > 0 ? i - a.window + 1 : 0); };

    // keys any row of this CTA sees: [lo_of(t0), t1] (lo_of is non-decreasing in the token); none if t1 < s_b
    const int jt0 = lo_of(t0) / kKeys;
    const int n_tiles = t1 < s_b ? 0 : t1 / kKeys - jt0 + 1;

    const __half* kbase = a.k + (int64_t)b * a.kv_sb + (int64_t)kvh * a.kv_sh;
    const __half* vbase = a.v + (int64_t)b * a.kv_sb + (int64_t)kvh * a.kv_sh;
    auto load_tile = [&](int j, int stage) {
        const uint32_t dk = sKV + stage * 2 * kTileBytes, dv = dk + kTileBytes;
        #pragma unroll
        for (int it = 0; it < 8; ++it) {
            const int idx = tid + it * kThreads, r = idx >> 4, c = idx & 15;
            const int key = j * kKeys + r;
            const bool ok = key < a.n;
            const int64_t off = (int64_t)(ok ? key : 0) * a.kv_st + c * 8;
            cp16(dk + prompt_swz(r, c), kbase + off, ok);
            cp16(dv + prompt_swz(r, c), vbase + off, ok);
        }
    };

    if (n_tiles > 0) {
        #pragma unroll
        for (int it = 0; it < 8; ++it) {
            const int idx = tid + it * kThreads, r = idx >> 4, c = idx & 15;
            const int t = t0 + r / a.hc, hg = r % a.hc;
            const bool ok = r < a.mt * a.hc && t < a.n && hg < nh;
            const __half* src = a.q + (int64_t)b * a.q_sb + (int64_t)(kvh * a.G + h0 + (ok ? hg : 0)) * a.q_sh +
                                (int64_t)(ok ? t : 0) * a.q_st + c * 8;
            cp16(sQ + prompt_swz(r, c), src, ok);
        }
        load_tile(jt0, 0);
        cp_commit();
        if (n_tiles > 1) load_tile(jt0 + 1, 1);
        cp_commit();
    }

    // the two rows of this thread's accumulator fragments: warp * 16 + lane / 4 and 8 further
    const int g = lane >> 2, tq = lane & 3;
    int tok[2];
    #pragma unroll
    for (int x = 0; x < 2; ++x) tok[x] = t0 + (warp * 16 + g + 8 * x) / a.hc;
    const int lo_max = lo_of(t1);

    float o[16][4];
    #pragma unroll
    for (int i = 0; i < 16; ++i) o[i][0] = o[i][1] = o[i][2] = o[i][3] = 0.f;
    float m[2] = {-INFINITY, -INFINITY}, l[2] = {0.f, 0.f};
    uint32_t qf[8][4];
    constexpr float kScaleLog2 = 0.08838834764831845f * 1.4426950408889634f;   // 1/sqrt(128) * log2(e)

    for (int it = 0; it < n_tiles; ++it) {
        const int j = jt0 + it, stage = it & 1;
        cp_wait_all_but_one();
        __syncthreads();
        if (it == 0) {
            #pragma unroll
            for (int ks = 0; ks < 8; ++ks) ldsm_x4(qf[ks], sQ + prompt_swz(warp * 16 + (lane & 15), 2 * ks + (lane >> 4)));
        }
        const uint32_t sK = sKV + stage * 2 * kTileBytes, sV = sK + kTileBytes;

        // S = Q . K^T over the tile: 16 rows x 64 keys per warp
        float s[8][4];
        #pragma unroll
        for (int i = 0; i < 8; ++i) s[i][0] = s[i][1] = s[i][2] = s[i][3] = 0.f;
        #pragma unroll
        for (int ks = 0; ks < 8; ++ks) {
            #pragma unroll
            for (int nb2 = 0; nb2 < 4; ++nb2) {
                uint32_t kb[4];
                ldsm_x4(kb, sK + prompt_swz(nb2 * 16 + (lane & 7) + ((lane >> 4) << 3), 2 * ks + ((lane >> 3) & 1)));
                mma_16816(s[2 * nb2], qf[ks][0], qf[ks][1], qf[ks][2], qf[ks][3], kb[0], kb[1]);
                mma_16816(s[2 * nb2 + 1], qf[ks][0], qf[ks][1], qf[ks][2], qf[ks][3], kb[2], kb[3]);
            }
        }

        // keys outside a row's [lo, i] -> -inf; a tile wholly inside every row's range needs no test
        if (j * kKeys < lo_max || j * kKeys + kKeys - 1 > t0) {
            #pragma unroll
            for (int x = 0; x < 2; ++x) {
                const int i = tok[x], lo = lo_of(i);
                #pragma unroll
                for (int nb = 0; nb < 8; ++nb) {
                    #pragma unroll
                    for (int e = 0; e < 2; ++e) {
                        const int key = j * kKeys + nb * 8 + 2 * tq + e;
                        if (key < lo || key > i) s[nb][2 * x + e] = -INFINITY;
                    }
                }
            }
        }

        // online softmax (base 2, scaled logits), fp32
        #pragma unroll
        for (int x = 0; x < 2; ++x) {
            float mx = -INFINITY;
            #pragma unroll
            for (int nb = 0; nb < 8; ++nb) mx = fmaxf(mx, fmaxf(s[nb][2 * x], s[nb][2 * x + 1]));
            mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, 1));
            mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, 2));
            const float m_new = fmaxf(m[x], mx * kScaleLog2);
            const float m_use = m_new == -INFINITY ? 0.f : m_new;     // a row with nothing visible yet stays at 0
            const float alpha = exp2f(m[x] - m_use);
            m[x] = m_new;
            float sum = 0.f;
            #pragma unroll
            for (int nb = 0; nb < 8; ++nb) {
                #pragma unroll
                for (int e = 0; e < 2; ++e) {
                    const float p = exp2f(fmaf(s[nb][2 * x + e], kScaleLog2, -m_use));
                    s[nb][2 * x + e] = p;
                    sum += p;
                }
            }
            l[x] = l[x] * alpha + sum;
            #pragma unroll
            for (int db = 0; db < 16; ++db) { o[db][2 * x] *= alpha; o[db][2 * x + 1] *= alpha; }
        }

        // O += P . V: P (fp16) straight from the S fragments as the A operand
        #pragma unroll
        for (int kk = 0; kk < 4; ++kk) {
            const uint32_t pa0 = h2_as_u32(__floats2half2_rn(s[2 * kk][0], s[2 * kk][1]));
            const uint32_t pa1 = h2_as_u32(__floats2half2_rn(s[2 * kk][2], s[2 * kk][3]));
            const uint32_t pa2 = h2_as_u32(__floats2half2_rn(s[2 * kk + 1][0], s[2 * kk + 1][1]));
            const uint32_t pa3 = h2_as_u32(__floats2half2_rn(s[2 * kk + 1][2], s[2 * kk + 1][3]));
            #pragma unroll
            for (int db2 = 0; db2 < 8; ++db2) {
                uint32_t vb[4];
                ldsm_x4_t(vb, sV + prompt_swz(kk * 16 + (lane & 7) + ((lane >> 3) & 1) * 8, 2 * db2 + (lane >> 4)));
                mma_16816(o[2 * db2], pa0, pa1, pa2, pa3, vb[0], vb[1]);
                mma_16816(o[2 * db2 + 1], pa0, pa1, pa2, pa3, vb[2], vb[3]);
            }
        }

        __syncthreads();                                  // every warp is done with this stage
        if (it + 2 < n_tiles) load_tile(j + 2, stage);
        cp_commit();
    }

    // O / l -> fp16, staged through the warp's own 16 rows of the Q tile (read only by this warp, at tile 0), then
    // written as 16-byte rows of out [B, n, H, 128].  A row with no visible key is exactly zero.
    #pragma unroll
    for (int x = 0; x < 2; ++x) {
        l[x] += __shfl_xor_sync(0xffffffffu, l[x], 1);
        l[x] += __shfl_xor_sync(0xffffffffu, l[x], 2);
    }
    const int rA = warp * 16 + g;
    #pragma unroll
    for (int db = 0; db < 16; ++db) {
        #pragma unroll
        for (int x = 0; x < 2; ++x) {
            const float inv = l[x] > 0.f ? 1.f / l[x] : 0.f;
            const __half2 h = l[x] > 0.f ? __floats2half2_rn(o[db][2 * x] * inv, o[db][2 * x + 1] * inv)
                                         : __floats2half2_rn(0.f, 0.f);
            const uint32_t addr = sQ + prompt_swz(rA + 8 * x, db) + 4 * tq;
            asm volatile("st.shared.b32 [%0], %1;" ::"r"(addr), "r"(h2_as_u32(h)) : "memory");
        }
    }
    __syncwarp();
    #pragma unroll
    for (int it = 0; it < 8; ++it) {
        const int idx = lane + 32 * it, r = warp * 16 + (idx >> 4), c = idx & 15;
        const int t = t0 + r / a.hc, hg = r % a.hc;
        if (r < a.mt * a.hc && t < a.n && hg < nh) {
            uint4 w;
            asm volatile("ld.shared.v4.b32 {%0,%1,%2,%3}, [%4];"
                         : "=r"(w.x), "=r"(w.y), "=r"(w.z), "=r"(w.w) : "r"(sQ + prompt_swz(r, c)) : "memory");
            const int64_t row = ((int64_t)b * a.n + t) * a.H + (int64_t)kvh * a.G + h0 + hg;
            *reinterpret_cast<uint4*>(a.out + row * kD + c * 8) = w;
        }
    }
}

}  // namespace kivi

using namespace kivi;

extern "C" int kivi_prompt_attention_f16(const void* q, const void* k, const void* v, void* out,
                                         int batch, int num_heads, int num_kv_heads, int n,
                                         int64_t q_sb, int64_t q_sh, int64_t q_st,
                                         int64_t kv_sb, int64_t kv_sh, int64_t kv_st,
                                         const int32_t* kv_start, int window, void* stream)
{
    if (!q || !k || !v || !out) return KIVI_ERR_NULL;
    if (batch <= 0 || batch > 65535 || num_heads <= 0 || n <= 0 || window < 0) return KIVI_ERR_SHAPE;
    if (num_kv_heads <= 0 || num_heads % num_kv_heads != 0) return KIVI_ERR_GQA;
    PromptArgs a;
    a.G = num_heads / num_kv_heads;
    a.hc = a.G < kRows ? a.G : kRows;
    a.mt = kRows / a.hc;
    a.chunks = (a.G + a.hc - 1) / a.hc;
    if ((int64_t)num_kv_heads * a.chunks > 65535) return KIVI_ERR_SHAPE;      // grid.y
    // 16-byte cp.async / uint4 accesses: every row of 128 halves must start on a 16-byte boundary
    const int64_t strides[6] = {q_sb, q_sh, q_st, kv_sb, kv_sh, kv_st};
    for (int64_t s : strides)
        if (s % 8 != 0) return KIVI_ERR_ALIGN;
    if (!aligned_to(q, 16) || !aligned_to(k, 16) || !aligned_to(v, 16) || !aligned_to(out, 16) ||
        (kv_start && !aligned_to(kv_start, 4)))
        return KIVI_ERR_ALIGN;
    DeviceInfo info;
    if (int e = device_info(&info)) return e;
    static std::atomic<unsigned long long> done{0};
    if (int e = ensure_dynamic_smem(prompt_attention_kernel, kSmemBytes, info.ordinal, done)) return e;
    a.q = (const __half*)q; a.k = (const __half*)k; a.v = (const __half*)v; a.out = (__half*)out;
    a.q_sb = q_sb; a.q_sh = q_sh; a.q_st = q_st; a.kv_sb = kv_sb; a.kv_sh = kv_sh; a.kv_st = kv_st;
    a.kv_start = kv_start;
    a.H = num_heads; a.n = n; a.window = window;
    const dim3 grid((unsigned)((n + a.mt - 1) / a.mt), (unsigned)(num_kv_heads * a.chunks), (unsigned)batch);
    prompt_attention_kernel<<<grid, kThreads, kSmemBytes, (cudaStream_t)stream>>>(a);
    return post_launch();
}
