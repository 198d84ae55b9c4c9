// kivi_decode.cu -- C-ABI entry of the decode attention; the kernels live in kivi_attn.cuh and are instantiated
// per (k_bits, v_bits) pair in kivi_attn_k{2,4}v{2,4}.cu (compiled in parallel).
#include <cstdlib>
#include "kivi_attn.cuh"

namespace kivi {
int attention_k2v2(AttnParams& p, int G, bool overlap_prologue, cudaStream_t st);
int attention_k4v4(AttnParams& p, int G, bool overlap_prologue, cudaStream_t st);
int attention_k2v4(AttnParams& p, int G, bool overlap_prologue, cudaStream_t st);
int attention_k4v2(AttnParams& p, int G, bool overlap_prologue, cudaStream_t st);
}

using namespace kivi;

// query heads of a KV head that share one unit's MMAs: from the cache geometry, or the explicit KIVI_CACHE_GQA_CHUNK
// field of cache->flags (the same struct sizes the workspace and launches, so both always agree).  Every chunk streams
// all of its KV head's packed blocks, so fewer chunks ceil(ratio / G) read fewer bytes.  The geometry picks the largest G
// in {1, 2, 4} that divides the ratio, except for odd ratios above 2, which would otherwise run one head per unit: they
// take G = 4 with a partly filled last chunk (its missing heads compute on q = 0 and write nothing).  Ratios that 2 but
// not 4 divides (6: Qwen2.5-1.5B) keep G = 2: at B 32, T 4096 on an H100 G = 4 measured up to 10 % slower there
// (DESIGN.md section 5), its two units per KV head leaving more of the GPU idle than the three of G = 2.
static int gqa_chunk(int ratio, int flags) {
    int G = ratio % 4 == 0 ? 4 : ratio % 2 == 0 ? 2 : ratio >= 3 ? 4 : 1;
    const int want = (flags >> KIVI_CACHE_GQA_CHUNK_SHIFT) & 7;
    if (want == 1 || want == 2 || want == 4) G = want;
    return G;
}

extern "C" int64_t kivi_decode_workspace_bytes(const kivi_cache_t* cache, int max_kv_len)
{
    CacheDesc c;
    int rc = make_desc(cache, &c);
    if (rc) return rc;
    if (max_kv_len <= 0) return KIVI_ERR_SHAPE;
    const int ratio = c.H / c.Hkv, G = gqa_chunk(ratio, cache->flags);
    return carve_workspace(c, c.B * c.Hkv * cdiv(ratio, G), G, max_kv_len, nullptr, nullptr);
}

// Test hook (tests/test_qwen2_cpu.py): the work-unit geometry of the decode attention for a GQA ratio and cache flags,
// evaluated on the host.  Returns G (query heads per unit) and stores ceil(ratio / G) (units per KV head) in *hchunks.
extern "C" int kivi_debug_gqa_chunk(int ratio, int flags, int* hchunks)
{
    if (ratio < 1 || !hchunks) return KIVI_ERR_SHAPE;
    const int G = gqa_chunk(ratio, flags);
    *hchunks = cdiv(ratio, G);
    return G;
}

// all entries: kv_start == NULL and window == 0 is the unpadded call (the kernels without any padding logic)
static int decode_attention(const kivi_cache_t* cache, const void* q, const void* k_new, const void* v_new,
                            const int32_t* kv_start, int window, const void* mask, void* out, void* workspace,
                            int64_t workspace_bytes, void* dbg_logits, void* dbg_probs, int64_t dbg_stride, int max_kv_len,
                            void* stream)
{
    AttnParams p;
    int rc = make_desc(cache, &p.c);
    if (rc) return rc;
    if (!q || !k_new || !v_new || !out || !workspace) return KIVI_ERR_NULL;
    if (max_kv_len <= 0) return KIVI_ERR_SHAPE;
    if (max_kv_len > p.c.k_cap_blocks * kBlockTokens) return KIVI_ERR_CAPACITY;
    if (reinterpret_cast<uintptr_t>(workspace) % 256 != 0) return KIVI_ERR_ALIGN;
    if (reinterpret_cast<uintptr_t>(kv_start) % 4 != 0) return KIVI_ERR_ALIGN;
    p.q = (const __half*)q; p.k_new = (const __half*)k_new; p.v_new = (const __half*)v_new; p.mask = (const __half*)mask;
    p.kv_start = kv_start;
    p.window = window;
    p.out = (__half*)out; p.dbg_logits = (__half*)dbg_logits; p.dbg_probs = (__half*)dbg_probs; p.dbg_stride = dbg_stride;
    const bool overlap = (cache->flags & KIVI_CACHE_OVERLAP_PROLOGUE) != 0;   // the q.K^T launch may overlap its predecessor
    const int ratio = p.c.H / p.c.Hkv;
    const int G = gqa_chunk(ratio, cache->flags);
    p.hchunks = cdiv(ratio, G);
    p.n_units = p.c.B * p.c.Hkv * p.hchunks;
    p.max_kv_len = max_kv_len;
    const int64_t need = carve_workspace(p.c, p.n_units, G, max_kv_len, workspace, &p.w);
    if (need < 0) return (int)need;
    if (need > workspace_bytes) return KIVI_ERR_CAPACITY;
    cudaStream_t st = (cudaStream_t)stream;
    if (p.c.k_bits == 2 && p.c.v_bits == 2) return attention_k2v2(p, G, overlap, st);
    if (p.c.k_bits == 4 && p.c.v_bits == 4) return attention_k4v4(p, G, overlap, st);
    if (p.c.k_bits == 2 && p.c.v_bits == 4) return attention_k2v4(p, G, overlap, st);
    if (p.c.k_bits == 4 && p.c.v_bits == 2) return attention_k4v2(p, G, overlap, st);
    return KIVI_ERR_BITS;
}

extern "C" int kivi_decode_attention_f16(const kivi_cache_t* cache, const void* q, const void* k_new, const void* v_new,
                                         const void* mask, void* out, void* workspace, int64_t workspace_bytes,
                                         void* dbg_logits, void* dbg_probs, int64_t dbg_stride, int max_kv_len, void* stream)
{
    return decode_attention(cache, q, k_new, v_new, nullptr, 0, mask, out, workspace, workspace_bytes, dbg_logits, dbg_probs,
                            dbg_stride, max_kv_len, stream);
}

extern "C" int kivi_decode_attention_ragged_f16(const kivi_cache_t* cache, const void* q, const void* k_new, const void* v_new,
                                                const int32_t* kv_start, const void* mask, void* out, void* workspace,
                                                int64_t workspace_bytes, void* dbg_logits, void* dbg_probs, int64_t dbg_stride,
                                                int max_kv_len, void* stream)
{
    return decode_attention(cache, q, k_new, v_new, kv_start, 0, mask, out, workspace, workspace_bytes, dbg_logits, dbg_probs,
                            dbg_stride, max_kv_len, stream);
}

extern "C" int kivi_decode_attention_window_f16(const kivi_cache_t* cache, const void* q, const void* k_new, const void* v_new,
                                                const int32_t* kv_start, int window, const void* mask, void* out,
                                                void* workspace, int64_t workspace_bytes, void* dbg_logits, void* dbg_probs,
                                                int64_t dbg_stride, int max_kv_len, void* stream)
{
    if (window < 1) return KIVI_ERR_SHAPE;
    return decode_attention(cache, q, k_new, v_new, kv_start, window, mask, out, workspace, workspace_bytes, dbg_logits,
                            dbg_probs, dbg_stride, max_kv_len, stream);
}

// Test hook (tests/test_ranges_cpu.py): the work split of the decode kernels, evaluated on the host.  kernel 0 = q.K^T costs,
// 1 = p.V costs; out_lo receives (unit, item) of the first position of ranges 0 .. W (2 * (W + 1) ints, the last = the end);
// out_owner (may be NULL) receives owner(unit, item) for every position in order.  Returns W (or a negative error).
extern "C" int kivi_debug_range_split(int n_units, int n_b, int n_w, int w_cap, int kernel, int* out_lo, int* out_owner)
{
    if (n_units <= 0 || n_b < 0 || n_w < 0 || w_cap <= 0 || !out_lo) return KIVI_ERR_SHAPE;
    auto run = [&](auto rg) {
        for (int w = 0; w <= (int)rg.W; ++w) rg.lo(w, out_lo[2 * w], out_lo[2 * w + 1]);
        if (out_owner)
            for (int u = 0; u < n_units; ++u)
                for (int j = 0; j < rg.per_unit; ++j) out_owner[(long long)u * rg.per_unit + j] = rg.owner(u, j);
        return (int)rg.W;
    };
    if (kernel == 0) { Ranges<CostQK> rg; rg.init(n_units, n_b, n_w, w_cap); return run(rg); }
    Ranges<CostSV> rg; rg.init(n_units, n_b, n_w, w_cap);
    return run(rg);
}

// The stage sequence of every warp of a ragged or windowed call, evaluated on the host with the kernels' own cursor
// functions.  n_b = the store's packed blocks; items start at block j0 and are reported in the numbering of the whole
// store (item j + j0).  start_of(unit) = the unit's visible start.  issued: (warp, unit, item, half) of every copy the
// producer (ragged_seek + cursor_step) issues; consumed: the same for every stage the item loop waits on.
template <class SF>
static int replay_items(int n_units, int n_b, int n_w, int w_cap, int kernel, int j0, SF&& start_of, int* issued,
                        int* consumed, int64_t cap, int64_t* n_out)
{
    const int nb = n_b - j0;                                                  // packed blocks in the item sequence
    auto run = [&](auto rg) -> int {
        const int per_unit = rg.per_unit;
        int64_t ni = 0, nc = 0;
        auto put = [&](int* dst, int64_t& n, int w, int u, int j, int h) {
            if (n >= cap) return false;
            dst[4 * n] = w; dst[4 * n + 1] = u; dst[4 * n + 2] = j + j0; dst[4 * n + 3] = h;
            ++n;
            return true;
        };
        for (int w = 0; w < (int)rg.W; ++w) {
            int u_lo, j_lo, u_hi, j_hi;
            rg.lo(w, u_lo, j_lo); rg.lo(w + 1, u_hi, j_hi);
            const int n_mine = (u_hi - u_lo) * per_unit + (j_hi - j_lo);
            // producer: *_issue_next
            Cursor cur;
            cur.unit = u_lo; cur.j = j_lo; cur.half = 0; cur.left = n_mine; cur.s_unit = -1; cur.s_pos = 0;
            while (ragged_seek(cur, per_unit, nb, j0, start_of)) {
                if (!put(issued, ni, w, cur.unit, cur.j, cur.half)) return KIVI_ERR_CAPACITY;
                cursor_step(cur, per_unit, nb);
            }
            // consumer: the item loop of the kernels (one visit per unit)
            int unit = u_lo, j = j_lo, left = n_mine;
            while (left > 0) {
                const int n_here = left < per_unit - j ? left : per_unit - j;
                const int start = start_of(unit);
                for (int k = 0; k < n_here; ++k, ++j) {
                    if (ragged_skip(j, nb, j0, start)) continue;
                    if (j < nb) {
                        for (int h = 0; h < kParts; ++h)
                            if (!put(consumed, nc, w, unit, j, h)) return KIVI_ERR_CAPACITY;
                    } else if (j < per_unit - 1) {
                        if (!put(consumed, nc, w, unit, j, 0)) return KIVI_ERR_CAPACITY;
                    }
                }
                left -= n_here;
                if (j == per_unit) { j = 0; ++unit; }
            }
        }
        n_out[0] = ni; n_out[1] = nc;
        return (int)rg.W;
    };
    if (kernel == 0) { Ranges<CostQK> rg; rg.init(n_units, nb, n_w, w_cap); return run(rg); }
    Ranges<CostSV> rg; rg.init(n_units, nb, n_w, w_cap);
    return run(rg);
}

// Test hook (tests/test_ragged_cpu.py): the stage sequence of every warp of a ragged call.  kernel 0 = q.K^T (n_b = K
// blocks, n_w = K window items), 1 = p.V; unit_start[u] = the start of work unit u's sequence (clamped to kv_len as the
// kernels do).  n_out[0], n_out[1] receive the counts of issued / consumed entries; cap = entries (of 4 ints) each array
// holds.  Returns W, or a negative error.
extern "C" int kivi_debug_ragged_items(int n_units, int n_b, int n_w, int w_cap, int kernel, const int* unit_start, int kv_len,
                                       int* issued, int* consumed, int64_t cap, int64_t* n_out)
{
    if (n_units <= 0 || n_b < 0 || n_w < 0 || w_cap <= 0 || kv_len < 0) return KIVI_ERR_SHAPE;
    if (!unit_start || !issued || !consumed || !n_out) return KIVI_ERR_NULL;
    return replay_items(n_units, n_b, n_w, w_cap, kernel, 0, [&](int un) { return clamp_start(unit_start[un], kv_len); },
                        issued, consumed, cap, n_out);
}

// Test hook (tests/test_window_cpu.py): the same replay for a windowed call at shared length T (the new token at T - 1);
// unit_start NULL = no padding.  Items are numbered in the whole store: the first one issued is at least j0.
extern "C" int kivi_debug_window_items(int n_units, int n_b, int n_w, int w_cap, int kernel, const int* unit_start, int T,
                                       int window, int* issued, int* consumed, int64_t cap, int64_t* n_out)
{
    if (n_units <= 0 || n_b < 0 || n_w < 0 || w_cap <= 0 || T < 1 || window < 1) return KIVI_ERR_SHAPE;
    if (!issued || !consumed || !n_out) return KIVI_ERR_NULL;
    return replay_items(n_units, n_b, n_w, w_cap, kernel, window_first_block(T, window, n_b),
                        [&](int un) { return visible_start(unit_start ? unit_start[un] : 0, T, window); },
                        issued, consumed, cap, n_out);
}

#if KIVI_TIMELINE
#include <vector>
namespace kivi {
int timeline_k2v2(unsigned long long*); int timeline_k2v4(unsigned long long*);
int timeline_k4v2(unsigned long long*); int timeline_k4v4(unsigned long long*);
}
// tuning builds only (tools/timeline.py): the per-warp timestamps of the last attention call, [2][4096][8]
extern "C" int kivi_debug_timeline(unsigned long long* host_out)
{
    const size_t n = 2 * 4096 * 8;
    std::vector<unsigned long long> tmp(n);
    for (size_t i = 0; i < n; ++i) host_out[i] = 0;
    int (*fetch[4])(unsigned long long*) = {timeline_k2v2, timeline_k2v4, timeline_k4v2, timeline_k4v4};
    for (auto f : fetch) {
        const int rc = f(tmp.data());
        if (rc) return rc;
        for (size_t i = 0; i < n; ++i) if (tmp[i] > host_out[i]) host_out[i] = tmp[i];   // timestamps: the latest writer wins
    }
    return 0;
}
#endif
