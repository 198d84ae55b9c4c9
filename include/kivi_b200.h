/*
 * kivi_b200.h -- C ABI of libkivi_b200.so, the H100-native (sm_90a) implementation of the
 * KIVI decode hot path: 2/4-bit asymmetric pack of new K/V tokens and the batched dequant-GEMVs
 * q.K^T and softmax.V over the packed cache (+ fp16 residual window).
 *
 * This is the drop-in boundary.  Each entry point replaces one interface of the reference
 * (jy-yuan/KIVI @ 876b4d2); the reference-side binding a maintainer would add is shown in
 * INTEGRATION.md.  Rules common to all entry points:
 *   - plain C types only: device pointers, sizes, strides, a stream handle.  No torch types.
 *   - the CALLER owns every buffer, outputs included; nothing is allocated, nothing is freed.
 *   - asynchronous: work is enqueued on `stream` (a cudaStream_t passed as void*; NULL = the
 *     legacy default stream) and the call returns immediately.  No global state, re-entrant,
 *     CUDA-graph capturable.  The device is the current device of the calling thread and must
 *     own the pointers (the Python shim wraps calls in torch.cuda.device(tensor.device)).
 *   - return 0 on success, a negative KIVI_ERR_* for argument errors (nothing was enqueued),
 *     or a positive cudaError_t from the launch.  Never throws.
 *   - fp16 data are IEEE binary16 (`__half` bits); packed codes are little-endian in the
 *     32-bit word: element i of a word sits at bit i*bits (quant/new_pack.py:148-153).
 */
#ifndef KIVI_B200_H
#define KIVI_B200_H

#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define KIVI_OK              0
#define KIVI_ERR_BITS       -1   /* bits not in the supported set                         */
#define KIVI_ERR_SHAPE      -2   /* a dimension / divisibility requirement is violated    */
#define KIVI_ERR_GQA        -3   /* nh % nh_kv != 0 or nh_kv <= 0                         */
#define KIVI_ERR_GROUP      -4   /* unsupported group_size                                */
#define KIVI_ERR_ALIGN      -5   /* pointer / stride alignment requirement violated       */
#define KIVI_ERR_NULL       -6   /* required pointer is NULL                              */
#define KIVI_ERR_LAYOUT     -7   /* unknown layout id                                     */
#define KIVI_ERR_CAPACITY   -8   /* cache capacity exceeded                               */
#define KIVI_ERR_UNSUPPORTED -9  /* valid in the reference, not implemented by this build */

#define KIVI_LAYOUT_REFERENCE 0  /* qB [U, K, N/fpi], scales/zeros [U, K, N/g]  (quant/matmul.py:189-191) */
#define KIVI_LAYOUT_KERNEL    1  /* qB [U, N/fpi, K], scales/zeros [U, N/g, K]  (quant/csrc/gemv_cuda.cu:255-259) */

/* Library identification. */
int         kivi_version(void);
const char* kivi_error_string(int code);
/* Number of kernel launches this library has enqueued since load (bench.py's gpu_launches). */
uint64_t    kivi_launch_count(void);

/* ------------------------------------------------------------------------------------------
 * Pack: asymmetric min/max quantisation along the LAST dim in groups of `group_size`,
 * OR-packed into int32 words.
 * Replaces triton_quantize_and_pack_along_last_dim(data, group_size, bit),
 *   quant/new_pack.py:217-252 (Triton _minmax_along_last_dim :158-177, ATen chain :238-242,
 *   Triton _pack_along_last_dim :132-154) -- one fused kernel instead of >= 9 launches.
 * Bit-exact on codes, scale and mn (fp16 rounding chain of SURVEY 8 a1); degenerate group
 * (mx == mn) -> code 0, scale 0.
 *   x     [rows, T]       fp16, contiguous
 *   code  [rows, T/fpi]   int32   (fpi = 32/bits)
 *   scale [rows, T/g]     fp16
 *   mn    [rows, T/g]     fp16
 * Requires bits in {2,4,8}, T % group_size == 0 (quant/new_pack.py:222), T % fpi == 0.
 * ------------------------------------------------------------------------------------------ */
int kivi_pack_lastdim_f16(const void* x, int64_t rows, int64_t T, int group_size, int bits,
                          void* code, void* scale, void* mn, void* stream);

/* ------------------------------------------------------------------------------------------
 * Batched "outer-dim" dequant-GEMV:  C[u_q, n] = sum_k A[u_q, k] * (scale*code + zero)[u_kv, k, n],
 * u_kv = u_q / (nh / nh_kv); groups and packing run along n.  fp32 accumulate, fp16 store.
 * Replaces
 *   layout KIVI_LAYOUT_KERNEL   : kivi_gemv.gemv_forward_cuda_outer_dim(in, kernel, scales, zeros,
 *                                 bit, group_size, nh, nh_kv), quant/csrc/gemv_cuda.h:12-20,
 *                                 quant/csrc/gemv_cuda.cu:511-557 (+ kernels :265-427);
 *   layout KIVI_LAYOUT_REFERENCE: the whole of cuda_bmm_fA_qB_outer, quant/matmul.py:178-219,
 *                                 WITHOUT its three transpose().contiguous() copies (:205,213-214).
 *   A      fp16, U_q = B*nh rows of K elements; row u at A + u*a_stride (elements), unit stride in k
 *   qB     int32, U_kv = B*nh_kv units, unit u at qB + u*qb_unit_stride (words);
 *            REFERENCE: word (k, n/fpi) at k*qb_row_stride + n/fpi
 *            KERNEL   : word (n/fpi, k) at (n/fpi)*qb_row_stride + k
 *   scales/zeros fp16, unit u at + u*sz_unit_stride (elements);
 *            REFERENCE: (k, n/g) at k*sz_row_stride + n/g ;  KERNEL: (n/g, k) at (n/g)*sz_row_stride + k
 *   C      fp16 [U_q, N] contiguous
 * Requires bits in {2,4} (8 also accepted on KIVI_LAYOUT_REFERENCE, the Triton surface
 * quant/matmul.py:112-175), nh % nh_kv == 0, group_size % fpi == 0, N % group_size == 0.
 * (M, the number of query rows per head, is 1: the reference kernel ignores blockIdx.z,
 *  quant/csrc/gemv_cuda.cu:538.)
 * ------------------------------------------------------------------------------------------ */
int kivi_bgemv_outer_f16(const void* A, int64_t a_stride,
                         const void* qB, int64_t qb_unit_stride, int64_t qb_row_stride,
                         const void* scales, const void* zeros, int64_t sz_unit_stride, int64_t sz_row_stride,
                         void* C, int B, int nh, int nh_kv, int K, int N,
                         int bits, int group_size, int layout, void* stream);

/* ------------------------------------------------------------------------------------------
 * Inner-dim (AWQ-style) GEMV: out[b, oc] = sum_ic in[b, ic] * (scale*code + zero)[oc, ic/g],
 * packing and groups along ic.
 * Replaces kivi_gemv.gemv_forward_cuda(in, kernel, scales, zeros, bit, group_size),
 *   quant/csrc/gemv_cuda.h:4-10, quant/csrc/gemv_cuda.cu:201-246 (kernels :60-184; 4-bit only,
 *   scales/zeros rows padded to sf_w = g64: ceil(ceil(IC/64/8)/2)*2*8, g128: ceil(IC/128/8)*8),
 *   and the Triton gemv_fwd / gemv_kernel_g64 of quant/gemv.py:16-90 (any bit, sf_w = IC/g).
 *   in [Bn, IC] fp16; kernel [OC, IC/fpi] int32; scales/zeros [OC, sf_w] fp16; out [Bn, OC] fp16.
 * The reference silently returns uninitialised memory for group sizes other than 64/128
 * (:227-245); here every group_size % fpi == 0 is computed.  IC % fpi == 0.
 * ------------------------------------------------------------------------------------------ */
int kivi_gemv_inner_f16(const void* in, const void* kernel, const void* scales, const void* zeros,
                        void* out, int Bn, int IC, int OC, int bits, int group_size, int64_t sf_w,
                        void* stream);

/* ------------------------------------------------------------------------------------------
 * Unpack + dequantise along the last dim in fp16: out = fp16(fp16(code * scale) + mn).
 * Replaces unpack_and_dequant_vcache / unpack_and_dequant_kcache (quant/new_pack.py:51-83),
 * the reference's own test oracle for the pack path.  bits in {2,4,8}.
 *   code [rows, T/fpi] int32; scale, mn [rows, T/g] fp16; out [rows, T] fp16.
 * ------------------------------------------------------------------------------------------ */
int kivi_unpack_dequant_lastdim_f16(const void* code, const void* scale, const void* mn,
                                    int64_t rows, int64_t T, int group_size, int bits,
                                    void* out, void* stream);

/* ==========================================================================================
 * Pre-allocated KIVI cache + fused decode attention (the hot path of
 * LlamaFlashAttention_KIVI.forward, models/llama_kivi.py:314-399, and its Mistral twin).
 *
 * The reference keeps a per-layer 9-tuple of tensors that it regrows with torch.cat every step
 * (:350-352, :391-395, :454-455).  Here the caller allocates fixed buffers once (sizes from
 * kivi_cache_sizes) and describes one LAYER's cache with a kivi_cache_t; `state` is a device
 * int32[8] shared by all layers of a model {tk, r, tv, L, vhead, kv_len, -, -}: tk = tokens in the
 * packed K store, r = tokens in the fp16 K window, tv = tokens in the packed V store, L = tokens in
 * the fp16 V window (ring buffer starting at vhead).  All sequences of the batch have the same
 * length, as in the reference (one kv_seq_len per cache, :309, :455); a left-padded batch keeps
 * that length and names each sequence's first real token (kivi_decode_attention_ragged_f16).
 * head_dim is 128 (every model the reference ships); group_size in {32,64,128};
 * residual_length % group_size == 0 (:344), residual_length in {32, 64, 128, 256}.
 * ========================================================================================== */
/* kivi_cache_t.flags.  KIVI_CACHE_OVERLAP_PROLOGUE: the caller promises that the kernel enqueued on the stream
 * directly before kivi_decode_attention_f16 never writes this cache (stores, windows) or its `state` -- true inside a
 * decoder layer, where that kernel produces q / k_new / v_new.  The q.K^T launch then starts under programmatic
 * dependent launch: it reads `state` and its first K blocks while that kernel drains, and waits for it only before
 * touching q / k_new.  Without the flag the q.K^T kernel is an ordinary launch (safe directly after
 * kivi_cache_advance / kivi_cache_prefill_f16 / a previous attention call on the same cache). */
#define KIVI_CACHE_OVERLAP_PROLOGUE 1
/* Bits 4..6 of kivi_cache_t.flags: how many query heads G of a KV head share one work unit of the decode attention
 * (their MMAs and every packed byte).  The ratio = nh/nh_kv query heads of a KV head form ceil(ratio / G) units, each of
 * which streams all of the KV head's packed blocks.  0 = chosen from the geometry: the largest G in {1, 2, 4} that divides
 * the ratio, except that odd ratios above 2 take 4 (ratio 1 -> 1, 2 -> 2, 3 -> 4, 4 -> 4, 5 -> 4, 6 -> 2, 7 -> 4, 8 -> 4);
 * or an explicit 1 / 2 / 4, whether or not it divides the ratio.
 * When it does not, the last unit of a KV head serves fewer than G heads: its missing heads compute on q = 0 and write
 * nothing.  kivi_decode_workspace_bytes and kivi_decode_attention_f16 must see the same value. */
#define KIVI_CACHE_GQA_CHUNK_SHIFT 4
#define KIVI_CACHE_GQA_CHUNK(g)    ((g) << KIVI_CACHE_GQA_CHUNK_SHIFT)

typedef struct kivi_cache {
    int32_t batch, num_heads, num_kv_heads, head_dim;
    int32_t k_bits, v_bits, group_size, residual_length;
    int32_t k_cap_blocks;   /* capacity of the K store in 128-token blocks   (kivi_cache_sizes out[0]) */
    int32_t v_cap_blocks;   /* capacity of the V store in 128-token blocks   (out[1]) */
    int32_t v_res_cap;      /* slots of the fp16 V ring buffer               (out[2]) */
    int32_t flags;          /* KIVI_CACHE_* bits, 0 = none */
    void* k_store;          /* out[3] bytes */
    void* v_store;          /* out[4] bytes */
    void* k_res;            /* out[5] bytes */
    void* v_res;            /* out[6] bytes */
    void* state;            /* device int32[8], shared by the layers of one model */
} kivi_cache_t;

/* Buffer sizes for a cache that can hold max_tokens tokens per sequence: out[0..2] = capacities
 * (k_cap_blocks, v_cap_blocks, v_res_cap), out[3..6] = bytes of k_store, v_store, k_res, v_res.
 * Both stores are sequences of 128 x 128 "inner x outer" blocks (K: channel x token, V: token x channel;
 * quantisation groups along the outer dim) whose codes are laid out as mma.sync A-operand fragments and
 * whose scales / zeros are laid out as the B-fragment builders read them: kivi_b200/csrc/kivi_decode.cuh. */
int kivi_cache_sizes(int batch, int num_kv_heads, int k_bits, int v_bits, int group_size,
                     int residual_length, int max_tokens, int64_t* out);

/* Prefill: split + quantise the prompt's K/V exactly as models/llama_kivi.py:425-452 and set `state`.
 *   k, v [B, Hkv, n, 128] fp16 contiguous (K after RoPE).  K: the first n - n%R tokens (all n if
 *   R | n, none if n < R) are quantised per channel in groups of g tokens straight into the blocked
 *   store (fused transpose + quantise); V: the first n - R tokens per token in groups of g channels. */
int kivi_cache_prefill_f16(const kivi_cache_t* cache, const void* k, const void* v, int n, void* stream);

/* Bytes of the scratch workspace kivi_decode_attention_f16 needs for this cache geometry and contexts of up to
 * max_kv_len tokens (negative: KIVI_ERR_*).  The caller allocates it once, ZERO-INITIALISED (it holds arrival
 * counters that every call leaves at zero), 256-B aligned; one workspace can serve all layers of a model when
 * the layers run on one stream. */
int64_t kivi_decode_workspace_bytes(const kivi_cache_t* cache, int max_kv_len);

/* One decode step of attention for one layer (models/llama_kivi.py:314-399):
 *   logits = [ q.Kq^T (dequantise in register) | q.K_full^T | q.k_new ]   each rounded to fp16 (:324-337)
 *   s      = fp16(logits * (1/sqrt(128))) (+ mask, max with finfo.min)     (:339, :369-372)
 *   p      = fp16(softmax_fp32(s))                                          (:375)
 *   out    = fp16( fp16(p[:tv].Vq) + fp16(p[tv:].[V_full; v_new]) )         (:382-384)
 * then, per unit, the cache data movement of :343-356 / :386-399: k_new joins the fp16 K window or,
 * when that completes R tokens, the window is quantised into the K store; v_new joins the fp16 V
 * ring and, once it holds more than R tokens, its oldest token is quantised into the V store.
 * `state` is READ ONLY here; call kivi_cache_advance once per step after the last layer.
 *   q [B, H, 128], k_new / v_new [B, Hkv, 128], out [B, H, 128]  fp16 contiguous
 *   mask: NULL or additive fp16 [B, kv_len + 1] (broadcast over heads, :364-372)
 *   workspace / workspace_bytes: see kivi_decode_workspace_bytes (scaled logits rows, per-block softmax
 *   statistics, partial output records, arrival counters); no bound on the context length
 *   dbg_logits / dbg_probs: NULL or fp16 [B, H, dbg_stride] receiving s and p (tests)
 *   max_kv_len: the value the workspace was sized with (>= kv_len + 1).
 * Two launches on `stream`, no CTA barrier in either: every warp of a persistent grid (one 16-warp CTA per SM) is an
 * autonomous worker that owns one contiguous range of the (unit, 128-token block) sequence and streams its packed
 * blocks HBM -> shared memory with cp.async.bulk (TMA) into private mbarrier stages.  (1) q.K^T: a warp writes the
 * fp16 logits of its blocks and one (max, sum exp) pair per unit it touches.  (2) p.V (programmatic dependent launch
 * on (1)): a warp normalises its logits slices with the unit's combined statistics, accumulates, and writes one
 * partial record per unit; the last arriver of a unit adds the records in fixed order, rounds, writes `out` and
 * updates the cache.  The contraction of a packed block runs on mma.sync (codes as exact fp16 denormals x a hi/lo
 * split of x*scale into two fp16, fp32 accumulate); the query heads of a KV head share the MMAs (GQA).  The split is
 * exact while |x*scale| >~ 2^-4 (the residual lo above fp16's smallest step 2^-24); x is brought into that range by
 * exact powers of two undone on the fp32 accumulators where it would not be: a query head with max|q| < 1/8 is scaled
 * into [1, 2) (2-bit K) or [4, 8) (4-bit K), and in a packed V block whose largest scale is below 1/16 the probabilities
 * are scaled up by a further power of two chosen from that scale and the softmax denominator.  Other inputs are computed
 * exactly as without the prescale.
 * Launch (1) reads `state` and its first K blocks at once: it is an ordinary launch unless cache->flags has
 * KIVI_CACHE_OVERLAP_PROLOGUE (see there). */
int kivi_decode_attention_f16(const kivi_cache_t* cache, const void* q, const void* k_new, const void* v_new,
                              const void* mask, void* out, void* workspace, int64_t workspace_bytes,
                              void* dbg_logits, void* dbg_probs, int64_t dbg_stride, int max_kv_len, void* stream);

/* The same step for a LEFT-PADDED batch: sequence b's tokens before position kv_start[b] are padding.
 *   kv_start: NULL (= all zeros: this is then kivi_decode_attention_f16) or a device int32[B]; with
 *   s_b = clamp(kv_start[b], 0, kv_len), the positions p < s_b of sequence b are excluded -- the same result as an
 *   additive finfo(fp16).min at those positions of `mask` -- and the new token is always visible.  `mask` keeps its
 *   meaning and may be combined with kv_start.  The offsets are read on the device: the call is CUDA-graph capturable
 *   and the caller may rewrite them between replays (not from the kernel enqueued directly before the call when
 *   cache->flags has KIVI_CACHE_OVERLAP_PROLOGUE).
 * A packed 128-token block (K or V) that lies wholly in the padding is neither read nor contracted; a partly padded block
 * and the fp16 window items are masked in their epilogues, so the HBM bytes read follow the visible tokens.  The cache
 * update is that of kivi_decode_attention_f16 (pad tokens stay in the K / V stores and their quantisation groups). */
int kivi_decode_attention_ragged_f16(const kivi_cache_t* cache, const void* q, const void* k_new, const void* v_new,
                                     const int32_t* kv_start, const void* mask, void* out, void* workspace,
                                     int64_t workspace_bytes, void* dbg_logits, void* dbg_probs, int64_t dbg_stride,
                                     int max_kv_len, void* stream);

/* The same step with a SLIDING WINDOW of `window` >= 1 tokens (Mistral's config.sliding_window; transformers keeps
 * kv_idx > q_idx - window).  With T = kv_len + 1 the shared length including the new token, sequence b sees the positions
 *   max(clamp(kv_start[b], 0, kv_len), T - window) <= p <= T - 1
 * (kv_start NULL = no padding) -- the same result as an additive finfo(fp16).min at the other positions of `mask`, which
 * keeps its meaning and may be combined with the window.  The window start moves every step and is computed on the device
 * from `state`: the call is CUDA-graph capturable.  The packed blocks before block j0 = min(n_blocks, max(0, T - window)
 * / 128) of each store lie wholly below the window: they are neither read nor counted in the work split, so the packed
 * bytes read per unit are (n_kb - j0k) * block_bytes(k_bits, g) + (n_vb - j0v) * block_bytes(v_bits, g), plus the fp16
 * windows (r + L) * 256 and the logits of the visible V blocks, at most ~ (window + 2 * 128) tokens' worth of each store
 * instead of kv_len.  A partly visible block and the window items are masked in their epilogues.  dbg_logits is defined
 * at the visible positions only; dbg_probs is 0 below the window start (entries of the blocks that are not read are
 * not written: pass a zeroed buffer, as for the ragged entry).  The cache update is that of
 * kivi_decode_attention_f16.  window < 1: KIVI_ERR_SHAPE. */
int kivi_decode_attention_window_f16(const kivi_cache_t* cache, const void* q, const void* k_new, const void* v_new,
                                     const int32_t* kv_start, int window, const void* mask, void* out, void* workspace,
                                     int64_t workspace_bytes, void* dbg_logits, void* dbg_probs, int64_t dbg_stride,
                                     int max_kv_len, void* stream);

/* Test hook: the (unit, item) work split of the two decode kernels evaluated on the host (kernel 0 = q.K^T, 1 = p.V cost
 * model); a unit has n_b packed blocks, n_w window items and the new token.  out_lo: 2 * (W + 1) ints, (unit, item) of the first
 * position of every range and of the end; out_owner: NULL or one int per position.  Returns the number of ranges W. */
int kivi_debug_range_split(int n_units, int n_b, int n_w, int w_cap, int kernel, int* out_lo, int* out_owner);

/* Test hook: the stage sequence of every warp of a ragged call (kernel 0 = q.K^T, 1 = p.V; unit_start[u] = the kv_start of
 * work unit u's sequence, clamped to kv_len), evaluated on the host with the kernels' own skip predicate and cursor walk.
 * issued / consumed: cap entries of 4 ints (warp, unit, item, half) each -- the copies the producer issues and the stages
 * the item loop waits on; n_out[0] / n_out[1] receive their counts.  Returns the number of ranges W or a KIVI_ERR_*. */
int kivi_debug_ragged_items(int n_units, int n_b, int n_w, int w_cap, int kernel, const int* unit_start, int kv_len,
                            int* issued, int* consumed, int64_t cap, int64_t* n_out);

/* Test hook: the same replay for a call of kivi_decode_attention_window_f16 at shared length T (the new token at T - 1)
 * with window >= 1.  n_b = the store's packed blocks; the item sequence of a unit starts at block j0 = min(n_b, max(0,
 * T - window) / 128), and items are reported in the numbering of the whole store (item j0 = packed block j0, item n_b + i =
 * window item i).  unit_start: NULL (no padding) or the kv_start of every unit's sequence. */
int kivi_debug_window_items(int n_units, int n_b, int n_w, int w_cap, int kernel, const int* unit_start, int T, int window,
                            int* issued, int* consumed, int64_t cap, int64_t* n_out);

/* Test hook: the work-unit geometry of the decode attention for GQA ratio `ratio` (>= 1) and kivi_cache_t.flags `flags`,
 * evaluated on the host with the code the entries use (KIVI_CACHE_GQA_CHUNK above).  Returns G, the query heads per work
 * unit, and stores ceil(ratio / G), the work units per KV head, in *hchunks; KIVI_ERR_SHAPE for ratio < 1 or a NULL
 * hchunks. */
int kivi_debug_gqa_chunk(int ratio, int flags, int* hchunks);

/* Advance `state` by one token (the bookkeeping of :343-356, :386-399); once per step, all layers. */
int kivi_cache_advance(const kivi_cache_t* cache, void* stream);

/* Copy the 8 words of `state` to host memory (synchronises `stream`).  state[6] is an error word that the decode kernels
 * set instead of touching memory when the device-side lengths exceed what the call declared (max_kv_len, window
 * capacities): KIVI_STATE_ERR_CAPACITY.  kivi_cache_refill_f16 / kivi_cache_shift_f16 / kivi_cache_shift_state set
 * KIVI_STATE_ERR_LENGTHS instead of writing when the device-side lengths are not those the call was given.
 * kivi_cache_reorder_f16 sets KIVI_STATE_ERR_ROWS instead of writing when a source row lies outside the batch.
 * kivi_cache_prefill_f16 / kivi_cache_import_f16 clear it. */
#define KIVI_STATE_ERR_CAPACITY 1
#define KIVI_STATE_ERR_LENGTHS  2
#define KIVI_STATE_ERR_ROWS     4   /* kivi_cache_reorder_f16: a source row outside [0, batch); nothing was written */
int kivi_cache_read_state(const kivi_cache_t* cache, int32_t* host_state8, void* stream);

/* ------------------------------------------------------------------------------------------
 * Continuous batching: the batch rows ("slots") of a live cache are reused without touching the other sequences.
 * All sequences keep the shared length T = tk + r = tv + L.  A new prompt of n <= T tokens goes into slot `seq`
 * right-aligned, at positions [T - n, T); the caller then sets kv_start[seq] = T - n and decodes with
 * kivi_decode_attention_ragged_f16.
 * ------------------------------------------------------------------------------------------ */
/* Refill the Hkv units of sequence `seq` (one layer) with a new prompt.  k, v [Hkv, n, 128] fp16 contiguous, K post-RoPE
 * at the prompt's own positions 0 .. n-1.  Lengths are passed by the host, as for kivi_cache_export_f16 (tk % R == 0,
 * r < R, L <= R, tk + r == tv + L, L == R once tv > 0; vhead < v_res_cap), and 1 <= n <= T.  With s = T - n the
 * sequence's units then hold EXACTLY what kivi_cache_prefill_f16 writes for the T-token sequence
 * x[p] = k/v[max(p - s, 0)] -- every block of the slot, the padding included -- with the V window rotated so that its
 * token i sits in ring slot (vhead + i) % v_res_cap.  The pad positions repeat the first real token: a per-channel K group
 * (packed, or still in the fp16 window until a later K flush) that mixes pad and real tokens then takes its min / max,
 * i.e. its scale and zero, from the real tokens alone; every other pad position is excluded by kv_start.
 * `state` and the other sequences are not written.  If the device-side lengths are not the ones passed, nothing is
 * written and KIVI_STATE_ERR_LENGTHS is set in state[6].  Three launches at most (K store, V store, windows). */
int kivi_cache_refill_f16(const kivi_cache_t* cache, int seq, const void* k, const void* v, int n,
                          int tk, int r, int tv, int L, int vhead, void* stream);

/* Drop the first `shift` positions of every sequence of one layer: block j of each K and V store moves to block
 * j - shift/128 (source and destination overlap; the move is ordered) and the vacated last shift/128 blocks that held
 * tokens are zeroed, as an import leaves the blocks past its lengths.  The fp16 K window and V ring do not move.
 * shift > 0, shift % max(128, R) == 0 (blocks, K flush periods and quantisation groups stay aligned), shift <= tk,
 * shift <= tv, with tk / tv the current lengths passed by the host (checked on the device like kivi_cache_refill_f16).
 * Call it for every layer, then kivi_cache_shift_state once.  The caller guarantees that no live sequence has
 * kv_start < shift: the dropped positions must be padding for every sequence that still decodes. */
int kivi_cache_shift_f16(const kivi_cache_t* cache, int shift, int tk, int tv, void* stream);

/* The bookkeeping of a shift, once per model after every layer's kivi_cache_shift_f16 (like kivi_cache_advance): tk, tv
 * and kv_len of `state` decrease by `shift`, r, L and vhead do not change, and every kv_start[b] decreases by `shift`
 * (kv_start: a device int32[B], or NULL).  RoPE positions are per sequence and do not change.  Same requirements on
 * `shift`; if the device-side tk or tv is below it, nothing changes and KIVI_STATE_ERR_LENGTHS is set. */
int kivi_cache_shift_state(const kivi_cache_t* cache, int shift, int32_t* kv_start, void* stream);

/* Beam search: reorder the batch rows of one layer.  For every b with src[b] != b, the Hkv units of sequence b become a
 * byte copy of the units of sequence src[b] AS THEY WERE BEFORE THE CALL, for any map (duplicates, swaps, cycles, chains).
 * A copied row receives the packed K blocks [0, ceil(tk/128)), the packed V blocks [0, ceil(tv/128)), and the whole fp16 K
 * window and V ring of each unit at full capacity (their win_unit swizzle kept; the ring head vhead is shared by all rows,
 * so ring slots map one to one).  tk and tv are read from `state` on the device, so a captured call follows the lengths as
 * they change between replays.  Nothing else is written: not the rows with src[b] == b, not the blocks past the live ones,
 * not `state`, not kv_start (the caller gathers kv_start[b] = kv_start[src[b]] itself).
 *   src: device int32[batch], read on the device (it may change between replays of a captured call).  If any entry lies
 *        outside [0, batch), nothing is written and KIVI_STATE_ERR_ROWS is set in state[6].
 *   scratch: device memory of at least kivi_cache_reorder_scratch_bytes(cache) bytes, 16-byte aligned.  A row that is
 *        rewritten AND read by another rewritten row is staged there first (launch 1); then every rewritten row copies
 *        from the scratch or from the cache (launch 2).  One scratch serves all layers of a model on one stream.
 * Two launches, no host synchronisation, no allocation; CUDA-graph capturable.  NULL pointers or a scratch that is too
 * small return KIVI_ERR_* before any launch. */
int64_t kivi_cache_reorder_scratch_bytes(const kivi_cache_t* cache);   /* one layer's rows at full capacity (< 0: KIVI_ERR_*) */
int kivi_cache_reorder_f16(const kivi_cache_t* cache, const int32_t* src, void* scratch, int64_t scratch_bytes, void* stream);

/* Copy the cache out in the reference's 9-tuple layout (models/llama_kivi.py:454-455); lengths are
 * passed by the host (it mirrors `state`).  k_code [U,128,tk/fpi] i32, k_scale/k_mn [U,128,tk/g],
 * k_full [U,r,128], v_code [U,tv,128/fpi] i32, v_scale/v_mn [U,tv,128/g], v_full [U,L,128]. */
int kivi_cache_export_f16(const kivi_cache_t* cache, int tk, int r, int tv, int L, int vhead,
                          void* k_code, void* k_scale, void* k_mn, void* k_full,
                          void* v_code, void* v_scale, void* v_mn, void* v_full, void* stream);

/* The inverse of kivi_cache_export_f16: load one layer's cache from the reference's 9-tuple (the object a model that
 * ran on the reference's hook holds, models/llama_kivi.py:454-455) and set `state` = {tk, r, tv, L, 0, tk + r}.
 * Same operand shapes as the export; tk % residual_length == 0, r < residual_length, L <= residual_length,
 * tk + r == tv + L (both count the tokens seen).  Pointers of empty parts (tk == 0, r == 0, tv == 0) may be NULL. */
int kivi_cache_import_f16(const kivi_cache_t* cache, int tk, int r, int tv, int L,
                          const void* k_code, const void* k_scale, const void* k_mn, const void* k_full,
                          const void* v_code, const void* v_scale, const void* v_mn, const void* v_full, void* stream);

/* ------------------------------------------------------------------------------------------
 * Glue kernels of the decode step around the hot path (not part of the KIVI operators; they
 * replace ~16 ATen elementwise launches per layer per step in kivi_b200/llama_kivi.py).  fp16 I/O,
 * arithmetic of the HF Llama modules the reference forks: every fp16 op rounds to fp16.
 *   kivi_add_rmsnorm_f16 : residual += x (x may be NULL); out = weight * fp16(residual * rsqrt(mean(residual^2)+eps));
 *                          rows >= 0, hidden % 8 == 0, hidden <= 16384; x, residual, weight and out 16-byte aligned
 *   kivi_rope_split_f16  : qkv [B,(H+2Hkv)*128] -> q [B,H,128], k [B,Hkv,128] (rotary at position pos[b], int64,
 *                          clamped to the table_rows rows of the cos / sin tables [table_rows, 128]), v;
 *                          1 <= B <= 65535, table_rows >= 1
 *   kivi_qk_norm_rope_split_f16 : kivi_rope_split_f16 with a per-head RMSNorm (Qwen3's q_norm / k_norm) before the
 *                          rotary: every q head n = fp16(q_norm_weight * fp16(x * rsqrt(mean(x^2) + eps))) over its 128
 *                          channels (fp32 statistics), every k head likewise with k_norm_weight [128]; v is copied.
 *                          Same requirements, plus non-NULL weights and a finite eps >= 0 (KIVI_ERR_SHAPE)
 *   kivi_silu_mul_f16   : gate_up [rows, 2*I] -> out [rows, I] = fp16(silu(gate)) * up;
 *                          1 <= rows <= 65535, I even; gate_up and out 4-byte aligned
 * Misaligned pointers return KIVI_ERR_ALIGN before any launch.
 * ------------------------------------------------------------------------------------------ */
int kivi_add_rmsnorm_f16(const void* x, void* residual, const void* weight, void* out,
                         int rows, int hidden, float eps, void* stream);
int kivi_rope_split_f16(const void* qkv, const void* cos_table, const void* sin_table, const void* pos,
                        void* q, void* k, void* v, int batch, int num_heads, int num_kv_heads, int table_rows,
                        void* stream);
int kivi_qk_norm_rope_split_f16(const void* qkv, const void* cos_table, const void* sin_table, const void* pos,
                                const void* q_norm_weight, const void* k_norm_weight, float eps,
                                void* q, void* k, void* v, int batch, int num_heads, int num_kv_heads, int table_rows,
                                void* stream);
int kivi_silu_mul_f16(const void* gate_up, void* out, int rows, int intermediate, void* stream);

/* ------------------------------------------------------------------------------------------
 * Prompt attention: the attention of a prompt over itself, in the prompt pass (not over the cache).
 *   q [B, H, n, 128], k / v [B, Hkv, n, 128] fp16 with a contiguous head dimension and element strides
 *     q_sb / q_sh / q_st (batch, head, token) and kv_sb / kv_sh / kv_st (shared by k and v): the strided views of
 *     the q / k / v projections.  K after RoPE.
 *   out [B, n, H, 128] fp16 contiguous (the layout o_proj reads).
 * Query head h reads KV head h / (H / Hkv); K and V are never expanded.  Query i of sequence b sees the keys
 *   lo <= j <= i,   lo = max(s_b, window > 0 ? i - window + 1 : 0),   s_b = clamp(kv_start[b], 0, n)
 * (kv_start NULL = 0; transformers' kv_idx > q_idx - window).  A query with no visible key (i < s_b) gets zeros.
 * Scale 1/sqrt(128); logits and the softmax in fp32 with a running maximum and sum; P rounded to fp16 for the P.V
 * product; fp32 accumulators.  Offsets are 64-bit.  Key tiles with no visible key for any query of a tile are not read,
 * so the work and the K / V bytes follow the visible pairs.
 * Requirements: q, k, v, out non-NULL and 16-byte aligned, every stride a multiple of 8 elements, kv_start 4-byte
 * aligned; batch in [1, 65535], num_heads >= 1, n >= 1, window >= 0 (KIVI_ERR_SHAPE), num_heads % num_kv_heads == 0
 * (KIVI_ERR_GQA).  One launch, no allocation, no synchronisation; CUDA-graph capturable.
 * ------------------------------------------------------------------------------------------ */
int kivi_prompt_attention_f16(const void* q, const void* k, const void* v, void* out,
                              int batch, int num_heads, int num_kv_heads, int n,
                              int64_t q_sb, int64_t q_sh, int64_t q_st,
                              int64_t kv_sb, int64_t kv_sh, int64_t kv_st,
                              const int32_t* kv_start, int window, void* stream);

/* ------------------------------------------------------------------------------------------
 * Suffix prompt attention: the last m tokens of a prompt over the whole prompt, whose first n - m tokens' K / V were
 * computed earlier (a stored prefix).
 *   q [B, H, m, 128]: the queries at positions n - m .. n - 1; k / v [B, Hkv, n, 128]; out [B, m, H, 128] fp16
 *   contiguous; strides, kv_start and window as in kivi_prompt_attention_f16.
 * Query t sits at position i = n - m + t and sees the keys max(s_b, i - window + 1) <= j <= i: the rule above with i
 * counted from the start of the keys.  The same kernel runs both entries and visits key tiles in ascending absolute
 * position, so a row meets the tiles where it sees a key in the same order in both.  Where n - m is not a multiple of a
 * CTA's tokens, a row may also visit tiles in which it sees nothing; those leave its online softmax exactly unchanged
 * (alpha 0 with no key seen yet, 1 after; every p 0).  Row t therefore equals row n - m + t of kivi_prompt_attention_f16
 * on the same q / k / v bit for bit (m = n: the same output).  Tiles below the window of a CTA's first query and below kv_start are never read, so the work
 * follows the suffix's visible pairs, not n^2.
 * Requirements: those of kivi_prompt_attention_f16, and 1 <= m <= n (KIVI_ERR_SHAPE).  One launch, no allocation, no
 * synchronisation; CUDA-graph capturable.
 * ------------------------------------------------------------------------------------------ */
int kivi_prompt_attention_suffix_f16(const void* q, const void* k, const void* v, void* out,
                                     int batch, int num_heads, int num_kv_heads, int m, int n,
                                     int64_t q_sb, int64_t q_sh, int64_t q_st,
                                     int64_t kv_sb, int64_t kv_sh, int64_t kv_st,
                                     const int32_t* kv_start, int window, void* stream);

/* Greedy sampling fused with its collective (the only exchange of the data-parallel decode, SURVEY 8e; the reference has
 * none).  next_local[b] = argmax_v logits[b, v] (first index among equal maxima, as torch.argmax; logits fp32 [batch, vocab],
 * models/llama_kivi.py:881); ids_feedback (may be NULL) receives the same ids (the next step's input buffer).
 * peer_buffers: NULL (one GPU), or a DEVICE array of `world` pointers, entry p = rank p's exchange buffer -- one symmetric
 * allocation per rank (peer-mapped over NVLink / NVSwitch), laid out as int64 tokens[2][world * batch] followed by
 * uint64 arrived[world], zero-initialised.  The kernel stores its ids into slot [step & 1][rank * batch + b] of EVERY rank's
 * buffer with plain peer stores, releases arrived[rank] on every peer, and waits (bounded, *err = 1 on time-out) until the
 * ids of all ranks for this step have arrived in its own buffer.  `step` is a device int32 the caller increments before each
 * call (the same on all ranks); all calls are CUDA-graph capturable. */
int kivi_greedy_sample_exchange_f32(const void* logits, int batch, int vocab, void* next_local, void* ids_feedback,
                                    const void* peer_buffers, int rank, int world, const void* step, void* err, void* stream);

/* Sampling: next_local[b] = one draw from row b of logits (fp32 [batch, vocab]) after temperature, top-k and top-p, applied in
 * the order of HF's logits warpers.  One launch, no sort, no scratch buffer.  All per-row parameters are DEVICE arrays [batch],
 * read by the kernel, so a captured call keeps working when the caller changes a row's parameters between replays.
 *   temperature[b] == 0 : the row is greedy: exactly the id of kivi_greedy_sample_exchange_f32 (first index among equal maxima, a
 *                         NaN wins); draw[b] does not change.  (A negative or NaN temperature is the caller's error.  The values live on the
 *                         device, so neither this entry point nor its ctypes wrapper can see them without a synchronisation;
 *                         kivi_b200's set_sampling / generate / serve validate them on the host before they are uploaded.
 *                         The kernel takes such a row as greedy rather than dividing by it.)
 *   otherwise             x_v = logits[b, v] / temperature[b] in fp32; a NaN logit counts as -inf.
 *   top_k[b] = k        : k <= 0 or k >= vocab: off.  Else keep every v with x_v >= the k-th largest x of the row (ties at the
 *                         threshold are all kept, as TopKLogitsWarper does).
 *   top_p[b] = p        : p >= 1: off.  Else, over the softmax of what top-k kept, keep the smallest set of highest-probability
 *                         tokens whose mass reaches p; p <= 0 keeps the maximum only.  Tokens of EQUAL logit stand or fall
 *                         together (TopPLogitsWarper drops part of a tie by sort order; here the whole tie is kept).
 *   draw                : u = (Philox4x32-10(key = seed[b], counter = (draw[b], 0)).x >> 8) * 2^-24, in [0, 1).  The id is the
 *                         first kept token, in ASCENDING TOKEN-ID order, whose cumulative kept mass exceeds u * S (S = the kept
 *                         mass) -- not torch.multinomial's order, and a pure function of (row, parameters, seed[b], draw[b]):
 *                         the batch size, the row's index and the run do not matter.  Then draw[b] += 1.
 * Tokens at -inf are never kept and never counted; at least one token is kept.  A row with a +inf among its scaled logits, or
 * with no finite logit, gets the greedy id and does not consume a draw.
 * Masses are exp(x_v - max_v x_v) rounded to multiples of 2^-40 and summed, compared and walked as integers; a token whose mass
 * rounds to 0 can be kept but cannot be drawn.
 * ids_feedback (may be NULL) receives the same ids (the next step's input buffer), next_local / ids_feedback are int64 [batch].
 * dbg_u / dbg_kept (NULL, or [batch]; tests): u and the number of kept tokens (0 and 1 for a row that took the greedy id).
 * Requirements: batch >= 0, 1 <= vocab <= 2^22; argument errors return KIVI_ERR_* before any launch.  Graph-capturable. */
int kivi_sample_f32(const void* logits, int batch, int vocab, const float* temperature, const int32_t* top_k, const float* top_p,
                    const uint64_t* seed, uint64_t* draw, void* next_local, void* ids_feedback, float* dbg_u, int32_t* dbg_kept,
                    void* stream);

/* Logits processing: scores = the logits after repetition, presence and frequency penalties, EOS suppression below a
 * minimum length and the masking of finished rows, for the greedy kernel or kivi_sample_f32 to choose from.  logits and
 * scores are fp32 [batch, vocab], distinct buffers; logits is only read.  Per-row state and parameters are DEVICE arrays, read
 * by the kernel, so a captured call follows later changes:
 *   counts   int32 [batch, vocab]       how many times each token was generated (kivi_logits_record)
 *   seen     uint32 [batch, ceil(vocab / 32)]   the prompt's tokens, bit v & 31 of word v >> 5
 *   n_new    int32 [batch], finished uint8 [batch]   (kivi_logits_record)
 *   repetition, presence, frequency   fp32 [batch];  min_new int32 [batch]
 *   eos_ids  int64 [n_eos], 0 <= n_eos <= 8 (may be NULL when n_eos = 0); ids outside [0, vocab) match no token
 * For each token v of row b, with x = logits[b, v], c = counts[b, v], in this order, every step one IEEE fp32 operation
 * rounded to nearest (no contraction):
 *   1. repetition (transformers' RepetitionPenaltyLogitsProcessor): if v is in seen or c > 0:  x = x < 0 ? x * p : x / p
 *   2. frequency, then presence (vLLM's order, generated tokens only):  x = x - f * float(c);  if c > 0: x = x - pres
 *   3. if n_new[b] < min_new[b]: x = -inf for every v in eos_ids (MinLength / MinNewTokensLength LogitsProcessor)
 *   4. if finished[b]: x = 0 at v = pad_id, -inf everywhere else (the rule of the `unfinished` mask of HF's greedy and
 *      sampling loops: both selection kernels then pick pad_id -- the greedy one as the only maximum, the sampler as
 *      the one finite token, which it keeps whatever its top-k and top-p; it consumes a draw like any sampled row)
 * A row with p == 1 and presence, frequency +0 skips steps 1-2 and reads neither counts nor seen (its scores equal its logits
 * bit for bit, NaN payloads included); a finished row reads nothing but its flag.  Parameter VALUES are the caller's
 * responsibility (kivi_b200's processing_rows validates them on the host).
 * Requirements: 0 <= batch <= 65535, vocab >= 1, 0 <= pad_id < vocab, seen 4-byte aligned; 128-bit accesses when vocab % 4 == 0
 * and logits / scores / counts are 16-byte aligned.  Argument errors return KIVI_ERR_* before any launch.  One launch,
 * graph-capturable. */
int kivi_logits_process_f32(const void* logits, void* scores, int batch, int vocab, const int32_t* counts, const uint32_t* seen,
                            const int32_t* n_new, const uint8_t* finished, const float* repetition, const float* presence,
                            const float* frequency, const int32_t* min_new, const int64_t* eos_ids, int n_eos, int64_t pad_id,
                            void* stream);

/* The state update after the token choice: t = tokens[b] (int64 [batch], e.g. next_local of the selection kernel):
 * counts[b, t] += 1 (t in [0, vocab)), n_new[b] += 1, finished[b] = 1 if t is one of eos_ids[0 .. n_eos).  One thread per row;
 * the same state layout and requirements as kivi_logits_process_f32 (batch >= 0).  One launch, graph-capturable. */
int kivi_logits_record(const void* tokens, int batch, int vocab, int32_t* counts, int32_t* n_new, uint8_t* finished,
                       const int64_t* eos_ids, int n_eos, void* stream);

/* Log-probabilities of chosen tokens under the softmax of their row, and the row's top N.  x = logits fp32 [batch, vocab]
 * (only read), tokens int64 [batch] (e.g. next_local of the selection kernel), 0 <= n_top = N <= 20.  Per row b:
 *   lse_b = m + log(sum_v exp(x[b, v] - m)), m the row's maximum (exp in fp32, the sum, the log and lse in fp64)
 *   logprob[b]            = float(x[b, t] - lse_b), t = tokens[b]; NaN when t is outside [0, vocab)
 *   top_ids[b, 0 .. N)    the N largest x[b, .] in descending order, ties by ascending id; a NaN ranks above +inf (all NaNs
 *                         first, by id, as torch.topk orders them) and -0 equals +0.  N > vocab: entries vocab .. N-1 are -1
 *   top_logprobs[b, j]    = float(x[b, top_ids[b, j]] - lse_b) (-inf for an id of -1), each value rounded once from fp64,
 *                         so the chosen token's logprob equals its entry in the list bit for bit when it appears there.
 * Special values give what torch.log_softmax(row.double()) gives: a NaN or +inf anywhere in the row, or a row with no finite
 * value, makes every value of the row NaN (ids are still ranked); a -inf token of a row with a finite maximum gets -inf.
 * Bound against the fp64 log_softmax r of the same row: |value - r| <= 2^-24 |r| + 2^-22 + 2^-24 * 104 (DESIGN.md: the final
 * rounding, exp's error, and the rounding of x - m for the terms exp does not flush to 0).
 * Row b's outputs depend only on row b and tokens[b] (every sum has a fixed order), and are bit-identical from run to run.
 * top_ids / top_logprobs ([batch, N]) may be NULL when N = 0.  Requirements: batch >= 0, 1 <= vocab <= 2^22; argument errors
 * return KIVI_ERR_* before any launch.  One launch, no scratch buffer, graph-capturable. */
int kivi_token_logprobs_f32(const void* logits, int batch, int vocab, const int64_t* tokens, int n_top, float* logprob,
                            int64_t* top_ids, float* top_logprobs, void* stream);

/* LoRA deltas of one projection group (q|k|v: 3 segments, o: 1, gate|up: 2, down: 1) for a batch of rows, each row with its
 * own adapter.  S adapters are stacked in slots 0 .. S-1:
 *   A      fp16 [S, n_seg, R, in]   (lora_A of segment g at [s, g]; ranks below R zero-padded)
 *   B      fp16 [S, out_total, R]   (lora_B rows of every segment, one after the other; zero-padded columns)
 *   scale  fp32 [S]                 (alpha / r, or alpha / sqrt(r) under rsLoRA)
 *   seg_off HOST int [n_seg + 1]    the segments' first columns, 0 = seg_off[0] < ... < seg_off[n_seg] = out_total;
 *                                   seg(o) = the g with seg_off[g] <= o < seg_off[g + 1]
 *   idx    int32 [rows] (device)    row b's slot; idx[b] < 0 (no adapter) or idx[b] >= S: row b of y is NOT written
 * x fp16 [rows, in] and y fp16 [rows, out_total] are contiguous.  For row b with slot a = idx[b] in [0, S):
 *   kivi_lora_shrink_f16:  ws[c, b, g R + j] = sum over k in chunk c of x[b, k] A[a, g, j, k]          (fp32, chunks of 512)
 *   kivi_lora_expand_f16:  t[b, e] = sum_c ws[c, b, e] (chunk order);
 *                          y[b, o] = fp16(float(y[b, o]) + d), d = scale[a] * sum_j B[a, o, j] t[b, seg(o) R + j],
 *                          except that d == 0 leaves y[b, o]'s bits as they are.
 * The shrink must precede the expand on the stream, with the same rows, in, n_seg, R, S and idx: two launches per group.
 * ws: fp32 workspace of kivi_lora_workspace_bytes(rows, in, n_seg, R) bytes, ceil(in / 512) * rows * n_seg * R floats.
 * Each CTA serves one slot and gathers that slot's rows from idx, so each present adapter's A and B are read once per call.
 * Every sum has an order fixed by the shapes: row b's output depends only on row b's x, y and adapter, bit for bit -- not on
 * the other rows, their adapters, S or the grid -- and is identical from run to run and under graph replay.
 * Error bound (finite inputs, no overflow): with v = y + scale * sum_j B[o, j] sum_k x_k A[g, j, k] in float64 and
 * M = |scale| sum_j |B[o, j]| sum_k |x_k A[g, j, k]|,
 *     |y_out - v| <= 2^-11 |v| + (1 + 2^-11) c (M + |v|) + 2^-25,    c = (in + R + 3) 2^-24
 * (fp16 x fp16 products are exact in fp32; the fp32 sums of length in and R, the scale and the add round each partial sum
 * at most once per term; then the final fp16 rounding, relative below 2^-11 and absolute 2^-25 among subnormals.)
 * Requirements: 0 <= rows <= 1024, in % 8 == 0 and in >= 8, 1 <= S <= 65535, n_seg in {1, 2, 3}, R % 8 == 0 and
 * 8 <= R <= 128 (KIVI_ERR_SHAPE); x, A, B 16-byte aligned (KIVI_ERR_ALIGN); non-NULL pointers (KIVI_ERR_NULL); the
 * expand also checks seg_off (KIVI_ERR_SHAPE).  Argument errors return before any launch; rows == 0 launches nothing.  No
 * allocation, graph-capturable (seg_off is read at the call).  kivi_lora_workspace_bytes returns KIVI_ERR_SHAPE (< 0) for
 * shapes the entries refuse. */
int64_t kivi_lora_workspace_bytes(int rows, int in, int n_seg, int rank);
int kivi_lora_shrink_f16(const void* x, int rows, int in, const void* A, int S, int n_seg, int rank, const int32_t* idx,
                         float* ws, void* stream);
int kivi_lora_expand_f16(const float* ws, int rows, int in, const void* B, const float* scale, int S, int n_seg, int rank,
                         const int* seg_off, const int32_t* idx, void* y, int out_total, void* stream);

/* Tensor-parallel residual-add + RMSNorm: the all-reduce after o_proj / down_proj fused into the norm that follows it.
 * With the rows of the attention heads and of the MLP columns sharded over `world` ranks, rank p holds a partial sum
 * partial_p [rows, hidden] fp16 of the projection.  Every rank computes the same bits:
 *     x = fp16( sum_{p = 0 .. world-1} fp32(partial_p) )      (fp32 additions in rank order, starting from partial_0)
 *     residual += x;  out = weight * fp16(residual * rsqrt(mean(residual^2) + eps))
 * i.e. exactly kivi_add_rmsnorm_f16(x, residual, weight, out).
 *
 * peer_buffers: NULL (world must be 1: x is the whole sum and the call IS kivi_add_rmsnorm_f16), or a DEVICE array of
 * `world` pointers, entry p = rank p's buffer -- one symmetric allocation per rank (peer-mapped over NVLink / NVSwitch),
 * zero-initialised, 16-byte aligned:
 *     half     partial[2][rows_max][hidden]    this rank's partial sums, double-buffered: call c uses slot c & 1
 *     uint64   arrived[world]                  arrived[q] = the last call number rank q has announced here
 * The caller writes its partial of call c into slot (c & 1) of ITS OWN buffer (the projection GEMM's output) before the call;
 * x is ignored.  The call number is e = *epoch + call + 1 (epoch: device int64; call: the index of this call within a
 * replay).  The kernel
 *   1. stores e into arrived[rank] of every peer (red.release.sys max, so pre-set counters are harmless),
 *   2. waits (ld.acquire.sys) until arrived[q] >= e for every q in its own buffer -- bounded: after ~ a second *err = 1 and it goes on
 *      instead of hanging the GPU (the host raises),
 *   3. reads slot (c & 1) of every peer's buffer and reduces.
 * The caller advances *epoch by the number of calls per replay, which must be even (two per layer), once per replay and
 * inside the same CUDA graph; consecutive calls then alternate slots across replays too.
 * Why two slots are enough: a peer reads rank r's slot (c & 1) during call c.  Rank r overwrites that slot next for call c+2,
 * with the GEMM that precedes call c+2 on its stream, i.e. after its call c+1 has returned -- and call c+1 returns only after
 * every peer has arrived at c+1, which each peer does at the start of its call c+1, after its call c (and all of its reads
 * of slot c & 1) has completed on its stream.  So no slot is written while a peer may still read it.
 * A row is split over a cluster of `cluster` CTAs (1, 2, 4 or 8; 0 = the default, one CTA per row) whose reductions are
 * arranged to give the same bits for every width.
 * Requirements: rows >= 0, rows <= rows_max, hidden % 8 == 0, hidden <= 16384, 1 <= world <= 8, 0 <= rank < world,
 * residual / weight / out 16-byte aligned; argument errors return KIVI_ERR_* before any launch.  Graph-capturable. */
int kivi_allreduce_add_rmsnorm_f16(const void* x, void* residual, const void* weight, void* out, int rows, int hidden,
                                   float eps, const void* peer_buffers, int rank, int world, int rows_max, int call,
                                   const void* epoch, void* err, int cluster, void* stream);

#ifdef __cplusplus
}
#endif
#endif /* KIVI_B200_H */
