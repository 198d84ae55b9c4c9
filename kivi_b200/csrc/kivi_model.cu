// kivi_model.cu -- small fused glue kernels of the decode step around the hot path (sm_90a):
// residual-add + RMSNorm, RoPE + q/k/v split, SiLU*mul.  They replace ~16 ATen elementwise launches per
// layer per step with 4; arithmetic follows the HF Llama modules the reference forks
// (models/llama_kivi.py star-imports transformers.models.llama): every fp16 op rounds to fp16.
#include "kivi_common.cuh"

#include <cooperative_groups.h>

#include <type_traits>

namespace cg = cooperative_groups;

namespace kivi {

constexpr int kNormThreads = 512, kNormMaxIter = 4;
constexpr int kNormMaxHidden = kNormMaxIter * kNormThreads * 8;           // 16384: every 8-element slice held in registers

// One row of residual-add + RMSNorm, the body of add_rmsnorm_kernel and allreduce_add_rmsnorm_kernel:
//   residual (fp16, in/out) += addend;  out = weight * fp16( residual * rsqrt(mean(residual^2) + eps) )
// (LlamaRMSNorm.forward: fp32 statistics, cast to fp16, then multiply by the fp16 weight).
// The row has 512 threads, spread over a cluster of C CTAs of 512 / C; thread vt owns the 8-element slices vt, vt + 512, ...
// and keeps them in registers between the two passes.  The per-thread and per-warp sums of squares and the order in which
// the 16 warp sums are added do not depend on C, so neither do the bits.
// ADD: addend(i) returns slice i of the addend as 4 __half2 (a uint4); without ADD the residual is only normalised.
template <int C, bool ADD, class Addend>
__device__ __forceinline__ void add_rmsnorm_row(Addend addend, __half* __restrict__ r, const __half* __restrict__ w,
                                                __half* __restrict__ out, int hidden, float eps, int vt)
{
    constexpr int kWarps = kNormThreads / C / 32;
    __shared__ float red[kWarps];
    const int nvec = hidden / 8;
    uint4 v[kNormMaxIter];
    float ss = 0.f;
    #pragma unroll
    for (int it = 0; it < kNormMaxIter; ++it) {
        const int i = vt + it * kNormThreads;
        if (i < nvec) {
            uint4 a;
            if (ADD) a = addend(i);                                      // issued first: the peer loads of the all-reduce
            uint4 u = *reinterpret_cast<const uint4*>(r + i * 8);
            __half2* h = reinterpret_cast<__half2*>(&u);
            if (ADD) {
                const __half2* ah = reinterpret_cast<const __half2*>(&a);
                #pragma unroll
                for (int e = 0; e < 4; ++e) h[e] = __hadd2_rn(h[e], ah[e]);
                *reinterpret_cast<uint4*>(r + i * 8) = u;
            }
            #pragma unroll
            for (int e = 0; e < 4; ++e) { const float2 f = __half22float2(h[e]); ss = fmaf(f.x, f.x, fmaf(f.y, f.y, ss)); }
            v[it] = u;
        }
    }
    ss = warp_sum(ss);
    if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = ss;
    float tot = 0.f;
    if constexpr (C == 1) {
        __syncthreads();
        #pragma unroll
        for (int i = 0; i < kWarps; ++i) tot += red[i];
    } else {
        cg::cluster_group cluster = cg::this_cluster();
        cluster.sync();
        #pragma unroll
        for (int c = 0; c < C; ++c) {
            const float* rr = cluster.map_shared_rank(red, c);
            #pragma unroll
            for (int i = 0; i < kWarps; ++i) tot += rr[i];
        }
        cluster.sync();                                                  // no CTA leaves while a peer CTA reads its red[]
    }
    const float rs = rsqrtf(tot / (float)hidden + eps);
    #pragma unroll
    for (int it = 0; it < kNormMaxIter; ++it) {
        const int i = vt + it * kNormThreads;
        if (i < nvec) {
            const __half2* h = reinterpret_cast<const __half2*>(&v[it]);
            const uint4 wv = __ldg(reinterpret_cast<const uint4*>(w) + i);
            const __half2* wh = reinterpret_cast<const __half2*>(&wv);
            uint4 o;
            __half2* oh = reinterpret_cast<__half2*>(&o);
            #pragma unroll
            for (int e = 0; e < 4; ++e) {
                const float2 f = __half22float2(h[e]);
                oh[e] = __hmul2_rn(wh[e], __floats2half2_rn(f.x * rs, f.y * rs));
            }
            *reinterpret_cast<uint4*>(out + i * 8) = o;
        }
    }
}

// One CTA per row; ADD: the addend is x (fp16, [rows, hidden]).
template <bool ADD>
__global__ void __launch_bounds__(kNormThreads)
add_rmsnorm_kernel(const __half* __restrict__ x, __half* __restrict__ residual, const __half* __restrict__ w,
                   __half* __restrict__ out, int hidden, float eps)
{
    const int row = blockIdx.x;
    const int64_t row_off = (int64_t)row * hidden;
    add_rmsnorm_row<1, ADD>([&](int i) { return __ldg(reinterpret_cast<const uint4*>(x + row_off) + i); },
                            residual + row_off, w, out + row_off, hidden, eps, threadIdx.x);
}

// qkv [B, (H + 2*Hkv) * 128] -> q [B,H,128], k [B,Hkv,128] (both rotated), v [B,Hkv,128]
// apply_rotary_pos_emb: x*cos + rotate_half(x)*sin, each op rounded to fp16; cos/sin rows = position pos[b]
__global__ void __launch_bounds__(64)
rope_split_kernel(const __half* __restrict__ qkv, const __half* __restrict__ cos_t, const __half* __restrict__ sin_t,
                  const long long* __restrict__ pos, __half* __restrict__ q, __half* __restrict__ k, __half* __restrict__ v,
                  int H, int Hkv, int table_rows)
{
    constexpr int D = 128;
    // the q.K^T kernel that follows is launched with programmatic serialization: let it set up and start streaming K blocks
    // while this kernel runs (it waits for our completion before it reads q / k / v)
    asm volatile("griddepcontrol.launch_dependents;");
    const int b = blockIdx.y, head = blockIdx.x, i = threadIdx.x;            // i < 64: pair (i, i + 64)
    const __half* src = qkv + ((int64_t)b * (H + 2 * Hkv) + head) * D;
    if (head >= H + Hkv) {                                                   // v: plain copy
        __half* dst = v + ((int64_t)b * Hkv + head - H - Hkv) * D;
        dst[i] = src[i]; dst[i + 64] = src[i + 64];
        return;
    }
    long long p = pos[b];
    p = p < 0 ? 0 : (p >= table_rows ? table_rows - 1 : p);                  // never read outside the tables (the host checks the range)
    const __half c0 = cos_t[p * D + i], c1 = cos_t[p * D + i + 64];
    const __half s0 = sin_t[p * D + i], s1 = sin_t[p * D + i + 64];
    const __half x0 = src[i], x1 = src[i + 64];
    __half* dst = head < H ? q + ((int64_t)b * H + head) * D : k + ((int64_t)b * Hkv + head - H) * D;
    dst[i] = __hadd_rn(__hmul_rn(x0, c0), __hmul_rn(__hneg(x1), s0));       // rotate_half: (-x2, x1)
    dst[i + 64] = __hadd_rn(__hmul_rn(x1, c1), __hmul_rn(x0, s1));
}

// gu [rows, 2*I] (gate | up) -> out [rows, I] = fp16(silu(gate)) * up
__global__ void __launch_bounds__(256)
silu_mul_kernel(const __half* __restrict__ gu, __half* __restrict__ out, int I)
{
    const int row = blockIdx.y;
    const int i = (blockIdx.x * blockDim.x + threadIdx.x) * 2;
    if (i >= I) return;
    const float2 g = __half22float2(*reinterpret_cast<const __half2*>(gu + (int64_t)row * 2 * I + i));
    const __half2 u = *reinterpret_cast<const __half2*>(gu + (int64_t)row * 2 * I + I + i);
    const __half2 a = __floats2half2_rn(g.x / (1.f + expf(-g.x)), g.y / (1.f + expf(-g.y)));
    *reinterpret_cast<__half2*>(out + (int64_t)row * I + i) = __hmul2_rn(a, u);
}

// Whether the candidate (ov, oi) replaces (best, bi) when two argmax results merge: the larger value, the lower index among
// equal values, and a NaN beats every number (the lower index among NaNs), like torch.argmax.
__device__ __forceinline__ bool argmax_takes(float ov, int oi, float best, int bi)
{
    return (ov != ov) ? (!(best != best) || oi < bi) : (!(best != best) && (ov > best || (ov == best && oi < bi)));
}

// ------------------------------------------------------------------------------------------------
// Greedy sampling fused with its collective.  One block per sequence: argmax over the vocabulary (first index among equal
// maxima, like torch.argmax), then thread 0 stores the id into this rank's slot of EVERY rank's token buffer -- plain stores
// to peer memory over NVLink / NVSwitch (the buffers are one symmetric allocation, torch.distributed._symmetric_memory) --
// and releases a per-rank arrival counter on every peer.  Block 0 then waits (bounded) until all ranks' ids of this step have
// arrived here.  Argmax is local to a sequence, so the data-parallel replicas exchange 8 bytes per sequence and nothing of
// the next step depends on the exchange: no rank ever blocks another one's critical path.
//   peer[p]  : rank p's buffer: int64 tokens[2][world * B] (double-buffered by step parity), then uint64 arrived[world]
//   step     : device counter, incremented by the caller BEFORE the launch (inside the same CUDA graph)
// ------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256)
greedy_exchange_kernel(const float* __restrict__ logits, int V, long long* __restrict__ next_local, long long* __restrict__ ids_feedback,
                       long long* const* __restrict__ peer, int B, int rank, int world, const int* __restrict__ step_ptr, int* __restrict__ err)
{
    __shared__ float smax[8];
    __shared__ int sidx[8];
    const int b = blockIdx.x, tid = threadIdx.x;
    const float* row = logits + (long long)b * V;
    float best = -INFINITY;
    int bi = 0x7fffffff;
    for (int i = tid; i < V; i += 256) {
        const float v = row[i];
        if (v > best || (v == best && i < bi) || (v != v && !(best != best))) { best = v; bi = i; }   // a NaN wins, like torch.argmax
    }
    #pragma unroll
    for (int o = 16; o >= 1; o >>= 1) {
        const float ov = __shfl_xor_sync(0xffffffffu, best, o);
        const int oi = __shfl_xor_sync(0xffffffffu, bi, o);
        if (argmax_takes(ov, oi, best, bi)) { best = ov; bi = oi; }
    }
    if ((tid & 31) == 0) { smax[tid >> 5] = best; sidx[tid >> 5] = bi; }
    __syncthreads();
    if (tid == 0) {
        for (int w = 1; w < 8; ++w) {
            const float ov = smax[w];
            const int oi = sidx[w];
            if (argmax_takes(ov, oi, best, bi)) { best = ov; bi = oi; }
        }
        const long long tok = bi;
        next_local[b] = tok;
        if (ids_feedback) ids_feedback[b] = tok;
        if (peer) {
            const int step = *step_ptr;
            const long long slot = (long long)(step & 1) * world * B + (long long)rank * B + b;
            for (int p = 0; p < world; ++p) peer[p][slot] = tok;
            __threadfence_system();                                         // the ids are visible system-wide before the arrivals
            for (int p = 0; p < world; ++p)
                atomicAdd_system(reinterpret_cast<unsigned long long*>(peer[p] + 2ll * world * B + rank), 1ull);
        }
    }
    if (peer && b == 0 && tid < world) {                                     // all ranks' ids of this step are here before the kernel ends
        const unsigned long long want = (unsigned long long)(*step_ptr) * (unsigned long long)B;
        const volatile unsigned long long* cnt = reinterpret_cast<const volatile unsigned long long*>(peer[rank] + 2ll * world * B + tid);
        long long spins = 0;
        while (*cnt < want) {
            if (++spins > (1ll << 24)) { *err = 1; break; }                  // ~ a second: a peer is gone; report instead of hanging the GPU
            __nanosleep(64);
        }
        __threadfence_system();
    }
}

// ------------------------------------------------------------------------------------------------
// Sampling (temperature -> top-k -> top-p -> one draw), semantics in include/kivi_b200.h.  One CTA per row, no sort: both
// thresholds are selections by histogram (sample_select), exact in the order-preserving 32-bit key of the scaled logit.
// Every sum the result depends on is an integer sum -- token counts, and exp(x - max) as 40-bit fixed point in a
// uint64 -- so neither the order of the shared-memory atomics nor the row's place in the batch can change a bit of it.
// STAGED: the scaled row is kept in shared memory after the first pass; otherwise every pass re-reads it (from L2).
// ------------------------------------------------------------------------------------------------
constexpr int kSampleThreads = 1024, kSampleWarps = kSampleThreads / 32;
constexpr int kSampleBins = 2048;                                        // two bins per thread
constexpr int kSampleStageMax = 50 * 1024;                               // tokens: 200 KB of the SM's 227 KB, the rest is below
constexpr int kSampleCand = 2048;                                        // listed tokens of a selection's chosen bucket
constexpr uint32_t kSampleKeyFinite = 0x00800000u;                       // the smallest key above that of -inf
constexpr int kSampleMaxVocab = 1 << 22;                                 // 2^22 masses of at most 2^40 fit a uint64

struct SampleShared {
    unsigned long long hist[kSampleBins];
    unsigned long long warp_sum[kSampleWarps];                           // block reductions; the segment masses of the walk
    int warp_cnt[kSampleWarps];
    float warp_max[kSampleWarps], warp_xmax[kSampleWarps];
    int warp_idx[kSampleWarps];
    int cand[kSampleCand];
    int cand_n;
    unsigned long long pick_above;
    uint32_t pick_digit;
    float xmax;
    int greedy_id;
};

// x ascending <=> key ascending, for x without NaN and without -0
__device__ __forceinline__ uint32_t sample_key(float x)
{
    const uint32_t b = __float_as_uint(x);
    return b ^ ((b >> 31) ? 0xffffffffu : 0x80000000u);
}

// logit / temperature; a NaN becomes -inf (never sampled) and -0 becomes +0 (equal logits have equal keys)
__device__ __forceinline__ float sample_scaled(float logit, float temperature)
{
    const float x = logit / temperature;
    return (x != x) ? -INFINITY : (x == 0.f ? 0.f : x);
}

// exp(x - max) in units of 2^-40: at most 2^40, and 0 for x = -inf
__device__ __forceinline__ unsigned long long sample_mass(float x, float xmax)
{
    return __float2ull_rn(expf(x - xmax) * 1099511627776.f);
}

// first word of Philox4x32-10 with key (key.lo, key.hi) and counter (counter.lo, counter.hi, 0, 0)
__device__ __forceinline__ uint32_t philox4x32_10(unsigned long long key, unsigned long long counter)
{
    uint32_t c0 = (uint32_t)counter, c1 = (uint32_t)(counter >> 32), c2 = 0, c3 = 0;
    uint32_t k0 = (uint32_t)key, k1 = (uint32_t)(key >> 32);
    #pragma unroll
    for (int r = 0; r < 10; ++r) {
        const uint32_t h0 = __umulhi(0xD2511F53u, c0), l0 = 0xD2511F53u * c0;
        const uint32_t h1 = __umulhi(0xCD9E8D57u, c2), l1 = 0xCD9E8D57u * c2;
        const uint32_t n0 = h1 ^ c1 ^ k0, n2 = h0 ^ c3 ^ k1;
        c0 = n0; c1 = l1; c2 = n2; c3 = l0;
        k0 += 0x9E3779B9u; k1 += 0xBB67AE85u;
    }
    return c0;
}

// Bin of a scaled logit in the first level of a selection: linear in x, 1/64 wide, over the 32 units below the row's maximum
// (2047 = the maximum's bin, 0 = everything lower, -inf included).  Monotone in x, so it orders tokens as their keys do, and
// unlike the key's leading bits (sign, exponent) it spreads a row of logits over many bins.
__device__ __forceinline__ int sample_bucket(float x, float xmax)
{
    const float d = (xmax - x) * 64.f;
    return d < 2047.f ? 2047 - (int)d : 0;
}

// The bin d with  above + hist[d+1 ..] < target <= above + hist[d ..]  into s.pick_digit, and the weight above it into
// s.pick_above: a suffix sum over the bins, two per thread.  Called by all threads, after a barrier that follows the last add.
// The callers' targets never exceed above + the histogram's total, so exactly one thread writes the pick: it is written
// between this function's two barriers and read after the second, and nothing else ever writes it.
template <class Bin>
__device__ __forceinline__ void sample_find_bin(unsigned long long above, unsigned long long target, SampleShared& s)
{
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const Bin* hist = reinterpret_cast<const Bin*>(s.hist);
    const unsigned long long h0 = hist[2 * tid], h1 = hist[2 * tid + 1];
    unsigned long long v = h0 + h1;
    #pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
        const unsigned long long y = __shfl_down_sync(0xffffffffu, v, o);
        if (lane + o < 32) v += y;
    }
    if (lane == 0) s.warp_sum[warp] = v;
    __syncthreads();
    unsigned long long a = above + v - (h0 + h1);                        // weight above bin 2 * tid + 1
    for (int w = warp + 1; w < kSampleWarps; ++w) a += s.warp_sum[w];
    if (a < target && target <= a + h1) { s.pick_digit = 2 * tid + 1; s.pick_above = a; }
    else if (a + h1 < target && target <= a + h1 + h0) { s.pick_digit = 2 * tid; s.pick_above = a + h1; }
    __syncthreads();
}

// The largest key t for which the tokens with key >= max(t, floor) weigh at least `target`; a token weighs its mass (MASS,
// uint64 bins) or 1 (uint32 bins: native shared-memory adds).  x(i) is the scaled logit of token i.  Four levels of 2048
// bins: sample_bucket, then the 11 + 11 + 10 bits of the key among the tokens of the chosen bucket.
// Level 0 reads the row and adds with plain atomics, except into bin 0, which a cold or masked row fills: those lanes add
// once per warp.  Level 1 reads the row again and lists the chosen bucket's tokens in s.cand (in any order: every sum over
// them is an integer sum); levels 2 and 3 read that list -- a few dozen tokens -- or the row once more when the bucket
// holds more than the list does.  From level 1 on the tokens share the key's leading bits, so lanes that hit the same bin
// add once.
template <bool MASS, class X>
__device__ __noinline__ uint32_t sample_select(X x, int V, uint32_t floor, float xmax, unsigned long long target,
                                               SampleShared& s)
{
    using Bin = typename std::conditional<MASS, unsigned long long, uint32_t>::type;
    Bin* hist = reinterpret_cast<Bin*>(s.hist);
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    uint32_t prefix = 0;
    int bucket = 0;
    unsigned long long above = 0;                                        // weight of the tokens above the current bin's range
    #pragma unroll 1
    for (int level = 0; level < 4; ++level) {
        const int shift = level == 1 ? 21 : level == 2 ? 10 : 0;
        const uint32_t digits = level == 3 ? 1023u : 2047u;
        const uint32_t known = level <= 1 ? 0u : level == 2 ? 0xffe00000u : 0xfffffc00u;
        hist[2 * tid] = 0;
        hist[2 * tid + 1] = 0;
        if (level == 0 && tid == 0) s.cand_n = 0;
        const bool listed = level >= 2 && s.cand_n <= kSampleCand;       // written during level 1, two barriers ago
        const int n = listed ? s.cand_n : V;
        __syncthreads();
        for (int base = warp * 32; base < n; base += kSampleThreads) {
            const int j = base + lane;
            float xi = 0.f;
            uint32_t key = 0;
            int bk = -1, i = j;
            bool active = j < n;
            if (active) {
                if (listed) i = s.cand[j];
                xi = x(i);
                key = sample_key(xi);
                if (!listed) bk = sample_bucket(xi, xmax);
                active = (listed || (key >= floor && (level == 0 || bk == bucket))) && (key & known) == prefix;
            }
            if (level == 0) {
                Bin w = 1;
                if (MASS && active) w = sample_mass(xi, xmax);
                const uint32_t low = __ballot_sync(0xffffffffu, active && bk == 0);
                if (active && bk == 0) {
                    if (MASS) w = ((unsigned long long)__reduce_add_sync(low, (uint32_t)((unsigned long long)w >> 20)) << 20)
                                  + __reduce_add_sync(low, (uint32_t)w & 0xfffffu);
                    else w = __popc(low);
                    if (lane == __ffs(low) - 1) atomicAdd(&hist[0], w);
                } else if (active) {
                    atomicAdd(&hist[bk], w);
                }
                continue;
            }
            const uint32_t live = __ballot_sync(0xffffffffu, active);
            if (!live) continue;
            if (level == 1) {                                            // list the bucket: one counter add per warp
                int at = 0;
                if (lane == __ffs(live) - 1) at = atomicAdd(&s.cand_n, __popc(live));
                at = __shfl_sync(0xffffffffu, at, __ffs(live) - 1) + __popc(live & ((1u << lane) - 1));
                if (active && at < kSampleCand) s.cand[at] = i;
            }
            const uint32_t bin = active ? ((key >> shift) & digits) : 0xffffffffu;
            const uint32_t peers = __match_any_sync(0xffffffffu, bin);
            if (active) {
                Bin w;
                if (MASS) {
                    const unsigned long long q = sample_mass(xi, xmax);
                    w = ((unsigned long long)__reduce_add_sync(peers, (uint32_t)(q >> 20)) << 20)
                        + __reduce_add_sync(peers, (uint32_t)q & 0xfffffu);
                } else {
                    w = __popc(peers);
                }
                if (lane == __ffs(peers) - 1) atomicAdd(&hist[bin], w);
            }
        }
        __syncthreads();
        sample_find_bin<Bin>(above, target, s);
        if (level == 0) bucket = s.pick_digit;
        else prefix |= s.pick_digit << shift;
        above = s.pick_above;
    }
    return prefix;
}

// Mass and number of the tokens with key >= floor, per warp segment: warp w owns the tokens [w * seg, (w + 1) * seg).
// Returns the total mass; s.warp_sum / s.warp_cnt hold the segments'.
template <class X>
__device__ __noinline__ unsigned long long sample_segments(X x, int V, int seg, uint32_t floor, float xmax, SampleShared& s)
{
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    unsigned long long m = 0;
    int n = 0;
    const int end = min(V, (warp + 1) * seg);
    for (int i = warp * seg + lane; i < end; i += 32) {
        const float xi = x(i);
        if (sample_key(xi) >= floor) { m += sample_mass(xi, xmax); ++n; }
    }
    #pragma unroll
    for (int o = 16; o >= 1; o >>= 1) { m += __shfl_xor_sync(0xffffffffu, m, o); n += __shfl_xor_sync(0xffffffffu, n, o); }
    __syncthreads();                                                     // the previous reader of warp_sum is done
    if (lane == 0) { s.warp_sum[warp] = m; s.warp_cnt[warp] = n; }
    __syncthreads();
    unsigned long long tot = 0;
    for (int w = 0; w < kSampleWarps; ++w) tot += s.warp_sum[w];
    return tot;
}

template <bool STAGED>
__global__ void __launch_bounds__(kSampleThreads, 1)
sample_kernel(const float* __restrict__ logits, int V, const float* __restrict__ temperature, const int* __restrict__ top_k,
              const float* __restrict__ top_p, const unsigned long long* __restrict__ seed, unsigned long long* __restrict__ draw,
              long long* __restrict__ next_local, long long* __restrict__ ids_feedback, float* __restrict__ dbg_u,
              int* __restrict__ dbg_kept)
{
    extern __shared__ float sx[];                                        // STAGED: the scaled row
    __shared__ SampleShared s;
    const int b = blockIdx.x, tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const float* row = logits + (long long)b * V;
    const float T = temperature[b];
    const bool sampled = T > 0.f;

    // pass 0: the greedy id (the rule of greedy_exchange_kernel) and the maximum of the scaled row
    float best = -INFINITY, xmax = -INFINITY;
    int bi = 0x7fffffff;
    for (int i = tid; i < V; i += kSampleThreads) {
        const float v = __ldg(row + i);
        if (argmax_takes(v, i, best, bi)) { best = v; bi = i; }
        if (sampled) {
            const float xi = sample_scaled(v, T);
            if (STAGED) sx[i] = xi;
            xmax = fmaxf(xmax, xi);
        }
    }
    #pragma unroll
    for (int o = 16; o >= 1; o >>= 1) {
        const float ov = __shfl_xor_sync(0xffffffffu, best, o);
        const int oi = __shfl_xor_sync(0xffffffffu, bi, o);
        if (argmax_takes(ov, oi, best, bi)) { best = ov; bi = oi; }
        xmax = fmaxf(xmax, __shfl_xor_sync(0xffffffffu, xmax, o));
    }
    if (lane == 0) { s.warp_max[warp] = best; s.warp_idx[warp] = bi; s.warp_xmax[warp] = xmax; }
    __syncthreads();
    if (tid == 0) {
        for (int w = 1; w < kSampleWarps; ++w) {
            const float ov = s.warp_max[w];
            const int oi = s.warp_idx[w];
            if (argmax_takes(ov, oi, best, bi)) { best = ov; bi = oi; }
            xmax = fmaxf(xmax, s.warp_xmax[w]);
        }
        s.greedy_id = bi;
        s.xmax = xmax;
    }
    __syncthreads();
    xmax = s.xmax;
    if (!sampled || !(xmax > -INFINITY) || xmax == INFINITY) {           // greedy row; no finite logit; a +inf
        if (tid == 0) {
            const long long tok = s.greedy_id;
            next_local[b] = tok;
            if (ids_feedback) ids_feedback[b] = tok;
            if (dbg_u) dbg_u[b] = 0.f;
            if (dbg_kept) dbg_kept[b] = 1;
        }
        return;
    }
    auto x = [&](int i) { return STAGED ? sx[i] : sample_scaled(__ldg(row + i), T); };

    uint32_t floor = kSampleKeyFinite;                                   // kept: key >= floor
    const int k = top_k[b];
    if (k > 0 && k < V) floor = max(floor, sample_select<false>(x, V, 0u, xmax, (unsigned long long)k, s));
    const int seg = cdiv(cdiv(V, kSampleWarps), 32) * 32;
    unsigned long long S = sample_segments(x, V, seg, floor, xmax, s);
    const float p = top_p[b];
    if (!(p >= 1.f)) {
        unsigned long long target = 1;                                   // p <= 0: the maximum (mass 2^40) only
        if (p > 0.f) {
            const double t = ceil((double)p * (double)S);
            target = t >= (double)S ? S : max((unsigned long long)t, 1ull);
        }
        floor = max(floor, sample_select<true>(x, V, floor, xmax, target, s));
        S = sample_segments(x, V, seg, floor, xmax, s);
    }

    // the draw: the first kept token, in token-id order, whose cumulative mass exceeds floor(u * S)
    const unsigned long long d = draw[b];
    const unsigned long long n24 = philox4x32_10(seed[b], d) >> 8;
    const unsigned long long want = (__umul64hi(n24, S) << 40) | ((n24 * S) >> 24);
    unsigned long long run = 0;
    int ws = 0, kept = 0;
    for (int w = 0; w < kSampleWarps; ++w) kept += s.warp_cnt[w];
    while (ws < kSampleWarps - 1 && run + s.warp_sum[ws] <= want) run += s.warp_sum[ws++];
    if (warp != ws) return;
    const int end = min(V, (ws + 1) * seg);
    for (int base = ws * seg; base < end; base += 32) {
        const int i = base + lane;
        unsigned long long q = 0;
        if (i < end) {
            const float xi = x(i);
            if (sample_key(xi) >= floor) q = sample_mass(xi, xmax);
        }
        #pragma unroll
        for (int o = 1; o < 32; o <<= 1) {
            const unsigned long long y = __shfl_up_sync(0xffffffffu, q, o);
            if (lane >= o) q += y;
        }
        const uint32_t over = __ballot_sync(0xffffffffu, run + q > want);
        if (over) {
            if (lane == 0) {
                const long long tok = base + __ffs(over) - 1;
                next_local[b] = tok;
                if (ids_feedback) ids_feedback[b] = tok;
                draw[b] = d + 1;
                if (dbg_u) dbg_u[b] = (float)n24 * 5.9604644775390625e-8f;
                if (dbg_kept) dbg_kept[b] = kept;
            }
            return;
        }
        run += __shfl_sync(0xffffffffu, q, 31);
    }
}

// ------------------------------------------------------------------------------------------------
// Logits processing between lm_head and the token choice, contract in include/kivi_b200.h (kivi_logits_process_f32).
// logits_process_kernel: an element-wise pass, 4 tokens per thread (one 128-bit load of logits and of counts when the
// rows are 16-byte aligned, VEC), grid (chunks of the row, rows), so one row already fills the GPU.  The 4 tokens of a
// thread lie in one 32-bit word of the prompt bits.  A row whose penalties are neutral reads neither counts nor bits;
// a finished row reads nothing but its flag.  Every operation is an IEEE fp32 operation with round-to-nearest and no
// contraction, so a torch restatement of the same sequence gives the same bits.
// logits_record_kernel: one thread per row, after the token choice.
// ------------------------------------------------------------------------------------------------
constexpr int kProcThreads = 128, kProcMaxEos = 8;

template <bool VEC>
__global__ void __launch_bounds__(kProcThreads)
logits_process_kernel(const float* __restrict__ logits, float* __restrict__ scores, int V, const int* __restrict__ counts,
                      const uint32_t* __restrict__ seen, int words, const int* __restrict__ n_new,
                      const uint8_t* __restrict__ finished, const float* __restrict__ repetition,
                      const float* __restrict__ presence, const float* __restrict__ frequency,
                      const int* __restrict__ min_new, const long long* __restrict__ eos, int n_eos, long long pad)
{
    const int b = blockIdx.y;
    const int v0 = (blockIdx.x * kProcThreads + threadIdx.x) * 4;
    if (v0 >= V) return;
    const long long off = (long long)b * V + v0;
    float x[4];
    if (finished[b]) {                                                   // only the pad id stays finite: it is chosen
        #pragma unroll
        for (int e = 0; e < 4; ++e) x[e] = v0 + e == pad ? 0.f : -INFINITY;
    } else {
        if (VEC) {
            const float4 l = *reinterpret_cast<const float4*>(logits + off);
            x[0] = l.x; x[1] = l.y; x[2] = l.z; x[3] = l.w;
        } else {
            #pragma unroll
            for (int e = 0; e < 4; ++e) x[e] = v0 + e < V ? logits[off + e] : 0.f;
        }
        const float p = repetition[b], pr = presence[b], f = frequency[b];
        // neutral: p == 1 and both penalties +0 (a -0 frequency is not neutral: x - (-0 * 0) turns -0 into +0)
        if (p != 1.f || __float_as_uint(pr) != 0u || __float_as_uint(f) != 0u) {
            int c[4];
            if (VEC) {
                const int4 ci = *reinterpret_cast<const int4*>(counts + off);
                c[0] = ci.x; c[1] = ci.y; c[2] = ci.z; c[3] = ci.w;
            } else {
                #pragma unroll
                for (int e = 0; e < 4; ++e) c[e] = v0 + e < V ? counts[off + e] : 0;
            }
            const uint32_t bits = seen[(long long)b * words + (v0 >> 5)] >> (v0 & 31);
            #pragma unroll
            for (int e = 0; e < 4; ++e) {
                float y = x[e];
                if (((bits >> e) & 1u) || c[e] > 0) y = y < 0.f ? __fmul_rn(y, p) : __fdiv_rn(y, p);
                y = __fsub_rn(y, __fmul_rn(f, (float)c[e]));
                if (c[e] > 0) y = __fsub_rn(y, pr);
                x[e] = y;
            }
        }
        if (n_new[b] < min_new[b]) {
            for (int k = 0; k < n_eos; ++k) {
                const long long d = eos[k] - v0;
                if (d >= 0 && d < 4) x[d] = -INFINITY;
            }
        }
    }
    if (VEC) {
        *reinterpret_cast<float4*>(scores + off) = make_float4(x[0], x[1], x[2], x[3]);
    } else {
        #pragma unroll
        for (int e = 0; e < 4; ++e) if (v0 + e < V) scores[off + e] = x[e];
    }
}

__global__ void __launch_bounds__(kProcThreads)
logits_record_kernel(const long long* __restrict__ tokens, int B, int V, int* __restrict__ counts, int* __restrict__ n_new,
                     uint8_t* __restrict__ finished, const long long* __restrict__ eos, int n_eos)
{
    const int b = blockIdx.x * kProcThreads + threadIdx.x;
    if (b >= B) return;
    const long long t = tokens[b];
    if (t >= 0 && t < V) counts[(long long)b * V + t] += 1;
    n_new[b] += 1;
    bool stop = false;
    for (int k = 0; k < n_eos; ++k) stop |= eos[k] == t;
    if (stop) finished[b] = 1;
}

// ------------------------------------------------------------------------------------------------
// Tensor-parallel residual-add + RMSNorm: the all-reduce of the o_proj / down_proj partial sums fused into the norm that
// consumes them.  Every rank reads the `world` partials of this call straight from the peers' symmetric buffers (layout in
// include/kivi_b200.h), sums them in fp32 in rank order, rounds to fp16 and runs add_rmsnorm_row on that addend, the body of
// add_rmsnorm_kernel<true>: every rank gets the bits add_rmsnorm gives for the rank-order sum.
//
// A row is split over a cluster of C CTAs of 512 / C threads: CTA c of the cluster plays threads [c * 512 / C, (c+1) * 512 / C)
// of the one-CTA kernel, so C only decides how many SMs issue the N * hidden * 2 bytes of peer loads of a row.
// ------------------------------------------------------------------------------------------------
template <int C>
__global__ void __launch_bounds__(kNormThreads / C, 1)
allreduce_add_rmsnorm_kernel(const __half* const* __restrict__ peer, __half* __restrict__ residual, const __half* __restrict__ w,
                             __half* __restrict__ out, int hidden, float eps, int rank, int world, long long slot_off,
                             long long counters_off, const long long* __restrict__ epoch_ptr, int call, int* __restrict__ err)
{
    const int row = blockIdx.x / C, crank = blockIdx.x % C;
    const int vt = crank * (kNormThreads / C) + threadIdx.x;            // the thread of the one-CTA kernel this one plays
    const unsigned long long epoch = (unsigned long long)(*epoch_ptr + call + 1);
    if (blockIdx.x == 0 && threadIdx.x < world) {                        // this rank's partial of the call is written: arrive
        unsigned long long* a = reinterpret_cast<unsigned long long*>(
            reinterpret_cast<char*>(const_cast<__half*>(peer[threadIdx.x])) + counters_off) + rank;
        asm volatile("red.release.sys.global.max.u64 [%0], %1;" :: "l"(a), "l"(epoch) : "memory");
    }
    if (threadIdx.x < world) {                                           // every rank's partial of the call is written
        const unsigned long long* cnt = reinterpret_cast<const unsigned long long*>(
            reinterpret_cast<const char*>(peer[rank]) + counters_off) + threadIdx.x;
        long long spins = 0;
        unsigned long long seen;
        for (;;) {
            asm volatile("ld.acquire.sys.global.u64 %0, [%1];" : "=l"(seen) : "l"(cnt) : "memory");
            if (seen >= epoch) break;
            if (++spins > (1ll << 24)) { *err = 1; break; }              // ~ a second: a peer is gone; report instead of hanging
            __nanosleep(64);
        }
    }
    __syncthreads();                                                     // the acquires above order every thread's reads below

    const long long slice_off = slot_off / 2 + (long long)row * hidden;  // in halves, from the start of a rank's buffer
    const int64_t row_off = (int64_t)row * hidden;
    add_rmsnorm_row<C, true>([&](int i) {
        uint4 pv[8];                                                     // all peer loads in flight before the first add
        #pragma unroll
        for (int p = 0; p < 8; ++p)
            if (p < world) pv[p] = __ldcg(reinterpret_cast<const uint4*>(peer[p] + slice_off) + i);
        float2 acc[4];
        #pragma unroll
        for (int e = 0; e < 4; ++e) acc[e] = __half22float2(reinterpret_cast<const __half2*>(&pv[0])[e]);
        #pragma unroll
        for (int p = 1; p < 8; ++p) {
            if (p < world) {
                const __half2* ph = reinterpret_cast<const __half2*>(&pv[p]);
                #pragma unroll
                for (int e = 0; e < 4; ++e) { const float2 f = __half22float2(ph[e]); acc[e].x += f.x; acc[e].y += f.y; }
            }
        }
        uint4 a;
        #pragma unroll
        for (int e = 0; e < 4; ++e) reinterpret_cast<__half2*>(&a)[e] = __floats2half2_rn(acc[e].x, acc[e].y);
        return a;
    }, residual + row_off, w, out + row_off, hidden, eps, vt);
}

}  // namespace kivi

using namespace kivi;

// the checks both residual-add + RMSNorm entry points begin with
static int check_rmsnorm_args(const void* residual, const void* weight, const void* out, int rows, int hidden)
{
    if (!residual || !weight || !out) return KIVI_ERR_NULL;
    if (rows < 0 || hidden <= 0 || hidden % 8 != 0 || hidden > kNormMaxHidden) return KIVI_ERR_SHAPE;
    return KIVI_OK;
}

extern "C" int kivi_allreduce_add_rmsnorm_f16(const void* x, void* residual, const void* weight, void* out,
                                              int rows, int hidden, float eps,
                                              const void* peer_buffers, int rank, int world, int rows_max, int call,
                                              const void* epoch, void* err, int cluster, void* stream)
{
    if (int e = check_rmsnorm_args(residual, weight, out, rows, hidden)) return e;
    if (world < 1 || world > 8 || rank < 0 || rank >= world) return KIVI_ERR_SHAPE;
    if (!peer_buffers) {                                                 // one rank: x is the whole sum
        if (world != 1) return KIVI_ERR_NULL;
        return kivi_add_rmsnorm_f16(x, residual, weight, out, rows, hidden, eps, stream);
    }
    if (!epoch || !err) return KIVI_ERR_NULL;
    if (rows > rows_max || call < 0) return KIVI_ERR_SHAPE;
    if (cluster != 0 && cluster != 1 && cluster != 2 && cluster != 4 && cluster != 8) return KIVI_ERR_SHAPE;
    if (!aligned_to(residual, 16) || !aligned_to(weight, 16) || !aligned_to(out, 16) || !aligned_to(epoch, 8))
        return KIVI_ERR_ALIGN;
    if (rows == 0) return KIVI_OK;
    const long long slot_bytes = (long long)rows_max * hidden * 2;
    const long long slot_off = (long long)(call & 1) * slot_bytes, counters_off = 2 * slot_bytes;
    // cluster == 0: one CTA per row, the fastest width at every rows / hidden / world measured (tools/tp_bench.py kernel,
    // ranks emulated in one GPU's memory; over NVLink the widths have not been compared)
    const int C = cluster ? cluster : 1;
    cudaLaunchConfig_t cfg = {};
    cfg.gridDim = dim3(rows * C);
    cfg.blockDim = dim3(kNormThreads / C);
    cfg.stream = (cudaStream_t)stream;
    cudaLaunchAttribute attr[1];
    attr[0].id = cudaLaunchAttributeClusterDimension;
    attr[0].val.clusterDim.x = C;
    attr[0].val.clusterDim.y = 1;
    attr[0].val.clusterDim.z = 1;
    cfg.attrs = attr;
    cfg.numAttrs = C > 1 ? 1 : 0;
    auto kernel = C == 1 ? allreduce_add_rmsnorm_kernel<1> : C == 2 ? allreduce_add_rmsnorm_kernel<2>
                : C == 4 ? allreduce_add_rmsnorm_kernel<4> : allreduce_add_rmsnorm_kernel<8>;
    const cudaError_t e = cudaLaunchKernelEx(&cfg, kernel, (const __half* const*)peer_buffers, (__half*)residual,
                                             (const __half*)weight, (__half*)out, hidden, eps, rank, world, slot_off,
                                             counters_off, (const long long*)epoch, call, (int*)err);
    if (e != cudaSuccess) return (int)e;
    return post_launch();
}

extern "C" int kivi_greedy_sample_exchange_f32(const void* logits, int batch, int vocab, void* next_local, void* ids_feedback,
                                               const void* peer_buffers, int rank, int world, const void* step, void* err,
                                               void* stream)
{
    if (!logits || !next_local) return KIVI_ERR_NULL;
    if (batch <= 0 || vocab <= 0) return KIVI_ERR_SHAPE;
    if (peer_buffers && (!step || !err || world < 1 || rank < 0 || rank >= world || world > 256)) return KIVI_ERR_SHAPE;
    greedy_exchange_kernel<<<batch, 256, 0, (cudaStream_t)stream>>>(
        (const float*)logits, vocab, (long long*)next_local, (long long*)ids_feedback, (long long* const*)peer_buffers,
        batch, rank, world, (const int*)step, (int*)err);
    return post_launch();
}

extern "C" int kivi_sample_f32(const void* logits, int batch, int vocab, const float* temperature, const int32_t* top_k,
                               const float* top_p, const uint64_t* seed, uint64_t* draw, void* next_local, void* ids_feedback,
                               float* dbg_u, int32_t* dbg_kept, void* stream)
{
    if (!logits || !temperature || !top_k || !top_p || !seed || !draw || !next_local) return KIVI_ERR_NULL;
    if (batch < 0 || vocab < 1 || vocab > kSampleMaxVocab) return KIVI_ERR_SHAPE;
    if (batch == 0) return KIVI_OK;
    DeviceInfo info;
    if (int e = device_info(&info)) return e;
    // a row that fits beside the histogram is staged in shared memory (Llama-2's 32000 tokens); a longer one (Llama-3's
    // 128256) is re-read from L2 by every pass
    const int row_bytes = vocab * (int)sizeof(float);
    const bool staged = vocab <= kSampleStageMax && row_bytes + (int)sizeof(SampleShared) <= info.max_smem_optin;
    if (staged) {
        static std::atomic<unsigned long long> done{0};
        if (int e = ensure_dynamic_smem(sample_kernel<true>, kSampleStageMax * (int)sizeof(float), info.ordinal, done)) return e;
    }
    auto kernel = staged ? sample_kernel<true> : sample_kernel<false>;
    kernel<<<batch, kSampleThreads, staged ? row_bytes : 0, (cudaStream_t)stream>>>(
        (const float*)logits, vocab, temperature, top_k, top_p, (const unsigned long long*)seed, (unsigned long long*)draw,
        (long long*)next_local, (long long*)ids_feedback, dbg_u, dbg_kept);
    return post_launch();
}

extern "C" int kivi_logits_process_f32(const void* logits, void* scores, int batch, int vocab, const int32_t* counts,
                                       const uint32_t* seen, const int32_t* n_new, const uint8_t* finished,
                                       const float* repetition, const float* presence, const float* frequency,
                                       const int32_t* min_new, const int64_t* eos_ids, int n_eos, int64_t pad_id,
                                       void* stream)
{
    if (!logits || !scores || !counts || !seen || !n_new || !finished || !repetition || !presence || !frequency || !min_new)
        return KIVI_ERR_NULL;
    if (n_eos > 0 && !eos_ids) return KIVI_ERR_NULL;
    if (batch < 0 || batch > 65535 || vocab < 1 || n_eos < 0 || n_eos > kProcMaxEos || pad_id < 0 || pad_id >= vocab)
        return KIVI_ERR_SHAPE;
    if (!aligned_to(seen, 4)) return KIVI_ERR_ALIGN;
    if (batch == 0) return KIVI_OK;
    // 128-bit accesses when every row starts on a 16-byte boundary
    const bool vec = vocab % 4 == 0 && aligned_to(logits, 16) && aligned_to(scores, 16) && aligned_to(counts, 16);
    const dim3 grid(cdiv(cdiv(vocab, 4), kProcThreads), batch);
    auto kernel = vec ? logits_process_kernel<true> : logits_process_kernel<false>;
    kernel<<<grid, kProcThreads, 0, (cudaStream_t)stream>>>(
        (const float*)logits, (float*)scores, vocab, counts, seen, cdiv(vocab, 32), n_new, finished, repetition, presence,
        frequency, min_new, (const long long*)eos_ids, n_eos, (long long)pad_id);
    return post_launch();
}

extern "C" int kivi_logits_record(const void* tokens, int batch, int vocab, int32_t* counts, int32_t* n_new,
                                  uint8_t* finished, const int64_t* eos_ids, int n_eos, void* stream)
{
    if (!tokens || !counts || !n_new || !finished) return KIVI_ERR_NULL;
    if (n_eos > 0 && !eos_ids) return KIVI_ERR_NULL;
    if (batch < 0 || vocab < 1 || n_eos < 0 || n_eos > kProcMaxEos) return KIVI_ERR_SHAPE;
    if (batch == 0) return KIVI_OK;
    logits_record_kernel<<<cdiv(batch, kProcThreads), kProcThreads, 0, (cudaStream_t)stream>>>(
        (const long long*)tokens, batch, vocab, counts, n_new, finished, (const long long*)eos_ids, n_eos);
    return post_launch();
}

extern "C" int kivi_add_rmsnorm_f16(const void* x, void* residual, const void* weight, void* out,
                                    int rows, int hidden, float eps, void* stream)
{
    if (int e = check_rmsnorm_args(residual, weight, out, rows, hidden)) return e;
    // the kernel moves 8 halves per uint4 access: a view that starts off a 16-byte boundary would fault
    if ((x && !aligned_to(x, 16)) || !aligned_to(residual, 16) || !aligned_to(weight, 16) || !aligned_to(out, 16))
        return KIVI_ERR_ALIGN;
    if (rows == 0) return KIVI_OK;
    cudaStream_t st = (cudaStream_t)stream;
    if (x) add_rmsnorm_kernel<true><<<rows, 512, 0, st>>>((const __half*)x, (__half*)residual,
                                                                            (const __half*)weight, (__half*)out, hidden, eps);
    else   add_rmsnorm_kernel<false><<<rows, 512, 0, st>>>(nullptr, (__half*)residual,
                                                                             (const __half*)weight, (__half*)out, hidden, eps);
    return post_launch();
}

extern "C" int kivi_rope_split_f16(const void* qkv, const void* cos_table, const void* sin_table, const void* pos,
                                   void* q, void* k, void* v, int batch, int num_heads, int num_kv_heads, int table_rows,
                                   void* stream)
{
    if (!qkv || !cos_table || !sin_table || !pos || !q || !k || !v) return KIVI_ERR_NULL;
    if (batch <= 0 || num_heads <= 0 || num_kv_heads <= 0 || batch > 65535 || table_rows <= 0) return KIVI_ERR_SHAPE;
    rope_split_kernel<<<dim3(num_heads + 2 * num_kv_heads, batch), 64, 0, (cudaStream_t)stream>>>(
        (const __half*)qkv, (const __half*)cos_table, (const __half*)sin_table, (const long long*)pos,
        (__half*)q, (__half*)k, (__half*)v, num_heads, num_kv_heads, table_rows);
    return post_launch();
}

extern "C" int kivi_silu_mul_f16(const void* gate_up, void* out, int rows, int intermediate, void* stream)
{
    if (!gate_up || !out) return KIVI_ERR_NULL;
    if (rows <= 0 || intermediate <= 0 || intermediate % 2 != 0 || rows > 65535) return KIVI_ERR_SHAPE;
    if (!aligned_to(gate_up, 4) || !aligned_to(out, 4)) return KIVI_ERR_ALIGN;      // half2 accesses
    silu_mul_kernel<<<dim3(cdiv(intermediate / 2, 256), rows), 256, 0, (cudaStream_t)stream>>>(
        (const __half*)gate_up, (__half*)out, intermediate);
    return post_launch();
}
