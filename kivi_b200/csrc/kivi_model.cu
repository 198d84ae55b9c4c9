// kivi_model.cu -- small fused glue kernels of the decode step around the hot path (sm_90a):
// residual-add + RMSNorm, RoPE + q/k/v split, SiLU*mul.  They replace ~16 ATen elementwise launches per
// layer per step with 4; arithmetic follows the HF Llama modules the reference forks
// (models/llama_kivi.py star-imports transformers.models.llama): every fp16 op rounds to fp16.
#include "kivi_common.cuh"

#include <cooperative_groups.h>

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

static bool aligned_to(const void* p, uintptr_t bytes) { return reinterpret_cast<uintptr_t>(p) % bytes == 0; }

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
