// kivi_lora.cu -- LoRA deltas of the decode step's projection groups, one adapter per batch row (sm_90a).  Contract in
// include/kivi_b200.h (kivi_lora_shrink_f16 / kivi_lora_expand_f16).
//
// Both kernels give every CTA one adapter slot s (blockIdx.y) and one slice of the weights; the CTA gathers the rows whose
// idx is s into shared memory and exits when there are none.  So each present adapter's A and B are read once per call,
// whatever the number of its rows, and an absent slot costs one scan of idx.
//   shrink: CTA (K chunk, A-row group, s): the K chunk's partial of t[b, e] = sum_k x[b, k] A[s, e, k] for its 16 A rows
//           e = g * R + j and every row b of s, into ws[chunk, b, e].  The CTA holds its A slice in registers and streams the
//           rows' x chunks through shared memory.
//   expand: CTA (column tile, s): t[b, e] = the chunks' partials summed in chunk order, then
//           y[b, o] = fp16(float(y[b, o]) + scale[s] * sum_j B[s, o, j] t[b, seg(o) R + j]) for the tile's columns.
// Every sum runs in an order fixed by the shapes alone (lane order, then the warp's xor tree, then chunk order; j ascending),
// so a row's result depends on that row's x, y and adapter only.  No float atomics.
#include "kivi_common.cuh"

namespace kivi {

constexpr int kLoraThreads = 256;
constexpr int kLoraChunk = 512;            // K elements per shrink CTA: 2 uint4 per lane
constexpr int kLoraRowsPerWarp = 2;        // A rows per warp
constexpr int kLoraARows = kLoraRowsPerWarp * (kLoraThreads / 32);      // 16 A rows per shrink CTA
constexpr int kLoraXTile = 16;             // rows of x staged at a time (16 KB)
constexpr int kLoraMaxRows = 1024;
constexpr int kLoraMaxRank = 128;
constexpr int kLoraCols = 128;             // columns per expand CTA
constexpr int kLoraT = 2048;               // fp32 t values staged per expand tile

struct LoraSegs { int off[4]; int n; };

// rows b with idx[b] == s, into list (any order: a row's result does not depend on its place); returns their number
__device__ __forceinline__ int lora_rows(const int* __restrict__ idx, int rows, int s, int* list, int* count)
{
    if (threadIdx.x == 0) *count = 0;
    __syncthreads();
    for (int b = threadIdx.x; b < rows; b += kLoraThreads)
        if (idx[b] == s) list[atomicAdd(count, 1)] = b;
    __syncthreads();
    return *count;
}

__global__ void __launch_bounds__(kLoraThreads, 1)
lora_shrink_kernel(const __half* __restrict__ x, int rows, int in, const __half* __restrict__ A, int NR,
                   const int* __restrict__ idx, float* __restrict__ ws, int groups)
{
    __shared__ int list[kLoraMaxRows];
    __shared__ int count;
    __shared__ __align__(16) __half xs[kLoraXTile][kLoraChunk];
    const int s = blockIdx.y, chunk = blockIdx.x / groups, group = blockIdx.x % groups;
    const int n = lora_rows(idx, rows, s, list, &count);
    if (n == 0) return;
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int k0 = chunk * kLoraChunk;

    float a[kLoraRowsPerWarp][16];
    #pragma unroll
    for (int i = 0; i < kLoraRowsPerWarp; ++i) {
        const int e = group * kLoraARows + warp + 8 * i;
        #pragma unroll
        for (int v = 0; v < 2; ++v) {
            const int k = k0 + v * 256 + lane * 8;
            uint4 u = make_uint4(0, 0, 0, 0);
            if (e < NR && k < in) u = __ldg(reinterpret_cast<const uint4*>(A + ((int64_t)s * NR + e) * in + k));
            const __half2* h = reinterpret_cast<const __half2*>(&u);
            #pragma unroll
            for (int q = 0; q < 4; ++q) {
                const float2 f = __half22float2(h[q]);
                a[i][v * 8 + 2 * q] = f.x;
                a[i][v * 8 + 2 * q + 1] = f.y;
            }
        }
    }

    for (int r0 = 0; r0 < n; r0 += kLoraXTile) {
        const int nr = min(kLoraXTile, n - r0);
        __syncthreads();                                                  // the previous tile is consumed
        for (int i = threadIdx.x; i < nr * (kLoraChunk / 8); i += kLoraThreads) {
            const int rr = i / (kLoraChunk / 8), kk = (i % (kLoraChunk / 8)) * 8;
            uint4 u = make_uint4(0, 0, 0, 0);
            if (k0 + kk < in) u = __ldg(reinterpret_cast<const uint4*>(x + (int64_t)list[r0 + rr] * in + k0 + kk));
            *reinterpret_cast<uint4*>(&xs[rr][kk]) = u;
        }
        __syncthreads();
        for (int rr = 0; rr < nr; ++rr) {
            float xf[16];
            #pragma unroll
            for (int v = 0; v < 2; ++v) {
                const uint4 u = *reinterpret_cast<const uint4*>(&xs[rr][v * 256 + lane * 8]);
                const __half2* h = reinterpret_cast<const __half2*>(&u);
                #pragma unroll
                for (int q = 0; q < 4; ++q) {
                    const float2 f = __half22float2(h[q]);
                    xf[v * 8 + 2 * q] = f.x;
                    xf[v * 8 + 2 * q + 1] = f.y;
                }
            }
            const int64_t row = list[r0 + rr];
            #pragma unroll
            for (int i = 0; i < kLoraRowsPerWarp; ++i) {
                const int e = group * kLoraARows + warp + 8 * i;
                if (e >= NR) continue;                                    // uniform over the warp
                float acc = 0.f;
                #pragma unroll
                for (int q = 0; q < 16; ++q) acc = fmaf(a[i][q], xf[q], acc);
                acc = warp_sum(acc);
                if (lane == 0) ws[((int64_t)chunk * rows + row) * NR + e] = acc;
            }
        }
    }
}

__global__ void __launch_bounds__(kLoraThreads)
lora_expand_kernel(const float* __restrict__ ws, int rows, int chunks, int NR, int R, const __half* __restrict__ B,
                   const float* __restrict__ scale, const int* __restrict__ idx, __half* __restrict__ y, int out,
                   LoraSegs segs)
{
    __shared__ int list[kLoraMaxRows];
    __shared__ int count;
    __shared__ __align__(16) __half Bs[kLoraMaxRank][kLoraCols];          // B tile transposed: Bs[j][c]
    __shared__ float ts[kLoraT];
    const int s = blockIdx.y, c0 = blockIdx.x * kLoraCols;
    const int n = lora_rows(idx, rows, s, list, &count);
    if (n == 0) return;
    const int cols = min(kLoraCols, out - c0);
    auto seg_of = [&](int o) { int g = 0; while (g + 1 < segs.n && o >= segs.off[g + 1]) ++g; return g; };
    const int g_lo = seg_of(c0), g_hi = seg_of(c0 + cols - 1);
    const int e_lo = g_lo * R, n_e = (g_hi - g_lo + 1) * R;              // the t entries this tile's columns read

    const int vecs = R / 8;
    for (int i = threadIdx.x; i < cols * vecs; i += kLoraThreads) {
        const int c = i / vecs, j = (i % vecs) * 8;
        const uint4 u = __ldg(reinterpret_cast<const uint4*>(B + ((int64_t)s * out + c0 + c) * R + j));
        const __half* h = reinterpret_cast<const __half*>(&u);
        #pragma unroll
        for (int q = 0; q < 8; ++q) Bs[j + q][c] = h[q];
    }
    const int c = threadIdx.x % kLoraCols, slot = threadIdx.x / kLoraCols;
    const int o = c0 + c;
    const int eoff = o < out ? seg_of(o) * R - e_lo : 0;
    const float sc = scale[s];
    const int tile = kLoraT / n_e;                                        // rows whose t fits in ts
    const int64_t chunk_stride = (int64_t)rows * NR;

    for (int r0 = 0; r0 < n; r0 += tile) {
        const int nr = min(tile, n - r0);
        __syncthreads();                                                  // Bs is staged / the previous tile is consumed
        for (int i = threadIdx.x; i < nr * n_e; i += kLoraThreads) {
            const int rr = i / n_e, e = i % n_e;
            const float* p = ws + (int64_t)list[r0 + rr] * NR + e_lo + e;
            float acc = p[0];
            for (int k = 1; k < chunks; ++k) acc += p[k * chunk_stride];
            ts[rr * n_e + e] = acc;
        }
        __syncthreads();
        if (o >= out) continue;
        for (int rr = slot; rr < nr; rr += kLoraThreads / kLoraCols) {
            const float* t = ts + rr * n_e + eoff;
            float acc = 0.f;
            for (int j = 0; j < R; ++j) acc = fmaf(__half2float(Bs[j][c]), t[j], acc);
            const float d = sc * acc;
            if (d != 0.f) {                                               // a zero delta leaves y's bits (-0 included)
                __half* py = y + (int64_t)list[r0 + rr] * out + o;
                *py = __float2half_rn(__half2float(*py) + d);
            }
        }
    }
}

}  // namespace kivi

using namespace kivi;

// the checks both entries share: shapes of x / t, the stack and the row indices
static int check_lora_args(int rows, int in, int S, int n_seg, int rank)
{
    if (rows < 0 || rows > kLoraMaxRows || in < 8 || in % 8 != 0 || S < 1 || S > 65535 || n_seg < 1 || n_seg > 3 ||
        rank < 8 || rank > kLoraMaxRank || rank % 8 != 0)
        return KIVI_ERR_SHAPE;
    return KIVI_OK;
}

extern "C" int64_t kivi_lora_workspace_bytes(int rows, int in, int n_seg, int rank)
{
    const int e = check_lora_args(rows, in, 1, n_seg, rank);
    if (e != KIVI_OK) return e;
    return (int64_t)cdiv(in, kLoraChunk) * rows * n_seg * rank * (int64_t)sizeof(float);
}

extern "C" int kivi_lora_shrink_f16(const void* x, int rows, int in, const void* A, int S, int n_seg, int rank,
                                    const int32_t* idx, float* ws, void* stream)
{
    if (!x || !A || !idx || !ws) return KIVI_ERR_NULL;
    const int e = check_lora_args(rows, in, S, n_seg, rank);
    if (e != KIVI_OK) return e;
    if (!aligned_to(x, 16) || !aligned_to(A, 16) || !aligned_to(ws, 4) || !aligned_to(idx, 4)) return KIVI_ERR_ALIGN;
    if (rows == 0) return KIVI_OK;
    const int NR = n_seg * rank, groups = cdiv(NR, kLoraARows);
    lora_shrink_kernel<<<dim3(cdiv(in, kLoraChunk) * groups, S), kLoraThreads, 0, (cudaStream_t)stream>>>(
        (const __half*)x, rows, in, (const __half*)A, NR, (const int*)idx, ws, groups);
    return post_launch();
}

extern "C" int kivi_lora_expand_f16(const float* ws, int rows, int in, const void* B, const float* scale, int S, int n_seg,
                                    int rank, const int* seg_off, const int32_t* idx, void* y, int out_total, void* stream)
{
    if (!ws || !B || !scale || !seg_off || !idx || !y) return KIVI_ERR_NULL;
    const int e = check_lora_args(rows, in, S, n_seg, rank);
    if (e != KIVI_OK) return e;
    if (out_total < 1 || out_total > 65535 * kLoraCols || seg_off[0] != 0 || seg_off[n_seg] != out_total)
        return KIVI_ERR_SHAPE;
    LoraSegs segs{{0, 0, 0, 0}, n_seg};
    for (int g = 0; g <= n_seg; ++g) {
        if (g > 0 && seg_off[g] <= seg_off[g - 1]) return KIVI_ERR_SHAPE;
        segs.off[g] = seg_off[g];
    }
    if (!aligned_to(B, 16) || !aligned_to(ws, 4) || !aligned_to(scale, 4) || !aligned_to(idx, 4) || !aligned_to(y, 2))
        return KIVI_ERR_ALIGN;
    if (rows == 0) return KIVI_OK;
    lora_expand_kernel<<<dim3(cdiv(out_total, kLoraCols), S), kLoraThreads, 0, (cudaStream_t)stream>>>(
        ws, rows, cdiv(in, kLoraChunk), n_seg * rank, rank, (const __half*)B, scale, (const int*)idx, (__half*)y, out_total,
        segs);
    return post_launch();
}
