// k4_distloss.cu -- the distortion loss of the LLFF and unbounded configs (weight_distortion > 0):
// torch_efficient_distloss.flatten_eff_distloss (run_sr.py:16, :536-542, :977-989) and its gradient, and
// ub360_utils_cuda.segment_cumsum, the op behind the reference's DistortionLoss (lib/dcvgo.py:385-409).
//
// Input: a flat sample list w [M], m [M] (fp32) and ray_id [M] (int64, non-decreasing); a segment is a maximal
// run of equal ray_id.  Per sample the exclusive in-segment prefixes W<i = sum_{j<i} w_j, WM<i = sum_{j<i} w_j m_j
// and the suffixes W>i, WM>i give
//     L       = ( sum_i 2 w_i (m_i W<i - WM<i) + interval/3 sum_i w_i^2 ) / n,          n = max(ray_id) + 1
//     dL/dw_i = g/n ( 2 m_i (W<i - W>i) + 2 (WM>i - WM<i) + 2/3 interval w_i ).
//
// A chunk scan plus a carry pass, so that every sum has a fixed order (a decoupled look-back would sum the
// predecessors' aggregates in whatever order they happen to be published, and the bits would change run to run):
//   dl_tile_kernel    one pass over the samples, one CTA per tile of DL_TILE samples: the tile's segmented-scan
//                     aggregates (its first and last segment's sums, whether it holds a head), the loss terms with
//                     the prefixes restarted at the tile start, and the tile's largest ray id.
//   dl_carry_kernel   one CTA over the tiles: the prefix carried into each tile from the left and the suffix carried
//                     in from the right (segmented scans of the tile aggregates), the loss (tile terms plus each
//                     tile's carry correction 2 (W_in sum_first w m - WM_in sum_first w), summed in fp64), n.
//   dl_apply_kernel   one pass over the samples: prefixes (segment_cumsum) or prefixes and suffixes (the gradient)
//                     of every sample from the tile scan and the carries.
// The forward is tile + carry; the backward is apply alone, reading the carries the forward left in the workspace
// (48 B per 2048 samples) instead of prefixes saved per sample: 16 B/sample read + 4 B written, no extra 8 B/sample
// write in the forward and read in the backward.  Nothing synchronises the host: n stays on the device.
#include <climits>
#include "k4_internal.cuh"

namespace {

constexpr int DL_T = 256;                       // threads of a tile CTA
constexpr int DL_IPT = 8;                       // samples per thread
constexpr int DL_TILE = DL_T * DL_IPT;
constexpr int DL_SK = DL_TILE + DL_TILE / 32;   // skewed shared arrays: blocked reads t * 8 + k hit 32 banks
constexpr int DL_CT = 1024;                     // threads of the carry CTA
constexpr unsigned FULL = 0xffffffffu;

struct DlTile {
    float t_w, t_wm;        // the tile's last segment: from its last head at position >= 1 (else the start) to its end
    float s_w, s_wm;        // the tile's first segment: from its start to its first tail at position <= DL_TILE - 2
    float loss;             // sum of the per-sample terms with the prefixes restarted at the tile start
    uint32_t flags;         // bit 0: the tile's first sample is a head; bit 1: a head at a position >= 1
    long long rid_max;
};
struct DlCarry { float in_w, in_wm, out_w, out_wm; };
struct DlHeader { long long n, reserved; };
static_assert(sizeof(DlTile) == 32 && sizeof(DlCarry) == 16 && sizeof(DlHeader) == 16, "workspace layout");

inline long long dl_tiles(long long M) { return (M + DL_TILE - 1) / DL_TILE; }

struct DlWs {
    DlHeader* hdr; DlTile* tiles; DlCarry* car;
    DlWs(void* ws, long long nt) {
        hdr = (DlHeader*)ws;
        tiles = (DlTile*)(hdr + 1);
        car = (DlCarry*)(tiles + nt);
    }
};

struct DlIn { const float* w; const float* m; const long long* rid; long long M; };

// a segmented-scan element: sums since the last head (f: a head was seen)
struct Seg { float w, wm; int f; };

__device__ __forceinline__ Seg seg_cat(Seg a, Seg b) {      // a precedes b
    if (!b.f) { b.w = a.w + b.w; b.wm = a.wm + b.wm; }
    b.f |= a.f;
    return b;
}

// Exclusive segmented scan over the CTA in thread order; *total receives the whole CTA's element.  sh holds
// NT / 32 + 1 elements.  Warp shuffles, then one thread over the warp totals: a fixed order.
template <int NT>
__device__ __forceinline__ Seg block_excl_scan(Seg v, Seg* sh, Seg* total) {
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    Seg inc = v;
#pragma unroll
    for (int d = 1; d < 32; d <<= 1) {
        Seg p;
        p.w = __shfl_up_sync(FULL, inc.w, d);
        p.wm = __shfl_up_sync(FULL, inc.wm, d);
        p.f = __shfl_up_sync(FULL, inc.f, d);
        if (lane >= d) inc = seg_cat(p, inc);
    }
    Seg ex;
    ex.w = __shfl_up_sync(FULL, inc.w, 1);
    ex.wm = __shfl_up_sync(FULL, inc.wm, 1);
    ex.f = __shfl_up_sync(FULL, inc.f, 1);
    if (lane == 0) ex = Seg{0.f, 0.f, 0};
    if (lane == 31) sh[warp] = inc;
    __syncthreads();
    if (threadIdx.x == 0) {
        Seg run{0.f, 0.f, 0};
        for (int i = 0; i < NT / 32; ++i) {
            const Seg t = sh[i];
            sh[i] = run;
            run = seg_cat(run, t);
        }
        sh[NT / 32] = run;
    }
    __syncthreads();
    ex = seg_cat(sh[warp], ex);
    *total = sh[NT / 32];
    __syncthreads();
    return ex;
}

// CTA sum / max in a fixed order (warp tree, then one thread over the warps); sh holds NT / 32 elements.
template <int NT, typename T, typename Op>
__device__ __forceinline__ T block_reduce(T v, T* sh, Op op) {
#pragma unroll
    for (int d = 16; d >= 1; d >>= 1) v = op(v, __shfl_down_sync(FULL, v, d));
    if ((threadIdx.x & 31) == 0) sh[threadIdx.x >> 5] = v;
    __syncthreads();
    if (threadIdx.x == 0)
        for (int i = 1; i < NT / 32; ++i) v = op(v, sh[i]);
    __syncthreads();
    return v;                                   // valid in thread 0
}

__device__ __forceinline__ int sk(int p) { return p + (p >> 5); }

// Coalesced loads of a tile into the skewed shared arrays; flags bit 0 = head (first sample of its segment),
// bit 1 = tail (last sample).  Past M: w = m = 0, a one-sample segment of its own.
__device__ __forceinline__ long long load_tile(const DlIn& in, long long base, float* sw, float* swm, float* sm, uint8_t* sfl) {
    long long rmax = LLONG_MIN;
#pragma unroll
    for (int k = 0; k < DL_IPT; ++k) {
        const int p = k * DL_T + threadIdx.x;
        const long long i = base + p;
        float w = 0.f, m = 0.f;
        uint8_t fl = 3;
        if (i < in.M) {
            w = __ldg(in.w + i);
            m = __ldg(in.m + i);
            const long long r = __ldg(in.rid + i);
            fl = (uint8_t)((i == 0 || __ldg(in.rid + i - 1) != r) | ((i == in.M - 1 || __ldg(in.rid + i + 1) != r) << 1));
            rmax = max(rmax, r);
        }
        sw[sk(p)] = w;
        swm[sk(p)] = __fmul_rn(w, m);
        sm[sk(p)] = m;
        sfl[p] = fl;
    }
    __syncthreads();
    return rmax;
}

// The thread's aggregate over its blocked samples j = t * DL_IPT + k, heads at tile position 0 ignored (the carry
// into the tile is 0 there), then the CTA scan: the prefix at the thread's first sample.
__device__ __forceinline__ Seg fwd_scan(const float* sw, const float* swm, const uint8_t* sfl, Seg* sh, Seg* total) {
    Seg agg{0.f, 0.f, 0};
#pragma unroll
    for (int k = 0; k < DL_IPT; ++k) {
        const int j = threadIdx.x * DL_IPT + k;
        const Seg e{sw[sk(j)], swm[sk(j)], (j != 0) && (sfl[j] & 1)};
        agg = seg_cat(agg, e);
    }
    return block_excl_scan<DL_T>(agg, sh, total);
}

__device__ __forceinline__ float dl_interval(float h, const float* d) { return d ? __ldg(d) : h; }

__global__ void __launch_bounds__(DL_T) dl_tile_kernel(const DlIn in, float interval, const float* __restrict__ d_interval,
                                                       DlTile* __restrict__ tiles) {
    __shared__ float sw[DL_SK], swm[DL_SK], sm[DL_SK];
    __shared__ uint8_t sfl[DL_TILE];
    __shared__ Seg sh[DL_T / 32 + 1];
    __shared__ float shf[DL_T / 32];
    __shared__ long long shl[DL_T / 32];
    const long long base = (long long)blockIdx.x * DL_TILE;
    const long long rmax_t = load_tile(in, base, sw, swm, sm, sfl);
    const float c3 = __fdiv_rn(dl_interval(interval, d_interval), 3.f);
    Seg total;
    const Seg ex = fwd_scan(sw, swm, sfl, sh, &total);
    float pw = ex.w, pwm = ex.wm, loss = 0.f, s_w = 0.f, s_wm = 0.f;
    bool first = !ex.f;                          // no head at a position >= 1 before this sample
#pragma unroll
    for (int k = 0; k < DL_IPT; ++k) {
        const int j = threadIdx.x * DL_IPT + k;
        const float w = sw[sk(j)], wm = swm[sk(j)], m = sm[sk(j)];
        if (j != 0 && (sfl[j] & 1)) { pw = 0.f; pwm = 0.f; first = false; }
        loss += 2.f * w * (m * pw - pwm) + c3 * w * w;
        if (first) { s_w += w; s_wm += wm; }
        pw += w;
        pwm += wm;
    }
    const auto add = [](float a, float b) { return a + b; };
    loss = block_reduce<DL_T>(loss, shf, add);
    s_w = block_reduce<DL_T>(s_w, shf, add);
    s_wm = block_reduce<DL_T>(s_wm, shf, add);
    const long long rmax = block_reduce<DL_T>(rmax_t, shl, [](long long a, long long b) { return a > b ? a : b; });
    if (threadIdx.x == 0)
        tiles[blockIdx.x] = DlTile{total.w, total.wm, s_w, s_wm, loss, (uint32_t)((sfl[0] & 1) | (total.f << 1)), rmax};
}

// a tile's first segment ends inside it: a head at a position >= 1, or its last sample is a tail (tile k + 1 starts
// with a head, or k is the last tile)
__device__ __forceinline__ bool tile_ends(const DlTile* tiles, long long nt, long long k) {
    return (tiles[k].flags & 2) || k == nt - 1 || (tiles[k + 1].flags & 1);
}

// One CTA.  Thread t owns a contiguous chunk of tiles; forward carries in tile order, backward carries in reverse
// tile order, each a per-thread pass, a CTA scan and a second per-thread pass.
__global__ void __launch_bounds__(DL_CT, 1) dl_carry_kernel(const DlTile* __restrict__ tiles, DlCarry* __restrict__ car, long long nt,
                                                         DlHeader* __restrict__ hdr, float* __restrict__ d_loss) {
    __shared__ Seg sh[DL_CT / 32 + 1];
    __shared__ double shd[DL_CT / 32];
    __shared__ long long shl[DL_CT / 32];
    const long long chunk = (nt + DL_CT - 1) / DL_CT;
    const long long lo = min(nt, (long long)threadIdx.x * chunk), hi = min(nt, lo + chunk);
    Seg total;
    // ---- from the left: the open segment's sums entering tile k (0 when tile k starts with a head)
    Seg agg{0.f, 0.f, 0};
    for (long long k = lo; k < hi; ++k) agg = seg_cat(agg, Seg{tiles[k].t_w, tiles[k].t_wm, tiles[k].flags != 0});
    Seg run = block_excl_scan<DL_CT>(agg, sh, &total);
    double loss = 0.0;
    long long rmax = LLONG_MIN;
    for (long long k = lo; k < hi; ++k) {
        const DlTile t = tiles[k];
        const bool head = t.flags & 1;
        const float in_w = head ? 0.f : run.w, in_wm = head ? 0.f : run.wm;
        car[k].in_w = in_w;
        car[k].in_wm = in_wm;
        loss += (double)t.loss + 2.0 * ((double)in_w * t.s_wm - (double)in_wm * t.s_w);
        rmax = max(rmax, t.rid_max);
        run = seg_cat(run, Seg{t.t_w, t.t_wm, t.flags != 0});
    }
    // ---- from the right, reversed index r <-> tile nt - 1 - r: the sums of the segment open at tile k's end over
    // the later tiles (0 when tile k ends with a tail)
    agg = Seg{0.f, 0.f, 0};
    for (long long r = lo; r < hi; ++r) {
        const long long k = nt - 1 - r;
        agg = seg_cat(agg, Seg{tiles[k].s_w, tiles[k].s_wm, tile_ends(tiles, nt, k)});
    }
    run = block_excl_scan<DL_CT>(agg, sh, &total);
    for (long long r = lo; r < hi; ++r) {
        const long long k = nt - 1 - r;
        const bool last_is_tail = k == nt - 1 || (tiles[k + 1].flags & 1);
        car[k].out_w = last_is_tail ? 0.f : run.w;
        car[k].out_wm = last_is_tail ? 0.f : run.wm;
        run = seg_cat(run, Seg{tiles[k].s_w, tiles[k].s_wm, tile_ends(tiles, nt, k)});
    }
    loss = block_reduce<DL_CT>(loss, shd, [](double a, double b) { return a + b; });
    rmax = block_reduce<DL_CT>(rmax, shl, [](long long a, long long b) { return a > b ? a : b; });
    if (threadIdx.x == 0) {
        hdr->n = rmax + 1;
        if (d_loss) *d_loss = (float)(loss / (double)(rmax + 1));
    }
}

// GRAD: out0 = dL/dw (coef = g / n, or g when !mean); else segment_cumsum: out0 = w prefix, out1 = w totals [n_rays],
// out2 = w*s prefix, out3 = w*s totals (the totals pre-zeroed, written at each segment's last sample).
template <bool GRAD>
__global__ void __launch_bounds__(DL_T) dl_apply_kernel(const DlIn in, const DlCarry* __restrict__ car, const DlHeader* __restrict__ hdr,
                                                        float interval, const float* __restrict__ d_interval,
                                                        const float* __restrict__ d_g, int mean, long long n_rays,
                                                        float* __restrict__ out0, float* __restrict__ out1,
                                                        float* __restrict__ out2, float* __restrict__ out3) {
    __shared__ float sw[DL_SK], swm[DL_SK], sm[DL_SK], spw[DL_SK], spwm[DL_SK];
    __shared__ uint8_t sfl[DL_TILE];
    __shared__ Seg sh[DL_T / 32 + 1];
    const long long base = (long long)blockIdx.x * DL_TILE;
    load_tile(in, base, sw, swm, sm, sfl);
    const DlCarry c = car[blockIdx.x];
    Seg total;
    Seg ex = fwd_scan(sw, swm, sfl, sh, &total);
    float pw = ex.f ? ex.w : c.in_w + ex.w, pwm = ex.f ? ex.wm : c.in_wm + ex.wm;
#pragma unroll
    for (int k = 0; k < DL_IPT; ++k) {
        const int j = threadIdx.x * DL_IPT + k;
        const float w = sw[sk(j)], wm = swm[sk(j)];
        if (j != 0 && (sfl[j] & 1)) { pw = 0.f; pwm = 0.f; }
        spw[sk(j)] = pw;                         // the thread's own samples: no other thread reads them before the sync
        spwm[sk(j)] = pwm;
        pw += w;
        pwm += wm;
        if (!GRAD && (sfl[j] & 2) && base + j < in.M) {
            const long long r = __ldg(in.rid + base + j);
            if (r >= 0 && r < n_rays) { out1[r] = pw; out3[r] = pwm; }
        }
    }
    if (GRAD) {
        __syncthreads();
        // suffixes: the same scan over the reversed tile, tails as heads (tile position DL_TILE - 1's ignored)
        Seg agg{0.f, 0.f, 0};
#pragma unroll
        for (int k = 0; k < DL_IPT; ++k) {
            const int rj = threadIdx.x * DL_IPT + k, p = DL_TILE - 1 - rj;
            agg = seg_cat(agg, Seg{sw[sk(p)], swm[sk(p)], (rj != 0) && (sfl[p] & 2)});
        }
        const Seg rex = block_excl_scan<DL_T>(agg, sh, &total);
        float qw = rex.f ? rex.w : c.out_w + rex.w, qwm = rex.f ? rex.wm : c.out_wm + rex.wm;
        const float c23 = __fdiv_rn(2.f * dl_interval(interval, d_interval), 3.f);
        const float g = __ldg(d_g);
        const float coef = mean ? (float)((double)g / (double)hdr->n) : g;
        float gr[DL_IPT];
#pragma unroll
        for (int k = 0; k < DL_IPT; ++k) {
            const int rj = threadIdx.x * DL_IPT + k, p = DL_TILE - 1 - rj;
            const float w = sw[sk(p)], wm = swm[sk(p)], m = sm[sk(p)];
            if (rj != 0 && (sfl[p] & 2)) { qw = 0.f; qwm = 0.f; }
            gr[k] = coef * (2.f * (m * (spw[sk(p)] - qw) + (qwm - spwm[sk(p)])) + c23 * w);
            qw += w;
            qwm += wm;
        }
        __syncthreads();                         // every thread has read spw before it is overwritten
#pragma unroll
        for (int k = 0; k < DL_IPT; ++k) spw[sk(DL_TILE - 1 - (threadIdx.x * DL_IPT + k))] = gr[k];
    }
    __syncthreads();
#pragma unroll
    for (int k = 0; k < DL_IPT; ++k) {
        const int p = k * DL_T + threadIdx.x;
        const long long i = base + p;
        if (i >= in.M) break;
        out0[i] = spw[sk(p)];
        if (!GRAD) out2[i] = spwm[sk(p)];
    }
}

int dl_check_ws(const void* d_workspace, size_t workspace_bytes, int64_t M) {
    if (!d_workspace || (uintptr_t)d_workspace % 16) return K4_ERR_INVALID_ARG;
    if (workspace_bytes < k4_op_distloss_workspace_bytes(M)) return K4_ERR_WORKSPACE;
    return K4_OK;
}

// the tile pass and the carry pass (forward; segment_cumsum's first half)
void dl_scan(const DlIn& in, float interval, const float* d_interval, void* d_workspace, float* d_loss, cudaStream_t s) {
    const long long nt = dl_tiles(in.M);
    DlWs ws(d_workspace, nt);
    dl_tile_kernel<<<(unsigned)nt, DL_T, 0, s>>>(in, interval, d_interval, ws.tiles);
    dl_carry_kernel<<<1, DL_CT, 0, s>>>(ws.tiles, ws.car, nt, ws.hdr, d_loss);
}

#define DL_CHECK_LAUNCH()                                  \
    do {                                                   \
        cudaError_t e_ = cudaGetLastError();               \
        if (e_ != cudaSuccess) { k4_set_cuda_error(e_, "k4_distloss launch"); return K4_ERR_CUDA; } \
        return K4_OK;                                      \
    } while (0)

}  // namespace

extern "C" {

size_t k4_op_distloss_workspace_bytes(int64_t n_samples) {
    if (n_samples < 1) return 0;
    return sizeof(DlHeader) + (size_t)dl_tiles(n_samples) * (sizeof(DlTile) + sizeof(DlCarry));
}

int k4_op_distloss_forward(const float* d_w, const float* d_m, const int64_t* d_ray_id, int64_t n_samples, float interval,
                           const float* d_interval, float* d_loss, void* d_workspace, size_t workspace_bytes, k4_stream_t stream) {
    if (n_samples < 1 || !d_w || !d_m || !d_ray_id || !d_loss) return K4_ERR_INVALID_ARG;
    const int st = dl_check_ws(d_workspace, workspace_bytes, n_samples);
    if (st != K4_OK) return st;
    dl_scan(DlIn{d_w, d_m, (const long long*)d_ray_id, n_samples}, interval, d_interval, d_workspace, d_loss, (cudaStream_t)stream);
    DL_CHECK_LAUNCH();
}

int k4_op_distloss_backward(const float* d_w, const float* d_m, const int64_t* d_ray_id, int64_t n_samples, float interval,
                            const float* d_interval, const float* d_grad_loss, int32_t divide_by_n, const void* d_workspace,
                            size_t workspace_bytes, float* d_grad_w, k4_stream_t stream) {
    if (n_samples < 1 || !d_w || !d_m || !d_ray_id || !d_grad_loss || !d_grad_w) return K4_ERR_INVALID_ARG;
    const int st = dl_check_ws(d_workspace, workspace_bytes, n_samples);
    if (st != K4_OK) return st;
    const long long nt = dl_tiles(n_samples);
    DlWs ws(const_cast<void*>(d_workspace), nt);
    dl_apply_kernel<true><<<(unsigned)nt, DL_T, 0, (cudaStream_t)stream>>>(
        DlIn{d_w, d_m, (const long long*)d_ray_id, n_samples}, ws.car, ws.hdr, interval, d_interval, d_grad_loss, divide_by_n != 0, 0,
        d_grad_w, nullptr, nullptr, nullptr);
    DL_CHECK_LAUNCH();
}

int k4_op_segment_cumsum(const float* d_w, const float* d_s, const int64_t* d_ray_id, int64_t n_samples, int64_t n_rays,
                         float* d_w_prefix, float* d_w_total, float* d_ws_prefix, float* d_ws_total, void* d_workspace,
                         size_t workspace_bytes, k4_stream_t stream) {
    if (n_samples < 1 || n_rays < 1 || !d_w || !d_s || !d_ray_id || !d_w_prefix || !d_w_total || !d_ws_prefix || !d_ws_total)
        return K4_ERR_INVALID_ARG;
    const int st = dl_check_ws(d_workspace, workspace_bytes, n_samples);
    if (st != K4_OK) return st;
    cudaStream_t s = (cudaStream_t)stream;
    K4_CUDA_TRY(cudaMemsetAsync(d_w_total, 0, (size_t)n_rays * sizeof(float), s));
    K4_CUDA_TRY(cudaMemsetAsync(d_ws_total, 0, (size_t)n_rays * sizeof(float), s));
    const DlIn in{d_w, d_s, (const long long*)d_ray_id, n_samples};
    dl_scan(in, 0.f, nullptr, d_workspace, nullptr, s);
    const long long nt = dl_tiles(n_samples);
    DlWs ws(d_workspace, nt);
    dl_apply_kernel<false><<<(unsigned)nt, DL_T, 0, s>>>(in, ws.car, ws.hdr, 0.f, nullptr, nullptr, 0, n_rays,
                                                         d_w_prefix, d_w_total, d_ws_prefix, d_ws_total);
    DL_CHECK_LAUNCH();
}

}  // extern "C"
