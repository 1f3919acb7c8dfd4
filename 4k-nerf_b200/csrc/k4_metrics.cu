// k4_metrics.cu -- the SSIM of render_viewpoints' eval_ssim (utils.rgb_ssim, lib/utils.py:88-134, the mip-NeRF variant)
// on the device, so that a rendered frame is scored where it was rendered.
//
// Per channel c of two [H, W, 3] images x0, x1 and a window of f taps w (computed on the host by utils.rgb_ssim's own
// expression), with blur(z) = the separable 'valid' correlation with w reversed, along axis 0 (rows) first and then
// along axis 1 (columns):
//     m0 = blur(x0), m1 = blur(x1), v0 = max(blur(x0 x0) - m0 m0, 0), v1 = max(blur(x1 x1) - m1 m1, 0),
//     cov = sign(c) min(sqrt(v0 v1), |c|) with c = blur(x0 x1) - m0 m1,
//     ssim = ((2 m0 m1 + c1)(2 cov + c2)) / ((m0 m0 + m1 m1 + c1)(v0 + v1 + c2))
// on the [H-f+1, W-f+1, 3] map, and its mean.  Everything is fp64 as in the numpy path (fp32 inputs are widened
// exactly); the formula's operations are the numpy path's, one rounding each (no contraction), so the map differs from
// numpy's only through the order of the tap sums.
//
//   ssim_tile_kernel    one CTA per SS_TH x SS_TW output tile, the three channels in turn: the channel's input halo
//                       (SS_TH + f - 1 rows, SS_TW + f - 1 columns of both images) is staged in shared memory as fp64,
//                       the vertical pass writes the five moment maps of the tile's rows to shared memory, and the
//                       horizontal pass plus the formula run in registers (SS_R outputs per thread along a row, so each
//                       moment read from shared memory feeds up to SS_R taps).  The CTA's sum of its map values, in a
//                       fixed order, goes to the workspace.
//   ssim_mean_kernel    one CTA: the per-tile sums in a fixed order, divided by the map's size.
// The tiles depend on (H, W, f) only, and no sum depends on timing: the mean is bitwise reproducible.  No atomics, no
// host synchronisation.
#include "k4_internal.cuh"

namespace {

constexpr int SS_TH = 32;                       // output rows of a tile (= a warp's lanes in the horizontal pass)
constexpr int SS_TW = 32;                       // output columns of a tile
constexpr int SS_R = 4;                         // outputs per thread in both passes
constexpr int SS_NT = SS_TH * SS_TW / SS_R;     // 256 threads: one horizontal item each
constexpr int SS_MEAN_NT = 1024;
constexpr unsigned FULL = 0xffffffffu;
static_assert(SS_TH == 32 && SS_TW % SS_R == 0 && SS_TH % SS_R == 0, "tile shape");

struct SsimArgs {
    const void* img0;
    const void* img1;
    long long st0[3], st1[3];                   // element strides of (row, column, channel)
    long long H, W, Ho, Wo;
    int f, tiles_x;
    double c1, c2;
    double win[K4_SSIM_MAX_FILTER];             // the taps as utils.rgb_ssim computes them (blur uses them reversed)
    double* map;                                // [Ho, Wo, 3] or nullptr
    double* partial;                            // [tiles]
};

// halo row stride in doubles: odd, so that the horizontal pass's lanes (one row each) hit distinct banks
__host__ __device__ inline int ss_hcp(int f) { return (SS_TW + f - 1) | 1; }
__host__ __device__ inline int ss_hr(int f) { return SS_TH + f - 1; }

size_t ss_smem_bytes(int f) {
    return sizeof(double) * ((size_t)K4_SSIM_MAX_FILTER + 1 + (size_t)ss_hcp(f) * (2 * ss_hr(f) + 5 * SS_TH));
}

long long ss_tiles(long long Ho, long long Wo) { return ((Ho + SS_TH - 1) / SS_TH) * ((Wo + SS_TW - 1) / SS_TW); }

template <typename T>
__device__ __forceinline__ double ss_load(const void* p, long long i) { return (double)__ldg((const T*)p + i); }

// numpy's sign(c) * minimum(sqrt(v0 v1), |c|), np.maximum(v, 0) and the ratio, one rounding per operation
__device__ __forceinline__ double ss_value(double m0, double m1, double s00, double s11, double s01, double c1, double c2) {
    double v0 = __dadd_rn(s00, -__dmul_rn(m0, m0));
    double v1 = __dadd_rn(s11, -__dmul_rn(m1, m1));
    v0 = v0 < 0.0 ? 0.0 : v0;
    v1 = v1 < 0.0 ? 0.0 : v1;
    const double c = __dadd_rn(s01, -__dmul_rn(m0, m1));
    const double r = __dsqrt_rn(__dmul_rn(v0, v1)), a = fabs(c);
    const double cov = (double)((c > 0.0) - (c < 0.0)) * (r < a ? r : a);
    const double num = __dmul_rn(__dadd_rn(__dmul_rn(__dmul_rn(2.0, m0), m1), c1), __dadd_rn(__dmul_rn(2.0, cov), c2));
    const double den = __dmul_rn(__dadd_rn(__dadd_rn(__dmul_rn(m0, m0), __dmul_rn(m1, m1)), c1), __dadd_rn(__dadd_rn(v0, v1), c2));
    return __ddiv_rn(num, den);
}

template <typename T>
__global__ void __launch_bounds__(SS_NT, 2) ssim_tile_kernel(const __grid_constant__ SsimArgs a) {
    extern __shared__ double smem[];
    __shared__ double sred[SS_NT / 32];
    const int f = a.f, hcp = ss_hcp(f), hr = ss_hr(f), hc = SS_TW + f - 1;
    double* sw = smem;                                   // sw[k] = win[f - 1 - k]: blur's reversed taps
    double* sx0 = smem + K4_SSIM_MAX_FILTER + 1;         // [hr][hcp] halo of x0, then of x1
    double* sx1 = sx0 + hr * hcp;
    double* sv = sx1 + hr * hcp;                         // [5][SS_TH][hcp]: vertical sums of x0, x1, x0 x0, x1 x1, x0 x1
    const int tid = threadIdx.x;
    const long long ty = blockIdx.x / a.tiles_x, tx = blockIdx.x - ty * a.tiles_x;
    const long long y0 = ty * SS_TH, x0 = tx * SS_TW;
    if (tid < f) sw[tid] = a.win[f - 1 - tid];
    const int xg = tid >> 5, r = tid & 31;               // horizontal item: tile row r, columns SS_R * xg + [0, SS_R)
    const long long y = y0 + r;
    double part = 0.0;
    for (int ch = 0; ch < 3; ++ch) {
        // ---- the channel's halo, zero outside the image (those entries feed only outputs outside the map)
        for (int i = tid; i < hr * hc; i += SS_NT) {
            const int row = i / hc, col = i - row * hc;
            const long long gy = y0 + row, gx = x0 + col;
            double u0 = 0.0, u1 = 0.0;
            if (gy < a.H && gx < a.W) {
                u0 = ss_load<T>(a.img0, gy * a.st0[0] + gx * a.st0[1] + ch * a.st0[2]);
                u1 = ss_load<T>(a.img1, gy * a.st1[0] + gx * a.st1[1] + ch * a.st1[2]);
            }
            sx0[row * hcp + col] = u0;
            sx1[row * hcp + col] = u1;
        }
        __syncthreads();
        // ---- vertical pass: rows SS_R * g + q of column j; input row i of the thread's window feeds tap k = i - q of
        // output q (k is the same for every lane: the branch is uniform)
        for (int it = tid; it < (SS_TH / SS_R) * hc; it += SS_NT) {
            const int g = it / hc, j = it - g * hc;
            double acc[SS_R][5];
#pragma unroll
            for (int q = 0; q < SS_R; ++q)
#pragma unroll
                for (int m = 0; m < 5; ++m) acc[q][m] = 0.0;
            const double* p0 = sx0 + (SS_R * g) * hcp + j;
            const double* p1 = sx1 + (SS_R * g) * hcp + j;
            for (int i = 0; i < f + SS_R - 1; ++i) {
                const double u0 = p0[i * hcp], u1 = p1[i * hcp];
                const double v[5] = {u0, u1, __dmul_rn(u0, u0), __dmul_rn(u1, u1), __dmul_rn(u0, u1)};
#pragma unroll
                for (int q = 0; q < SS_R; ++q) {
                    const int k = i - q;
                    if (k >= 0 && k < f) {
                        const double w = sw[k];
#pragma unroll
                        for (int m = 0; m < 5; ++m) acc[q][m] = fma(w, v[m], acc[q][m]);
                    }
                }
            }
#pragma unroll
            for (int q = 0; q < SS_R; ++q)
#pragma unroll
                for (int m = 0; m < 5; ++m) sv[(m * SS_TH + SS_R * g + q) * hcp + j] = acc[q][m];
        }
        __syncthreads();
        // ---- horizontal pass and the formula: outputs (r, SS_R * xg + q)
        double acc[SS_R][5];
#pragma unroll
        for (int q = 0; q < SS_R; ++q)
#pragma unroll
            for (int m = 0; m < 5; ++m) acc[q][m] = 0.0;
        const double* pv = sv + r * hcp + SS_R * xg;
        for (int i = 0; i < f + SS_R - 1; ++i) {
            double v[5];
#pragma unroll
            for (int m = 0; m < 5; ++m) v[m] = pv[m * SS_TH * hcp + i];
#pragma unroll
            for (int q = 0; q < SS_R; ++q) {
                const int k = i - q;
                if (k >= 0 && k < f) {
                    const double w = sw[k];
#pragma unroll
                    for (int m = 0; m < 5; ++m) acc[q][m] = fma(w, v[m], acc[q][m]);
                }
            }
        }
#pragma unroll
        for (int q = 0; q < SS_R; ++q) {
            const long long x = x0 + SS_R * xg + q;
            if (y < a.Ho && x < a.Wo) {
                const double s = ss_value(acc[q][0], acc[q][1], acc[q][2], acc[q][3], acc[q][4], a.c1, a.c2);
                part += s;
                if (a.map) a.map[(y * a.Wo + x) * 3 + ch] = s;
            }
        }
        // the next channel's halo overwrites sx only: every thread is past the vertical pass, and sv is rewritten only
        // after the next halo's __syncthreads, when every thread has finished this horizontal pass
    }
    // CTA sum in a fixed order: warp tree, then one thread over the warps
#pragma unroll
    for (int d = 16; d >= 1; d >>= 1) part += __shfl_down_sync(FULL, part, d);
    if ((tid & 31) == 0) sred[tid >> 5] = part;
    __syncthreads();
    if (tid == 0) {
        double s = sred[0];
        for (int i = 1; i < SS_NT / 32; ++i) s += sred[i];
        a.partial[blockIdx.x] = s;
    }
}

// One CTA: thread t sums a contiguous chunk of the tile sums in order, then a warp tree and one thread over the warps.
__global__ void __launch_bounds__(SS_MEAN_NT) ssim_mean_kernel(const double* __restrict__ partial, long long n, double count,
                                                               double* __restrict__ mean) {
    __shared__ double sred[SS_MEAN_NT / 32];
    const long long chunk = (n + SS_MEAN_NT - 1) / SS_MEAN_NT;
    const long long lo = min(n, (long long)threadIdx.x * chunk), hi = min(n, lo + chunk);
    double s = 0.0;
    for (long long i = lo; i < hi; ++i) s += partial[i];
#pragma unroll
    for (int d = 16; d >= 1; d >>= 1) s += __shfl_down_sync(FULL, s, d);
    if ((threadIdx.x & 31) == 0) sred[threadIdx.x >> 5] = s;
    __syncthreads();
    if (threadIdx.x == 0) {
        double t = sred[0];
        for (int i = 1; i < SS_MEAN_NT / 32; ++i) t += sred[i];
        *mean = t / count;
    }
}

template <typename T>
int ssim_launch(const SsimArgs& a, long long tiles, double* d_mean, cudaStream_t s) {
    const size_t smem = ss_smem_bytes(a.f);
    K4_CUDA_TRY(cudaFuncSetAttribute(ssim_tile_kernel<T>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    ssim_tile_kernel<T><<<(unsigned)tiles, SS_NT, smem, s>>>(a);
    ssim_mean_kernel<<<1, SS_MEAN_NT, 0, s>>>(a.partial, tiles, (double)(a.Ho * a.Wo * 3), d_mean);
    const cudaError_t e = cudaGetLastError();
    if (e != cudaSuccess) { k4_set_cuda_error(e, "k4_op_rgb_ssim launch"); return K4_ERR_CUDA; }
    return K4_OK;
}

bool ss_shape_ok(int64_t H, int64_t W, int32_t filter_size) {
    return filter_size >= 1 && filter_size <= K4_SSIM_MAX_FILTER && H >= filter_size && W >= filter_size &&
           H <= (1LL << 31) && W <= (1LL << 31) && ss_tiles(H - filter_size + 1, W - filter_size + 1) <= 0x7fffffffLL;
}

}  // namespace

extern "C" {

size_t k4_op_rgb_ssim_workspace_bytes(int64_t H, int64_t W, int32_t filter_size) {
    if (!ss_shape_ok(H, W, filter_size)) return 0;
    return sizeof(double) * (size_t)ss_tiles(H - filter_size + 1, W - filter_size + 1);
}

int k4_op_rgb_ssim(const void* d_img0, const void* d_img1, int32_t dtype, int64_t H, int64_t W, const int64_t strides0[3],
                   const int64_t strides1[3], const double* h_win, int32_t filter_size, double c1, double c2,
                   double* d_map, double* d_mean, void* d_workspace, size_t workspace_bytes, k4_stream_t stream) {
    if (!d_img0 || !d_img1 || !strides0 || !strides1 || !h_win || !d_mean || !d_workspace) return K4_ERR_INVALID_ARG;
    if ((dtype != K4_DTYPE_F32 && dtype != K4_DTYPE_F64) || !ss_shape_ok(H, W, filter_size)) return K4_ERR_INVALID_ARG;
    if ((uintptr_t)d_workspace % sizeof(double) || (uintptr_t)d_mean % sizeof(double) || (uintptr_t)d_map % sizeof(double))
        return K4_ERR_INVALID_ARG;
    if (workspace_bytes < k4_op_rgb_ssim_workspace_bytes(H, W, filter_size)) return K4_ERR_WORKSPACE;
    SsimArgs a{};
    a.img0 = d_img0;
    a.img1 = d_img1;
    for (int i = 0; i < 3; ++i) { a.st0[i] = strides0[i]; a.st1[i] = strides1[i]; }
    a.H = H;
    a.W = W;
    a.Ho = H - filter_size + 1;
    a.Wo = W - filter_size + 1;
    a.f = filter_size;
    a.tiles_x = (int)((a.Wo + SS_TW - 1) / SS_TW);
    a.c1 = c1;
    a.c2 = c2;
    for (int k = 0; k < filter_size; ++k) a.win[k] = h_win[k];
    a.map = d_map;
    a.partial = (double*)d_workspace;
    const long long tiles = ss_tiles(a.Ho, a.Wo);
    cudaStream_t s = (cudaStream_t)stream;
    return dtype == K4_DTYPE_F32 ? ssim_launch<float>(a, tiles, d_mean, s) : ssim_launch<double>(a, tiles, d_mean, s);
}

}  // extern "C"
