// k4_video.cu -- the video streams of run_sr.py --render_video (run_sr.py:1399-1463) on the device: the depth video's
// masked percentiles and rainbow frames, and the u8 quantisation of rendered frames, with render_video_flipy /
// render_video_rot90 folded into the store addressing.
//
// Masked quantiles (np.percentile(depths_vis[bgmaps < 0.1], q), method 'linear'):
//   depths_vis = depth * (1 - bg) + bg in fp32, one rounding per operation (numpy's float32 expression), selected where
//   bg < 0.1f (for float32 data numpy's compare against 0.1 and against 0.1f agree: no float lies between them).
//   Each value maps to an order-preserving uint32 key (NaN above everything).  The order statistics that numpy's
//   'linear' method reads (prev / next of both quantiles, 4 ranks) are found by a radix select on the key, 11 + 11 + 10
//   bits, one histogram pass over the data per digit:
//     vq_hist_kernel<0>     count, NaN count and the histogram of the top 11 bits of the selected keys
//     vq_select_kernel<0>   (1 CTA) the ranks from the count, then per rank the bin holding it and the rank within it
//     vq_hist_kernel<1>     per distinct rank prefix, the histogram of the next 11 bits of the keys under it
//     vq_select_kernel<1>
//     vq_hist_kernel<2>     the last 10 bits
//     vq_select_kernel<2>   the four keys, then numpy's _lerp in fp64
//   Counts are integers added by atomics, so the selected keys, and the results, are exact and bitwise reproducible.
//   Because integer histograms add exactly, the passes also run split (k4_op_masked_quantiles_hist / _select): every
//   rank adds its own frames into a caller-visible int64 histogram, the callers sum the histograms (an all-reduce), and
//   every rank runs the same select on the sum, so all ranks carry the same state into the next pass.  The histogram is
//   the fused op's [VQ_RANKS][VQ_BINS] plus, in pass 0, the count and the NaN count (the fused op keeps those two in its
//   state instead).
//
// Depth-video frames: x = 1 - clip((depths_vis - dmin) / (dmax - dmin), 0, 1) in fp64, matplotlib's Colormap.__call__
// index (trunc(256 x), 256 -> 255, NaN -> the 'bad' colour 0), then the host's u8 table (to8b of the colormap's rgb).
// Frame quantiser: to8b(x) = trunc(fp32 255 * clip(x, 0, 1)).  Both write u8 [H', W', 3] frames, flipped and rotated.
#include "k4_internal.cuh"

namespace {

constexpr int VQ_NT = 256;
constexpr int VQ_BINS = 2048;                  // 11-bit digits (the last one uses 1024 of them)
constexpr int VQ_RANKS = 4;
constexpr int VQ_MAX_CTAS = 1024;
__host__ __device__ constexpr int vq_shift(int p) { return p == 0 ? 21 : (p == 1 ? 10 : 0); }   // digit p's lowest bit
__host__ __device__ constexpr int vq_nbins(int p) { return p == 2 ? 1024 : 2048; }
constexpr unsigned FULL = 0xffffffffu;
constexpr float VQ_BG_BELOW = 0.1f;

struct VqState {
    unsigned long long count, nans;
    unsigned long long rank[VQ_RANKS];         // rank within the keys that share prefix[r]
    unsigned int prefix[VQ_RANKS];             // the key's bits above the current digit
    int slot[VQ_RANKS];                        // histogram of rank r in passes 1 and 2: the first rank with its prefix
    double gamma[2];
};
constexpr size_t VQ_STATE_BYTES = 256;
static_assert(sizeof(VqState) <= VQ_STATE_BYTES, "state");

struct VqArgs {
    const float* depth;
    const float* bg;
    long long sd[3], sb[3];                    // element strides of (frame, row, column)
    long long n, H, W, rows;                   // rows = n * H
    double q[2];
    VqState* st;
    unsigned long long* hist;                  // [VQ_RANKS][VQ_BINS]
    unsigned long long* tally;                 // pass 0's count and NaN count: st->count / nans, or after hist's bins
    double* out;                               // [2]
    long long* count;
};

__device__ __forceinline__ unsigned vq_key(float v) {
    const unsigned u = __float_as_uint(v);
    if (v != v) return 0xffffffffu;
    return (u & 0x80000000u) ? ~u : (u | 0x80000000u);
}

__device__ __forceinline__ float vq_value(unsigned k) { return __uint_as_float((k & 0x80000000u) ? (k & 0x7fffffffu) : ~k); }

// depths * (1 - bgmaps) + bgmaps of run_sr.py:1459, each operation rounded once in fp32 as numpy does
__device__ __forceinline__ float depth_vis(float d, float b) { return __fadd_rn(__fmul_rn(d, __fsub_rn(1.0f, b)), b); }

// sh[bin] += 1 for every lane with `on`, one shared atomic per distinct bin of the warp (all lanes call it)
__device__ __forceinline__ void vq_add(unsigned* sh, unsigned bin, bool on) {
    if (!__ballot_sync(FULL, on)) return;
    const unsigned peers = __match_any_sync(FULL, on ? bin : 0xffffffffu);
    if (on && __ffs(peers) - 1 == (int)(threadIdx.x & 31)) atomicAdd(&sh[bin], (unsigned)__popc(peers));
}

template <int P>
__global__ void __launch_bounds__(VQ_NT) vq_hist_kernel(const __grid_constant__ VqArgs a) {
    constexpr int NH = P == 0 ? 1 : VQ_RANKS;
    __shared__ unsigned sh[NH * VQ_BINS];
    __shared__ unsigned long long sred[2][VQ_NT / 32];
    const int tid = threadIdx.x;
    for (int i = tid; i < NH * VQ_BINS; i += VQ_NT) sh[i] = 0;
    unsigned prefix[VQ_RANKS];
    bool own[VQ_RANKS];
#pragma unroll
    for (int r = 0; r < VQ_RANKS; ++r) {
        prefix[r] = P == 0 ? 0u : a.st->prefix[r];
        own[r] = P == 0 ? r == 0 : a.st->slot[r] == r;
    }
    __syncthreads();
    unsigned long long cnt = 0, nans = 0;
    for (long long row = blockIdx.x; row < a.rows; row += gridDim.x) {
        const long long f = row / a.H, y = row - f * a.H;
        const float* pd = a.depth + f * a.sd[0] + y * a.sd[1];
        const float* pb = a.bg + f * a.sb[0] + y * a.sb[1];
        for (long long x0 = 0; x0 < a.W; x0 += VQ_NT) {       // uniform over the CTA: every lane reaches vq_add
            const long long x = x0 + tid;
            bool sel = false;
            unsigned key = 0;
            if (x < a.W) {
                const float b = __ldg(pb + x * a.sb[2]);
                const float v = depth_vis(__ldg(pd + x * a.sd[2]), b);
                sel = b < VQ_BG_BELOW;
                key = vq_key(v);
                if (P == 0 && sel) { ++cnt; nans += v != v; }
            }
            if (P == 0) {
                vq_add(sh, key >> vq_shift(0), sel);
            } else {
#pragma unroll
                for (int r = 0; r < VQ_RANKS; ++r)
                    if (own[r])                                 // uniform: from the state
                        vq_add(sh + r * VQ_BINS, (key >> vq_shift(P)) & (vq_nbins(P) - 1),
                               sel && (key >> vq_shift(P - 1)) == prefix[r]);
            }
        }
    }
    __syncthreads();
    for (int i = tid; i < NH * VQ_BINS; i += VQ_NT)
        if (sh[i]) atomicAdd(&a.hist[i], (unsigned long long)sh[i]);
    if (P == 0) {
#pragma unroll
        for (int d = 16; d >= 1; d >>= 1) {
            cnt += __shfl_down_sync(FULL, cnt, d);
            nans += __shfl_down_sync(FULL, nans, d);
        }
        if ((tid & 31) == 0) { sred[0][tid >> 5] = cnt; sred[1][tid >> 5] = nans; }
        __syncthreads();
        if (tid == 0) {
            unsigned long long c = 0, m = 0;
            for (int i = 0; i < VQ_NT / 32; ++i) { c += sred[0][i]; m += sred[1][i]; }
            if (c) atomicAdd(&a.tally[0], c);
            if (m) atomicAdd(&a.tally[1], m);
        }
    }
}

// numpy's _lerp(a, b, t) of two float32 order statistics and a float64 weight: the difference in fp32, the rest in fp64
__device__ __forceinline__ double vq_lerp(float a, float b, double t) {
    const double d = (double)__fsub_rn(b, a);
    return t >= 0.5 ? __dsub_rn((double)b, __dmul_rn(d, __dsub_rn(1.0, t))) : __dadd_rn((double)a, __dmul_rn(d, t));
}

// One CTA, warp r for rank r.  Pass 0 first turns the count into numpy's indexes (_get_indexes / _get_gamma of the
// 'linear' method: virtual index (n - 1) q, previous = floor, next = previous + 1, both n - 1 at or above the last
// index, where numpy's previous index is -1 and its gamma therefore virtual + 1).
template <int P>
__global__ void __launch_bounds__(32 * VQ_RANKS) vq_select_kernel(const __grid_constant__ VqArgs a) {
    VqState* st = a.st;
    const int w = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const unsigned long long n = P == 0 ? a.tally[0] : st->count;
    if (P == 0 && threadIdx.x == 0) {
        for (int j = 0; j < 2; ++j) {
            unsigned long long prev = 0, next = 0;
            const double v = __dmul_rn((double)(long long)(n - 1), a.q[j]);
            if (n == 0) {
                st->gamma[j] = 0.0;
            } else if (v >= (double)(long long)(n - 1)) {
                prev = next = n - 1;
                st->gamma[j] = __dadd_rn(v, 1.0);
            } else {
                const double fl = floor(v);
                prev = (unsigned long long)fl;
                next = prev + 1;
                st->gamma[j] = __dsub_rn(v, fl);
            }
            st->rank[2 * j] = prev;
            st->rank[2 * j + 1] = next;
            st->prefix[2 * j] = st->prefix[2 * j + 1] = 0;
        }
    }
    __syncthreads();
    // the bin of rank r among this pass's digit: each lane sums NB / 32 consecutive bins, an inclusive warp scan finds
    // the lane, the lane walks its bins
    constexpr int NB = vq_nbins(P), PER = NB / 32;
    const unsigned long long* h = a.hist + (size_t)(P == 0 ? 0 : st->slot[w]) * VQ_BINS;
    const unsigned long long rank = st->rank[w];
    unsigned long long s = 0;
    for (int i = 0; i < PER; ++i) s += h[lane * PER + i];
    unsigned long long incl = s;
#pragma unroll
    for (int d = 1; d < 32; d <<= 1) {
        const unsigned long long t = __shfl_up_sync(FULL, incl, d);
        if (lane >= d) incl += t;
    }
    const unsigned hit = __ballot_sync(FULL, incl > rank);
    const int L = hit ? __ffs(hit) - 1 : 31;
    unsigned bin = 0;
    unsigned long long below = 0;
    if (lane == L) {
        unsigned long long c = incl - s;
        int i = 0;
        for (; i < PER - 1 && c + h[L * PER + i] <= rank; ++i) c += h[L * PER + i];
        bin = L * PER + i;
        below = c;
    }
    bin = __shfl_sync(FULL, bin, L);
    below = __shfl_sync(FULL, below, L);
    __syncthreads();                                            // every warp has read the state's ranks and slots
    if (lane == 0) {
        st->prefix[w] = (st->prefix[w] << (P == 2 ? 10 : 11)) | bin;
        st->rank[w] = hit ? rank - below : 0;
    }
    __syncthreads();
    if (threadIdx.x == 0) {
        if (P == 0) {                                           // the tally into the state (a no-op in the fused op)
            st->count = n;
            st->nans = a.tally[1];
        }
        if (P < 2) {
            for (int r = 0; r < VQ_RANKS; ++r) {
                int k = 0;
                while (st->prefix[k] != st->prefix[r]) ++k;
                st->slot[r] = k;
            }
        } else {
            float v[VQ_RANKS];
            for (int r = 0; r < VQ_RANKS; ++r) v[r] = vq_value(st->prefix[r]);
            for (int j = 0; j < 2; ++j)
                a.out[j] = (n == 0 || st->nans) ? __longlong_as_double(0x7ff8000000000000LL) : vq_lerp(v[2 * j], v[2 * j + 1], st->gamma[j]);
            *a.count = (long long)n;
        }
    }
}

// ---- flip / rot90 addressing: output (oy, ox) of rot90(flip(m)) reads m at (y, x); m is H x W, k in 0..3
__device__ __forceinline__ void src_of(long long oy, long long ox, long long H, long long W, int flip, int k, long long& y,
                                       long long& x) {
    if (k == 0) { y = oy; x = ox; }
    else if (k == 1) { y = ox; x = W - 1 - oy; }
    else if (k == 2) { y = H - 1 - oy; x = W - 1 - ox; }
    else { y = H - 1 - ox; x = oy; }
    if (flip) y = H - 1 - y;
}

struct DvArgs {
    const float* depth;
    const float* bg;
    long long sd[3], sb[3];
    long long H, W, Ho, Wo;
    int flip, k;
    const double* range;                       // device [dmin, dmax]
    unsigned char* out;                        // [n, Ho, Wo, 3]
    unsigned char lut[256 * 3];
};

constexpr int DV_NT = 128;
constexpr int DV_ROWS = 16;                    // output rows per CTA of the depth video: the table is staged once for them

// grid (ceil(Wo / DV_NT), ceil(Ho / DV_ROWS), n): one output column of DV_ROWS rows per thread
__global__ void __launch_bounds__(DV_NT) depth_video_kernel(const __grid_constant__ DvArgs a) {
    __shared__ unsigned char lut[256 * 3];
    for (int i = threadIdx.x; i < 256 * 3; i += DV_NT) lut[i] = a.lut[i];
    __syncthreads();
    const long long ox = (long long)blockIdx.x * DV_NT + threadIdx.x, f = blockIdx.z;
    if (ox >= a.Wo) return;
    const double dmin = a.range[0], dmax = a.range[1];
    const long long oy_end = min(a.Ho, (long long)(blockIdx.y + 1) * DV_ROWS);
    for (long long oy = (long long)blockIdx.y * DV_ROWS; oy < oy_end; ++oy) {
        long long y, x;
        src_of(oy, ox, a.H, a.W, a.flip, a.k, y, x);
        const float b = __ldg(a.bg + f * a.sb[0] + y * a.sb[1] + x * a.sb[2]);
        const float v = depth_vis(__ldg(a.depth + f * a.sd[0] + y * a.sd[1] + x * a.sd[2]), b);
        // numpy 2 promotes float32 - float64 scalar to float64: the normalisation is fp64, one rounding per operation
        double c = __ddiv_rn(__dsub_rn((double)v, dmin), __dsub_rn(dmax, dmin));
        if (c == c) c = c < 0.0 ? 0.0 : (c > 1.0 ? 1.0 : c);       // np.clip propagates NaN
        const double t = __dsub_rn(1.0, c);
        unsigned char rgb[3] = {0, 0, 0};                           // NaN: the colormap's 'bad' colour (0, 0, 0, 0)
        if (t == t) {
            const double xa = t * 256.0;                            // exact; t is in [0, 1]
            const int i = xa == 256.0 ? 255 : (int)xa;
#pragma unroll
            for (int ch = 0; ch < 3; ++ch) rgb[ch] = lut[3 * i + ch];
        }
        unsigned char* o = a.out + ((f * a.Ho + oy) * a.Wo + ox) * 3;
#pragma unroll
        for (int ch = 0; ch < 3; ++ch) o[ch] = rgb[ch];
    }
}

struct FqArgs {
    const float* rgb;
    long long s[3];                            // element strides of (row, column, channel)
    long long H, W, Ho, Wo;
    int flip, k;
    unsigned char* out;                        // [Ho, Wo, 3]
};

// grid (ceil(Wo / DV_NT), Ho): to8b, (255 * np.clip(x, 0, 1)).astype(np.uint8) of a float32 frame
__global__ void __launch_bounds__(DV_NT) frame_u8_kernel(const __grid_constant__ FqArgs a) {
    const long long ox = (long long)blockIdx.x * DV_NT + threadIdx.x, oy = blockIdx.y;
    if (ox >= a.Wo) return;
    long long y, x;
    src_of(oy, ox, a.H, a.W, a.flip, a.k, y, x);
    const float* p = a.rgb + y * a.s[0] + x * a.s[1];
    unsigned char* o = a.out + (oy * a.Wo + ox) * 3;
#pragma unroll
    for (int ch = 0; ch < 3; ++ch) {
        const float v = fminf(fmaxf(__ldg(p + ch * a.s[2]), 0.0f), 1.0f);     // NaN -> 0, as the conversion of NaN
        o[ch] = (unsigned char)__float2uint_rz(__fmul_rn(255.0f, v));
    }
}

constexpr long long VQ_MAX_ROWS = 0x7fffffffLL;
static_assert(K4_MASKED_QUANTILES_HIST_LEN == VQ_RANKS * VQ_BINS + 2, "the header's histogram length");

bool vq_shape_ok(int64_t n, int64_t H, int64_t W) {
    return n >= 1 && H >= 1 && W >= 1 && n <= VQ_MAX_ROWS && H <= VQ_MAX_ROWS && W <= VQ_MAX_ROWS && n * H <= VQ_MAX_ROWS;
}

// frames with Ho rows of Wo pixels: the grid's y and z limits
bool frame_shape_ok(int64_t n, int64_t H, int64_t W) {
    return n >= 1 && H >= 1 && W >= 1 && n <= 65535 && H <= 65535 && W <= 65535;
}

VqArgs vq_args(const float* d_depth, const float* d_bgmap, int64_t n, int64_t H, int64_t W, const int64_t depth_strides[3],
               const int64_t bgmap_strides[3], void* d_state) {
    VqArgs a{};
    a.depth = d_depth;
    a.bg = d_bgmap;
    for (int i = 0; i < 3; ++i) { a.sd[i] = depth_strides[i]; a.sb[i] = bgmap_strides[i]; }
    a.n = n;
    a.H = H;
    a.W = W;
    a.rows = n * H;
    a.st = (VqState*)d_state;
    return a;
}

void vq_hist(int pass, const VqArgs& a, cudaStream_t s) {
    const unsigned grid = (unsigned)std::min<long long>(a.rows, VQ_MAX_CTAS);
    if (pass == 0) vq_hist_kernel<0><<<grid, VQ_NT, 0, s>>>(a);
    else if (pass == 1) vq_hist_kernel<1><<<grid, VQ_NT, 0, s>>>(a);
    else vq_hist_kernel<2><<<grid, VQ_NT, 0, s>>>(a);
}

void vq_select(int pass, const VqArgs& a, cudaStream_t s) {
    if (pass == 0) vq_select_kernel<0><<<1, 32 * VQ_RANKS, 0, s>>>(a);
    else if (pass == 1) vq_select_kernel<1><<<1, 32 * VQ_RANKS, 0, s>>>(a);
    else vq_select_kernel<2><<<1, 32 * VQ_RANKS, 0, s>>>(a);
}

bool q_ok(const double q[2]) { return q[0] >= 0.0 && q[0] <= 1.0 && q[1] >= 0.0 && q[1] <= 1.0; }

int rot_k(int32_t rot90) { return ((rot90 % 4) + 4) % 4; }

int launch_error(const char* where) {
    const cudaError_t e = cudaGetLastError();
    if (e != cudaSuccess) { k4_set_cuda_error(e, where); return K4_ERR_CUDA; }
    return K4_OK;
}

}  // namespace

extern "C" {

size_t k4_op_masked_quantiles_workspace_bytes(int64_t n, int64_t H, int64_t W) {
    if (!vq_shape_ok(n, H, W)) return 0;
    return VQ_STATE_BYTES + sizeof(unsigned long long) * VQ_RANKS * VQ_BINS;
}

int k4_op_masked_quantiles(const float* d_depth, const float* d_bgmap, int64_t n, int64_t H, int64_t W,
                           const int64_t depth_strides[3], const int64_t bgmap_strides[3], const double h_q[2],
                           double* d_quantiles, int64_t* d_count, void* d_workspace, size_t workspace_bytes,
                           k4_stream_t stream) {
    if (!d_depth || !d_bgmap || !depth_strides || !bgmap_strides || !h_q || !d_quantiles || !d_count || !d_workspace)
        return K4_ERR_INVALID_ARG;
    if (!vq_shape_ok(n, H, W) || !q_ok(h_q)) return K4_ERR_INVALID_ARG;
    if ((uintptr_t)d_workspace % 16 || (uintptr_t)d_quantiles % sizeof(double) || (uintptr_t)d_count % sizeof(int64_t) ||
        (uintptr_t)d_depth % sizeof(float) || (uintptr_t)d_bgmap % sizeof(float))
        return K4_ERR_INVALID_ARG;
    if (workspace_bytes < k4_op_masked_quantiles_workspace_bytes(n, H, W)) return K4_ERR_WORKSPACE;
    VqArgs a = vq_args(d_depth, d_bgmap, n, H, W, depth_strides, bgmap_strides, d_workspace);
    a.q[0] = h_q[0];
    a.q[1] = h_q[1];
    a.hist = (unsigned long long*)((char*)d_workspace + VQ_STATE_BYTES);
    a.tally = &a.st->count;
    a.out = d_quantiles;
    a.count = (long long*)d_count;
    cudaStream_t s = (cudaStream_t)stream;
    const size_t hist_bytes = sizeof(unsigned long long) * VQ_RANKS * VQ_BINS;
    // pass 0 fills histogram 0; before passes 1 and 2 the select kernel has read it, so the next pass starts from zero
    K4_CUDA_TRY(cudaMemsetAsync(d_workspace, 0, VQ_STATE_BYTES + hist_bytes, s));
    for (int p = 0; p < 3; ++p) {
        if (p) K4_CUDA_TRY(cudaMemsetAsync(a.hist, 0, hist_bytes, s));
        vq_hist(p, a, s);
        vq_select(p, a, s);
    }
    return launch_error("k4_op_masked_quantiles launch");
}

size_t k4_op_masked_quantiles_pass_workspace_bytes(void) { return VQ_STATE_BYTES; }

int k4_op_masked_quantiles_hist(int32_t pass, const float* d_depth, const float* d_bgmap, int64_t n, int64_t H, int64_t W,
                                const int64_t depth_strides[3], const int64_t bgmap_strides[3], int64_t* d_hist,
                                const void* d_workspace, size_t workspace_bytes, k4_stream_t stream) {
    if (pass < 0 || pass > 2 || !depth_strides || !bgmap_strides || !d_hist || !d_workspace) return K4_ERR_INVALID_ARG;
    if (n < 0 || !vq_shape_ok(n ? n : 1, H, W)) return K4_ERR_INVALID_ARG;       // a share may hold no frames
    if (n && (!d_depth || !d_bgmap || (uintptr_t)d_depth % sizeof(float) || (uintptr_t)d_bgmap % sizeof(float)))
        return K4_ERR_INVALID_ARG;
    if ((uintptr_t)d_workspace % 16 || (uintptr_t)d_hist % sizeof(int64_t)) return K4_ERR_INVALID_ARG;
    if (workspace_bytes < VQ_STATE_BYTES) return K4_ERR_WORKSPACE;
    if (n == 0) return K4_OK;
    VqArgs a = vq_args(d_depth, d_bgmap, n, H, W, depth_strides, bgmap_strides, const_cast<void*>(d_workspace));
    a.hist = (unsigned long long*)d_hist;
    a.tally = a.hist + VQ_RANKS * VQ_BINS;
    vq_hist(pass, a, (cudaStream_t)stream);
    return launch_error("k4_op_masked_quantiles_hist launch");
}

int k4_op_masked_quantiles_select(int32_t pass, const int64_t* d_hist, const double h_q[2], double* d_quantiles,
                                  int64_t* d_count, void* d_workspace, size_t workspace_bytes, k4_stream_t stream) {
    if (pass < 0 || pass > 2 || !d_hist || !h_q || !d_quantiles || !d_count || !d_workspace) return K4_ERR_INVALID_ARG;
    if (!q_ok(h_q)) return K4_ERR_INVALID_ARG;
    if ((uintptr_t)d_workspace % 16 || (uintptr_t)d_hist % sizeof(int64_t) || (uintptr_t)d_quantiles % sizeof(double) ||
        (uintptr_t)d_count % sizeof(int64_t))
        return K4_ERR_INVALID_ARG;
    if (workspace_bytes < VQ_STATE_BYTES) return K4_ERR_WORKSPACE;
    VqArgs a{};
    a.q[0] = h_q[0];
    a.q[1] = h_q[1];
    a.st = (VqState*)d_workspace;
    a.hist = (unsigned long long*)const_cast<int64_t*>(d_hist);          // read only: the select reads the histogram
    a.tally = a.hist + VQ_RANKS * VQ_BINS;
    a.out = d_quantiles;
    a.count = (long long*)d_count;
    vq_select(pass, a, (cudaStream_t)stream);
    return launch_error("k4_op_masked_quantiles_select launch");
}

int k4_op_depth_video_u8(const float* d_depth, const float* d_bgmap, int64_t n, int64_t H, int64_t W,
                         const int64_t depth_strides[3], const int64_t bgmap_strides[3], const double* d_range,
                         const uint8_t* h_lut, int32_t flip_y, int32_t rot90, uint8_t* d_out, k4_stream_t stream) {
    if (!d_depth || !d_bgmap || !depth_strides || !bgmap_strides || !d_range || !h_lut || !d_out) return K4_ERR_INVALID_ARG;
    if (!frame_shape_ok(n, H, W) || (flip_y != 0 && flip_y != 1)) return K4_ERR_INVALID_ARG;
    if ((uintptr_t)d_range % sizeof(double) || (uintptr_t)d_depth % sizeof(float) || (uintptr_t)d_bgmap % sizeof(float))
        return K4_ERR_INVALID_ARG;
    DvArgs a{};
    a.depth = d_depth;
    a.bg = d_bgmap;
    for (int i = 0; i < 3; ++i) { a.sd[i] = depth_strides[i]; a.sb[i] = bgmap_strides[i]; }
    a.H = H;
    a.W = W;
    a.k = rot_k(rot90);
    a.Ho = a.k & 1 ? W : H;
    a.Wo = a.k & 1 ? H : W;
    a.flip = flip_y;
    a.range = d_range;
    a.out = d_out;
    for (int i = 0; i < 256 * 3; ++i) a.lut[i] = h_lut[i];
    const dim3 grid((unsigned)((a.Wo + DV_NT - 1) / DV_NT), (unsigned)((a.Ho + DV_ROWS - 1) / DV_ROWS), (unsigned)n);
    depth_video_kernel<<<grid, DV_NT, 0, (cudaStream_t)stream>>>(a);
    return launch_error("k4_op_depth_video_u8 launch");
}

int k4_op_frame_u8(const float* d_rgb, int64_t H, int64_t W, const int64_t strides[3], int32_t flip_y, int32_t rot90,
                   uint8_t* d_out, k4_stream_t stream) {
    if (!d_rgb || !strides || !d_out) return K4_ERR_INVALID_ARG;
    if (!frame_shape_ok(1, H, W) || (flip_y != 0 && flip_y != 1) || (uintptr_t)d_rgb % sizeof(float)) return K4_ERR_INVALID_ARG;
    FqArgs a{};
    a.rgb = d_rgb;
    for (int i = 0; i < 3; ++i) a.s[i] = strides[i];
    a.H = H;
    a.W = W;
    a.k = rot_k(rot90);
    a.Ho = a.k & 1 ? W : H;
    a.Wo = a.k & 1 ? H : W;
    a.flip = flip_y;
    a.out = d_out;
    const dim3 grid((unsigned)((a.Wo + DV_NT - 1) / DV_NT), (unsigned)a.Ho);
    frame_u8_kernel<<<grid, DV_NT, 0, (cudaStream_t)stream>>>(a);
    return launch_error("k4_op_frame_u8 launch");
}

}  // extern "C"
