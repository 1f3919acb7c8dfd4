// k4_lpips.cu -- LPIPS 0.1 (lpips.LPIPS(net='vgg' | 'alex', version='0.1')), the perceptual metric of utils.rgb_lpips
// (lib/utils.py:137-149), on the device, so that a rendered or decoded frame is scored where it is.
//
// For two [H, W, 3] images x0, x1 in [0, 1] (fp32, read through element strides):
//     x = (2 x - 1 - shift) / scale                     per channel, fp32 (lpips' normalize=True and ScalingLayer)
//     f_k = tap k of the trunk (VGG16 relu1_2 .. relu5_3, or AlexNet relu1 .. relu5)
//     score = sum_k mean_pixels( sum_c lin_k[c] (f0_k / (|f0_k| + 1e-10) - f1_k / (|f1_k| + 1e-10))^2 )
// with |f| the L2 norm of a pixel's channel vector.
//
//   VGG16 convolutions   k4_sr.cu's wgmma implicit GEMM (conv3x3_ws_kernel<64>, through k4_conv3x3_relu_split): fp16
//                        operands, fp32 accumulation, bias + ReLU in the epilogue, one launch per block of 64 output
//                        channels.  Every activation and weight is an fp16 pair hi + lo, so the trunk is fp32-class
//                        (rounding fp16 operands once makes the score's error as large as torch's TF32 evaluation
//                        has, from the rounding noise of both images' features): activations are fp16 NHWC [hi | lo |
//                        hi] of C channels each, the layer a GEMM of K = 3 C.  The input layer's 9 channels are stored
//                        padded to 32 (zero weights beyond them).
//   AlexNet convolutions alex_conv_kernel: direct fp32 convolution (any K / stride / pad), NHWC fp32.  It only runs
//                        at the sizes AlexNet is used at (LR frames); 11x11 / stride 4 and 5x5 do not fit the 3x3 GEMM.
//   pooling              pool2_split_kernel (VGG, 2x2 / 2, the max of hi + lo) and pool3s2_f32_kernel (AlexNet, 3x3 / 2),
//                        floor sizes, exact.
//   head                 lpips_head_kernel<T, NV>: 8 lanes per pixel, the channel vectors in registers; norms, the
//                        normalised difference and the lin weights in fp64; one fp64 sum per CTA of 256 pixels, in a
//                        fixed order.  lpips_final_kernel sums them per tap in a fixed order, divides by the tap's
//                        pixel count and adds the five means.  No atomics, no host synchronisation: the score is
//                        bitwise reproducible.
#include <cstring>
#include <new>
#include <type_traits>

#include "k4_internal.cuh"

namespace {

constexpr unsigned FULL = 0xffffffffu;
constexpr int LP_VGG_CONVS = 13, LP_ALEX_CONVS = 5, LP_TAPS = 5;
constexpr int LP_MAX_SIDE = 16384;
constexpr int HD_NT = 256;                       // head: 8 warps of 32 / LANES pixels per step
constexpr int HD_PIX = 256;                      // pixels per head CTA
constexpr int FIN_NT = 1024;
constexpr int AX_PX = 16;                        // alex_conv_kernel: output pixels of a row per CTA
constexpr int AX_NT = 64;                        // ... and output channels per CTA

// lpips' ScalingLayer buffers (torch.Tensor of these doubles: fp32)
__constant__ float c_shift[3] = {-.030f, -.088f, -.188f};
__constant__ float c_scale[3] = {.458f, .448f, .450f};

enum { LP_CONV = 0, LP_POOL = 1 };
struct LpOp { int kind, conv, tap; };
// torchvision vgg16().features[:30] / alexnet().features[:12] as lpips slices them: convolutions (with their ReLU),
// pools, and the taps (outputs of slice1 .. slice5)
constexpr LpOp VGG_OPS[] = {{LP_CONV, 0, -1}, {LP_CONV, 1, 0}, {LP_POOL, -1, -1}, {LP_CONV, 2, -1}, {LP_CONV, 3, 1},
                            {LP_POOL, -1, -1}, {LP_CONV, 4, -1}, {LP_CONV, 5, -1}, {LP_CONV, 6, 2}, {LP_POOL, -1, -1},
                            {LP_CONV, 7, -1}, {LP_CONV, 8, -1}, {LP_CONV, 9, 3}, {LP_POOL, -1, -1}, {LP_CONV, 10, -1},
                            {LP_CONV, 11, -1}, {LP_CONV, 12, 4}};
constexpr LpOp ALEX_OPS[] = {{LP_CONV, 0, 0}, {LP_POOL, -1, -1}, {LP_CONV, 1, 1}, {LP_POOL, -1, -1}, {LP_CONV, 2, 2},
                             {LP_CONV, 3, 3}, {LP_CONV, 4, 4}};
constexpr int VGG_NOPS = sizeof(VGG_OPS) / sizeof(LpOp), ALEX_NOPS = sizeof(ALEX_OPS) / sizeof(LpOp);
constexpr int VGG_CIN[LP_VGG_CONVS] = {3, 64, 64, 128, 128, 256, 256, 256, 512, 512, 512, 512, 512};
constexpr int VGG_COUT[LP_VGG_CONVS] = {64, 64, 128, 128, 256, 256, 256, 512, 512, 512, 512, 512, 512};
struct AlexL { int K, s, p, cin, cout; };
constexpr AlexL ALEX_L[LP_ALEX_CONVS] = {{11, 4, 2, 3, 64}, {5, 1, 2, 64, 192}, {3, 1, 1, 192, 384}, {3, 1, 1, 384, 256},
                                          {3, 1, 1, 256, 256}};
constexpr int TAP_C[2][LP_TAPS] = {{64, 128, 256, 512, 512}, {64, 192, 384, 256, 256}};

int lp_nops(int net) { return net == K4_LPIPS_VGG ? VGG_NOPS : ALEX_NOPS; }
const LpOp& lp_op(int net, int s) { return net == K4_LPIPS_VGG ? VGG_OPS[s - 1] : ALEX_OPS[s - 1]; }
size_t lp_elem(int net) { return net == K4_LPIPS_VGG ? sizeof(__half) : sizeof(float); }

// Stored shape (h, w, c) of stage s: 0 = the scaled input (VGG: 32 channels, hi, lo, hi of the 3 real ones then
// zeros), s >= 1 = the output of op s (VGG: 3 C channels, hi | lo | hi).  False when a stage is empty (the image is too
// small for the trunk).
bool lp_shape(int net, long long H, long long W, int s, long long* h, long long* w, long long* c) {
    long long hh = H, ww = W, cc = net == K4_LPIPS_VGG ? 32 : 3;
    for (int i = 1; i <= s; ++i) {
        const LpOp& o = lp_op(net, i);
        if (net == K4_LPIPS_VGG) {
            if (o.kind == LP_CONV) cc = 3 * VGG_COUT[o.conv];
            else { hh /= 2; ww /= 2; }
        } else if (o.kind == LP_CONV) {
            const AlexL& L = ALEX_L[o.conv];
            hh = (hh + 2 * L.p - L.K) / L.s + 1;
            ww = (ww + 2 * L.p - L.K) / L.s + 1;
            cc = L.cout;
        } else {
            hh = hh >= 3 ? (hh - 3) / 2 + 1 : 0;
            ww = ww >= 3 ? (ww - 3) / 2 + 1 : 0;
        }
        if (hh < 1 || ww < 1) return false;
    }
    *h = hh; *w = ww; *c = cc;
    return true;
}

bool lp_size_ok(int net, long long H, long long W) {
    long long h, w, c;
    return (net == K4_LPIPS_VGG || net == K4_LPIPS_ALEX) && H >= 1 && W >= 1 && H <= LP_MAX_SIDE && W <= LP_MAX_SIDE &&
           lp_shape(net, H, W, lp_nops(net), &h, &w, &c);
}

// Workspace: per image two activation buffers (stage s lives in buffer s & 1), then the head's per-CTA sums per tap.
struct LpWs { size_t buf, partial_off[LP_TAPS], n_partial[LP_TAPS], total; };
LpWs lp_ws(int net, long long H, long long W) {
    LpWs L{};
    for (int s = 0; s <= lp_nops(net); ++s) {
        long long h, w, c;
        lp_shape(net, H, W, s, &h, &w, &c);
        const size_t b = (size_t)(h * w * c) * lp_elem(net);
        if (b > L.buf) L.buf = b;
    }
    L.buf = (L.buf + 255) / 256 * 256;
    size_t o = 4 * L.buf;
    for (int s = 1, k = 0; s <= lp_nops(net); ++s) {
        if (lp_op(net, s).tap < 0) continue;
        long long h, w, c;
        lp_shape(net, H, W, s, &h, &w, &c);
        L.partial_off[k] = o;
        L.n_partial[k] = (size_t)((h * w + HD_PIX - 1) / HD_PIX);
        o += 8 * L.n_partial[k];
        ++k;
    }
    L.total = o;
    return L;
}

// ---- input: 2x - 1 and the scaling layer, fp32 with one rounding per operation as torch computes them
template <bool F16>
__global__ void lpips_input_kernel(const float* __restrict__ img, long long s0, long long s1, long long s2, int H, int W,
                                   void* __restrict__ dst) {
    const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= (long long)H * W) return;
    const long long y = i / W, x = i - y * W;
    float v[3];
#pragma unroll
    for (int c = 0; c < 3; ++c) {
        const float t = __fsub_rn(__fmul_rn(2.f, __ldg(img + y * s0 + x * s1 + c * s2)), 1.f);
        v[c] = __fdiv_rn(__fsub_rn(t, c_shift[c]), c_scale[c]);
    }
    if (F16) {                                         // hi, lo, hi of the three channels, then zeros
        __half hi[3], lo[3];
#pragma unroll
        for (int c = 0; c < 3; ++c) {
            hi[c] = __float2half_rn(v[c]);
            lo[c] = __float2half_rn(v[c] - __half2float(hi[c]));
        }
        uint4 q[4] = {};
        __half2* h = reinterpret_cast<__half2*>(q);
        h[0] = __halves2half2(hi[0], hi[1]);
        h[1] = __halves2half2(hi[2], lo[0]);
        h[2] = __halves2half2(lo[1], lo[2]);
        h[3] = __halves2half2(hi[0], hi[1]);
        h[4] = __halves2half2(hi[2], __float2half_rn(0.f));
        uint4* d = reinterpret_cast<uint4*>(static_cast<__half*>(dst) + i * 32);
#pragma unroll
        for (int j = 0; j < 4; ++j) d[j] = q[j];
    } else {
        float* d = static_cast<float*>(dst) + i * 3;
        d[0] = v[0]; d[1] = v[1]; d[2] = v[2];
    }
}

// ---- VGG max-pool 2x2 / stride 2 (floor) on the [hi | lo | hi] layout of C channels: one thread per output pixel and
// channel; the value is hi + lo, compared in fp64 (exact), and the winner's pair is copied
__global__ void pool2_split_kernel(const __half* __restrict__ src, __half* __restrict__ dst, int h, int w, int C) {
    const int ho = h / 2, wo = w / 2;
    const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= (long long)ho * wo * C) return;
    const int c = (int)(i % C);
    const long long pix = i / C, yo = pix / wo, xo = pix - yo * wo;
    __half bh = __float2half_rn(0.f), bl = bh;
    double best = -INFINITY;
#pragma unroll
    for (int k = 0; k < 4; ++k) {
        const __half* p = src + (((2 * yo + (k >> 1)) * w + 2 * xo + (k & 1)) * 3 * C + c);
        const __half hi = p[0], lo = p[C];
        const double v = (double)__half2float(hi) + (double)__half2float(lo);
        if (v > best) { best = v; bh = hi; bl = lo; }
    }
    __half* d = dst + pix * 3 * C + c;
    d[0] = bh; d[C] = bl; d[2 * C] = bh;
}

// ---- AlexNet max-pool 3x3 / stride 2 (floor) on fp32 NHWC
__global__ void pool3s2_f32_kernel(const float* __restrict__ src, float* __restrict__ dst, int h, int w, int C) {
    const int ho = (h - 3) / 2 + 1, wo = (w - 3) / 2 + 1;
    const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= (long long)ho * wo * C) return;
    const int c = (int)(i % C);
    const long long pix = i / C, yo = pix / wo, xo = pix - yo * wo;
    float m = -INFINITY;
    for (int dy = 0; dy < 3; ++dy)
        for (int dx = 0; dx < 3; ++dx) m = fmaxf(m, __ldg(src + ((2 * yo + dy) * w + 2 * xo + dx) * C + c));
    dst[i] = m;
}

// ---- AlexNet convolution + bias + ReLU, direct fp32: a CTA computes AX_PX outputs of one row for AX_NT output
// channels (one per thread); per kernel row the input row segment it needs is staged in shared memory ([seg][cin],
// read as broadcasts), the weights ([K][K][cin][cout], so a warp's loads are contiguous) come from L1 / L2.
struct AlexConvArgs { const float* src; const float* w; const float* b; float* dst; int h, w_, cin, ho, wo, cout, K, stride, pad; };

__global__ void __launch_bounds__(AX_NT) alex_conv_kernel(const __grid_constant__ AlexConvArgs a) {
    extern __shared__ float srow[];
    const int co = blockIdx.y * AX_NT + threadIdx.x;
    const int tiles_x = (a.wo + AX_PX - 1) / AX_PX;
    const int oy = blockIdx.x / tiles_x, ox0 = (blockIdx.x - oy * tiles_x) * AX_PX;
    const int seg = (AX_PX - 1) * a.stride + a.K, ix0 = ox0 * a.stride - a.pad;
    float acc[AX_PX];
#pragma unroll
    for (int j = 0; j < AX_PX; ++j) acc[j] = 0.f;
    for (int ky = 0; ky < a.K; ++ky) {
        const int iy = oy * a.stride - a.pad + ky;
        if (iy < 0 || iy >= a.h) continue;                 // uniform over the CTA
        __syncthreads();
        for (int i = threadIdx.x; i < seg * a.cin; i += AX_NT) {
            const int j = i / a.cin, ci = i - j * a.cin, ix = ix0 + j;
            srow[i] = (ix >= 0 && ix < a.w_) ? __ldg(a.src + ((long long)iy * a.w_ + ix) * a.cin + ci) : 0.f;
        }
        __syncthreads();
        for (int kx = 0; kx < a.K; ++kx) {
            const float* wp = a.w + (size_t)(ky * a.K + kx) * a.cin * a.cout + co;
            const float* sp = srow + kx * a.cin;
            for (int ci = 0; ci < a.cin; ++ci) {
                const float wv = __ldg(wp + (size_t)ci * a.cout);
#pragma unroll
                for (int j = 0; j < AX_PX; ++j) acc[j] = fmaf(wv, sp[j * a.stride * a.cin + ci], acc[j]);
            }
        }
    }
    const float bv = __ldg(a.b + co);
#pragma unroll
    for (int j = 0; j < AX_PX; ++j)
        if (ox0 + j < a.wo) a.dst[((long long)oy * a.wo + ox0 + j) * a.cout + co] = fmaxf(acc[j] + bv, 0.f);
}

// torch [cout][cin][K][K] -> [K][K][cin][cout]
__global__ void alex_pack_kernel(const float* __restrict__ w, float* __restrict__ dst, int cout, int cin, int K) {
    const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= (long long)cout * cin * K * K) return;
    const int co = (int)(i % cout);
    long long r = i / cout;
    const int ci = (int)(r % cin);
    r /= cin;
    dst[i] = w[((long long)co * cin + ci) * K * K + r];
}

// ---- head: 8 lanes per pixel, lane l8 holds channels 8 (l8 + 8 v) .. +7 for v < NV (C = 64 NV), kept as loaded
// (fp16 VGG features in 4 registers per 8 channels) and widened on use
template <typename T> struct Raw8;
__device__ __forceinline__ float half_at(const uint4& q, int e) {
    const unsigned u = (e >> 1) == 0 ? q.x : ((e >> 1) == 1 ? q.y : ((e >> 1) == 2 ? q.z : q.w));
    return __half2float(__ushort_as_half((unsigned short)(u >> (16 * (e & 1)))));
}
template <> struct Raw8<__half> {                      // VGG: hi at channel c, lo at c + C; the value hi + lo (exact)
    uint4 h, l;
    __device__ __forceinline__ void load(const __half* p, int C) {
        h = __ldg(reinterpret_cast<const uint4*>(p));
        l = __ldg(reinterpret_cast<const uint4*>(p + C));
    }
    __device__ __forceinline__ void zero() { h = l = make_uint4(0, 0, 0, 0); }
    __device__ __forceinline__ double at(int e) const { return (double)half_at(h, e) + (double)half_at(l, e); }
};
template <> struct Raw8<float> {
    float4 a, b;
    __device__ __forceinline__ void load(const float* p, int) {
        a = __ldg(reinterpret_cast<const float4*>(p));
        b = __ldg(reinterpret_cast<const float4*>(p) + 1);
    }
    __device__ __forceinline__ void zero() { a = b = make_float4(0.f, 0.f, 0.f, 0.f); }
    __device__ __forceinline__ double at(int e) const {
        const float4& v = e < 4 ? a : b;
        const int i = e & 3;
        return i == 0 ? v.x : (i == 1 ? v.y : (i == 2 ? v.z : v.w));
    }
};
template <int LANES>
__device__ __forceinline__ double sum_lanes(double v) {
#pragma unroll
    for (int o = LANES / 2; o >= 1; o >>= 1) v += __shfl_xor_sync(FULL, v, o);   // a butterfly: every lane ends with
    return v;                                                                     // the same bits
}

// LANES lanes per pixel (32 / LANES pixels per warp and step), lane l holds channels 8 (l + LANES v) .. +7, v < NV:
// C = 8 LANES NV channels, stored with a pixel stride of 3 C (VGG's hi | lo | hi) or C (AlexNet)
template <typename T, int LANES, int NV>
__global__ void __launch_bounds__(HD_NT) lpips_head_kernel(const T* __restrict__ f0, const T* __restrict__ f1,
                                                           const float* __restrict__ lin, long long P, double* __restrict__ partial) {
    constexpr int C = 8 * LANES * NV, PPW = 32 / LANES;
    constexpr int PS = std::is_same<T, __half>::value ? 3 * C : C;
    __shared__ double sred[HD_NT / 32];
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, l = lane % LANES;
    double part = 0.0;
    for (int it = 0; it < HD_PIX / (PPW * (HD_NT / 32)); ++it) {
        const long long pix = (long long)blockIdx.x * HD_PIX + (it * (HD_NT / 32) + warp) * PPW + lane / LANES;
        const bool in = pix < P;
        Raw8<T> a[NV], b[NV];
#pragma unroll
        for (int v = 0; v < NV; ++v) {
            if (in) {
                a[v].load(f0 + pix * PS + 8 * (l + LANES * v), C);
                b[v].load(f1 + pix * PS + 8 * (l + LANES * v), C);
            } else {
                a[v].zero();
                b[v].zero();
            }
        }
        double s0 = 0.0, s1 = 0.0;
#pragma unroll
        for (int v = 0; v < NV; ++v)
#pragma unroll
            for (int e = 0; e < 8; ++e) {
                const double x = a[v].at(e), y = b[v].at(e);
                s0 += x * x;
                s1 += y * y;
            }
        const double n0 = __dsqrt_rn(sum_lanes<LANES>(s0)) + 1e-10, n1 = __dsqrt_rn(sum_lanes<LANES>(s1)) + 1e-10;
        double d = 0.0;
#pragma unroll
        for (int v = 0; v < NV; ++v)
#pragma unroll
            for (int e = 0; e < 8; ++e) {
                const double q = a[v].at(e) / n0 - b[v].at(e) / n1;
                d += (double)__ldg(lin + 8 * (l + LANES * v) + e) * (q * q);
            }
        d = sum_lanes<LANES>(d);
        if (l == 0 && in) part += d;
    }
#pragma unroll
    for (int o = 16; o >= 1; o >>= 1) part += __shfl_down_sync(FULL, part, o);
    if (lane == 0) sred[warp] = part;
    __syncthreads();
    if (threadIdx.x == 0) {
        double t = sred[0];
        for (int i = 1; i < HD_NT / 32; ++i) t += sred[i];
        partial[blockIdx.x] = t;
    }
}

struct FinalArgs { const double* partial[LP_TAPS]; long long n[LP_TAPS]; double count[LP_TAPS]; };

// One CTA: per tap, thread t sums a contiguous chunk of the CTA sums in order, then a warp tree and one thread over
// the warps; the mean of tap k is that sum / count k, and the score their sum in tap order.
__global__ void __launch_bounds__(FIN_NT) lpips_final_kernel(const __grid_constant__ FinalArgs a, double* __restrict__ out) {
    __shared__ double sred[FIN_NT / 32];
    __shared__ double smean[LP_TAPS];
    for (int k = 0; k < LP_TAPS; ++k) {
        const long long n = a.n[k], chunk = (n + FIN_NT - 1) / FIN_NT;
        const long long lo = min(n, (long long)threadIdx.x * chunk), hi = min(n, lo + chunk);
        double s = 0.0;
        for (long long i = lo; i < hi; ++i) s += a.partial[k][i];
#pragma unroll
        for (int o = 16; o >= 1; o >>= 1) s += __shfl_down_sync(FULL, s, o);
        if ((threadIdx.x & 31) == 0) sred[threadIdx.x >> 5] = s;
        __syncthreads();
        if (threadIdx.x == 0) {
            double t = sred[0];
            for (int i = 1; i < FIN_NT / 32; ++i) t += sred[i];
            smean[k] = t / a.count[k];
        }
        __syncthreads();
    }
    if (threadIdx.x == 0) *out = (((smean[0] + smean[1]) + smean[2]) + smean[3]) + smean[4];
}

unsigned blocks_for(long long n, int nt) { return (unsigned)((n + nt - 1) / nt); }

}  // namespace

struct k4_lpips {
    int net;
    K4Conv3x3Pack vgg[LP_VGG_CONVS];
    float* alex_w[LP_ALEX_CONVS];             // [K][K][cin][cout]
    float* alex_b[LP_ALEX_CONVS];
    float* lin[LP_TAPS];
};

namespace {

int lp_conv(const k4_lpips* n, int conv, const void* src, void* dst, long long h, long long w, cudaStream_t s) {
    if (n->net == K4_LPIPS_VGG)
        return k4_conv3x3_relu_split(n->vgg[conv], static_cast<const __half*>(src), (int)h, (int)w, static_cast<__half*>(dst), s);
    const AlexL& L = ALEX_L[conv];
    AlexConvArgs a{};
    a.src = static_cast<const float*>(src); a.w = n->alex_w[conv]; a.b = n->alex_b[conv]; a.dst = static_cast<float*>(dst);
    a.h = (int)h; a.w_ = (int)w; a.cin = L.cin; a.cout = L.cout; a.K = L.K; a.stride = L.s; a.pad = L.p;
    a.ho = (int)((h + 2 * L.p - L.K) / L.s + 1); a.wo = (int)((w + 2 * L.p - L.K) / L.s + 1);
    const int seg = (AX_PX - 1) * L.s + L.K;
    const dim3 grid((unsigned)(a.ho * ((a.wo + AX_PX - 1) / AX_PX)), (unsigned)(L.cout / AX_NT));
    alex_conv_kernel<<<grid, AX_NT, (size_t)seg * L.cin * sizeof(float), s>>>(a);
    K4_CUDA_TRY(cudaGetLastError());
    return K4_OK;
}

int lp_pool(const k4_lpips* n, const void* src, void* dst, long long h, long long w, long long c, cudaStream_t s) {
    if (n->net == K4_LPIPS_VGG) {
        pool2_split_kernel<<<blocks_for((h / 2) * (w / 2) * (c / 3), 256), 256, 0, s>>>(
            static_cast<const __half*>(src), static_cast<__half*>(dst), (int)h, (int)w, (int)(c / 3));
    } else {
        pool3s2_f32_kernel<<<blocks_for(((h - 3) / 2 + 1) * ((w - 3) / 2 + 1) * c, 256), 256, 0, s>>>(
            static_cast<const float*>(src), static_cast<float*>(dst), (int)h, (int)w, (int)c);
    }
    K4_CUDA_TRY(cudaGetLastError());
    return K4_OK;
}

// The head of one tap: VGG's widths 64, 128, 256, 512 (split fp16 features), AlexNet's 64, 192, 384, 256 (fp32).
int lp_head(int net, const void* f0, const void* f1, const float* lin, long long P, long long C, double* partial, cudaStream_t s) {
    const unsigned g = blocks_for(P, HD_PIX);
    const __half *h0 = static_cast<const __half*>(f0), *h1 = static_cast<const __half*>(f1);
    const float *s0 = static_cast<const float*>(f0), *s1 = static_cast<const float*>(f1);
    if (net == K4_LPIPS_VGG) {
        if (C == 64) lpips_head_kernel<__half, 8, 1><<<g, HD_NT, 0, s>>>(h0, h1, lin, P, partial);
        else if (C == 128) lpips_head_kernel<__half, 8, 2><<<g, HD_NT, 0, s>>>(h0, h1, lin, P, partial);
        else if (C == 256) lpips_head_kernel<__half, 8, 4><<<g, HD_NT, 0, s>>>(h0, h1, lin, P, partial);
        else lpips_head_kernel<__half, 16, 4><<<g, HD_NT, 0, s>>>(h0, h1, lin, P, partial);
    } else {
        if (C == 64) lpips_head_kernel<float, 8, 1><<<g, HD_NT, 0, s>>>(s0, s1, lin, P, partial);
        else if (C == 192) lpips_head_kernel<float, 8, 3><<<g, HD_NT, 0, s>>>(s0, s1, lin, P, partial);
        else if (C == 256) lpips_head_kernel<float, 8, 4><<<g, HD_NT, 0, s>>>(s0, s1, lin, P, partial);
        else lpips_head_kernel<float, 8, 6><<<g, HD_NT, 0, s>>>(s0, s1, lin, P, partial);
    }
    K4_CUDA_TRY(cudaGetLastError());
    return K4_OK;
}

// Runs stages 1 .. upto of the trunk on images 0 .. n_img-1, stage 0 already in buf[i][0]; with `heads`, the head of
// every tap on the pair.
int lp_trunk(const k4_lpips* n, long long H, long long W, int n_img, unsigned char* const (*buf)[2], int upto,
             unsigned char* ws, const LpWs& L, cudaStream_t s, bool heads) {
    for (int st = 1; st <= upto; ++st) {
        const LpOp& o = lp_op(n->net, st);
        long long h, w, c, ho, wo, co;
        lp_shape(n->net, H, W, st - 1, &h, &w, &c);
        lp_shape(n->net, H, W, st, &ho, &wo, &co);
        for (int i = 0; i < n_img; ++i) {
            const void* src = buf[i][(st - 1) & 1];
            void* dst = buf[i][st & 1];
            const int r = o.kind == LP_CONV ? lp_conv(n, o.conv, src, dst, h, w, s) : lp_pool(n, src, dst, h, w, c, s);
            if (r != K4_OK) return r;
        }
        if (heads && o.tap >= 0) {
            double* partial = reinterpret_cast<double*>(ws + L.partial_off[o.tap]);
            const long long C = n->net == K4_LPIPS_VGG ? co / 3 : co;
            const int r = lp_head(n->net, buf[0][st & 1], buf[1][st & 1], n->lin[o.tap], ho * wo, C, partial, s);
            if (r != K4_OK) return r;
        }
    }
    return K4_OK;
}

int lp_input(const k4_lpips* n, const float* img, const int64_t st[3], long long H, long long W, void* dst, cudaStream_t s) {
    const unsigned grid = blocks_for(H * W, 256);
    if (n->net == K4_LPIPS_VGG) lpips_input_kernel<true><<<grid, 256, 0, s>>>(img, st[0], st[1], st[2], (int)H, (int)W, dst);
    else lpips_input_kernel<false><<<grid, 256, 0, s>>>(img, st[0], st[1], st[2], (int)H, (int)W, dst);
    K4_CUDA_TRY(cudaGetLastError());
    return K4_OK;
}

bool lp_ptrs_ok(const void* ws, size_t bytes, const k4_lpips* n, long long H, long long W) {
    return ws && (uintptr_t)ws % 256 == 0 && bytes >= lp_ws(n->net, H, W).total;
}

}  // namespace

extern "C" {

int k4_lpips_destroy(k4_lpips* n) {
    if (!n) return K4_OK;
    for (int i = 0; i < LP_VGG_CONVS; ++i) k4_conv3x3_free(&n->vgg[i]);
    for (int i = 0; i < LP_ALEX_CONVS; ++i) { cudaFree(n->alex_w[i]); cudaFree(n->alex_b[i]); }
    for (int i = 0; i < LP_TAPS; ++i) cudaFree(n->lin[i]);
    delete n;
    return K4_OK;
}

int k4_lpips_create(int32_t net, const float* const* h_params, int32_t n_params, k4_stream_t stream, k4_lpips** out) {
    if (!out) return K4_ERR_INVALID_ARG;
    *out = nullptr;
    if (!h_params || (net != K4_LPIPS_VGG && net != K4_LPIPS_ALEX)) return K4_ERR_INVALID_ARG;
    const int n_conv = net == K4_LPIPS_VGG ? LP_VGG_CONVS : LP_ALEX_CONVS;
    if (n_params != 2 * n_conv + LP_TAPS) return K4_ERR_INVALID_ARG;
    for (int i = 0; i < n_params; ++i)
        if (!h_params[i]) return K4_ERR_INVALID_ARG;
    int st = k4_device_check();
    if (st != K4_OK) return st;
    cudaStream_t s = (cudaStream_t)stream;
    k4_lpips* n = new (std::nothrow) k4_lpips();
    if (!n) return K4_ERR_INVALID_ARG;
    memset(n, 0, sizeof(*n));
    n->net = net;
#define LP_TRY(x) do { st = (x); if (st != K4_OK) { k4_lpips_destroy(n); return st; } } while (0)
#define LP_CUDA(x) do { const cudaError_t e_ = (x); if (e_ != cudaSuccess) { k4_set_cuda_error(e_, #x); k4_lpips_destroy(n); return K4_ERR_CUDA; } } while (0)
    for (int i = 0; i < n_conv; ++i) {
        const float* w = h_params[2 * i];
        const float* b = h_params[2 * i + 1];
        if (net == K4_LPIPS_VGG) {
            LP_TRY(k4_conv3x3_pack(w, b, VGG_COUT[i], VGG_CIN[i], s, &n->vgg[i]));
        } else {
            const AlexL& L = ALEX_L[i];
            const long long nw = (long long)L.cout * L.cin * L.K * L.K;
            LP_CUDA(cudaMalloc(&n->alex_w[i], nw * sizeof(float)));
            LP_CUDA(cudaMalloc(&n->alex_b[i], L.cout * sizeof(float)));
            alex_pack_kernel<<<blocks_for(nw, 256), 256, 0, s>>>(w, n->alex_w[i], L.cout, L.cin, L.K);
            LP_CUDA(cudaGetLastError());
            LP_CUDA(cudaMemcpyAsync(n->alex_b[i], b, L.cout * sizeof(float), cudaMemcpyDeviceToDevice, s));
        }
    }
    for (int k = 0; k < LP_TAPS; ++k) {
        const int C = TAP_C[net][k];
        LP_CUDA(cudaMalloc(&n->lin[k], C * sizeof(float)));
        LP_CUDA(cudaMemcpyAsync(n->lin[k], h_params[2 * n_conv + k], C * sizeof(float), cudaMemcpyDeviceToDevice, s));
    }
    LP_CUDA(cudaStreamSynchronize(s));                  // the caller's parameters may be freed on return
#undef LP_TRY
#undef LP_CUDA
    *out = n;
    return K4_OK;
}

size_t k4_lpips_workspace_bytes(const k4_lpips* n, int64_t H, int64_t W) {
    if (!n || !lp_size_ok(n->net, H, W)) return 0;
    return lp_ws(n->net, H, W).total;
}

int k4_lpips_forward(const k4_lpips* n, const float* d_img0, const float* d_img1, const int64_t strides0[3],
                     const int64_t strides1[3], int64_t H, int64_t W, double* d_out, void* d_workspace, size_t workspace_bytes,
                     k4_stream_t stream) {
    if (!n || !d_img0 || !d_img1 || !strides0 || !strides1 || !d_out || !d_workspace) return K4_ERR_INVALID_ARG;
    if (!lp_size_ok(n->net, H, W) || (uintptr_t)d_out % 8 || (uintptr_t)d_workspace % 256) return K4_ERR_INVALID_ARG;
    const LpWs L = lp_ws(n->net, H, W);
    if (workspace_bytes < L.total) return K4_ERR_WORKSPACE;
    cudaStream_t s = (cudaStream_t)stream;
    unsigned char* ws = static_cast<unsigned char*>(d_workspace);
    unsigned char* const buf[2][2] = {{ws, ws + L.buf}, {ws + 2 * L.buf, ws + 3 * L.buf}};
    int st = lp_input(n, d_img0, strides0, H, W, buf[0][0], s);
    if (st == K4_OK) st = lp_input(n, d_img1, strides1, H, W, buf[1][0], s);
    if (st == K4_OK) st = lp_trunk(n, H, W, 2, buf, lp_nops(n->net), ws, L, s, true);
    if (st != K4_OK) return st;
    FinalArgs f{};
    for (int k = 0, stg = 1; stg <= lp_nops(n->net); ++stg) {
        if (lp_op(n->net, stg).tap < 0) continue;
        long long h, w, c;
        lp_shape(n->net, H, W, stg, &h, &w, &c);
        f.partial[k] = reinterpret_cast<const double*>(ws + L.partial_off[k]);
        f.n[k] = (long long)L.n_partial[k];
        f.count[k] = (double)(h * w);
        ++k;
    }
    lpips_final_kernel<<<1, FIN_NT, 0, s>>>(f, d_out);
    K4_CUDA_TRY(cudaGetLastError());
    return K4_OK;
}

int k4_testing_lpips_stage(const k4_lpips* n, const float* d_img, const int64_t strides[3], int64_t H, int64_t W,
                           int32_t stage, void* d_out, int64_t out_shape[3], void* d_workspace, size_t workspace_bytes,
                           k4_stream_t stream) {
    if (out_shape) out_shape[0] = out_shape[1] = out_shape[2] = 0;
    if (!n || !d_img || !strides || !out_shape || !d_workspace) return K4_ERR_INVALID_ARG;
    if (!lp_size_ok(n->net, H, W) || stage < 0 || stage > lp_nops(n->net) || (uintptr_t)d_workspace % 256)
        return K4_ERR_INVALID_ARG;
    const LpWs L = lp_ws(n->net, H, W);
    if (workspace_bytes < L.total) return K4_ERR_WORKSPACE;
    long long h, w, c;
    lp_shape(n->net, H, W, stage, &h, &w, &c);
    out_shape[0] = h; out_shape[1] = w; out_shape[2] = c;
    if (!d_out) return K4_OK;                           // a shape query
    cudaStream_t s = (cudaStream_t)stream;
    unsigned char* ws = static_cast<unsigned char*>(d_workspace);
    unsigned char* const buf[1][2] = {{ws, ws + L.buf}};
    int st = lp_input(n, d_img, strides, H, W, buf[0][0], s);
    if (st == K4_OK) st = lp_trunk(n, H, W, 1, buf, stage, ws, L, s, false);
    if (st != K4_OK) return st;
    K4_CUDA_TRY(cudaMemcpyAsync(d_out, buf[0][stage & 1], (size_t)(h * w * c) * lp_elem(n->net), cudaMemcpyDeviceToDevice, s));
    return K4_OK;
}

}  // extern "C"
