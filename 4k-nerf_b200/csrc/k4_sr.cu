// k4_sr.cu -- the VC-Decoder (SFTNet, lib/sr_esrnet.py:400-465) on sm_90a.
//
// Replaces the reference's 229 cuDNN convolutions + torch.cat copies + F.interpolate + leaky_relu
// launches per tile (SURVEY.md section 3.3) with
//
//   conv3x3_ws_kernel<N>   every 3x3 convolution as an im2col-free implicit GEMM on warpgroup MMAs (wgmma), one
//       persistent warp-specialised CTA per SM (TMA / cp.async producer warpgroup, two MMA + epilogue warpgroups,
//       5-6 stage shared-memory ring); see the comment at the kernel.  The SFT layers that follow a convolution run in
//       its epilogue (epilogue_sft);
//   sft_mma_kernel<COUT>   SFTLayer (lib/sr_esrnet.py:112-123) as its own pass (K4_SR_FUSE_SFT=0), mma.sync on the
//       same operand fragments as the fused epilogue; sft_kernel is its fp32 one-thread-per-pixel form (K4_SFT_FP32=1);
//   condnet_mma_kernel     CondNet (lib/sr_esrnet.py:440-444) of the depth condition (num_cond 1) on mma.sync, fp32-class
//       through a 3-term fp16 split; condnet_wide_mma_kernel<NKS> the same for a wide condition (num_cond 2..64: the
//       view-direction embedding), whose 3x3 layer is an implicit GEMM on the tensor cores as well;
//   condnet_kernel<WIDE>   CondNet, one thread per pixel, fp32 (the A/B reference, K4_CONDNET_FP32=1).
//
// Numerics: conv operands are fp16 (weights and activations), accumulation fp32, the residual trunk and all CondNet
// math stay fp32.  (The reference itself runs these convs with TF32 operands: torch.backends.cudnn.allow_tf32
// defaults to True.)
#include <cuda.h>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <new>

#include "k4_internal.cuh"
#include "k4_ptx.cuh"
#include "k4_wgmma.cuh"

// Intermediate activations and the condition map are rounded to fp16 with h2_sat: those of a trained checkpoint may
// exceed the fp16 range, and a clamped operand degrades gracefully where an inf poisons the frame.
//
// Programmatic dependent launch: every decoder kernel is launched with programmaticStreamSerialization (sr_launch), so
// its CTAs are scheduled while the previous kernel drains; what a kernel does before its pdl_wait_and_release()
// (barrier init, constant weights) overlaps the predecessor's tail.

namespace {

constexpr int SR_TY = 16;                            // output rows of a tile
constexpr int SR_HY = SR_TY + 2;                     // halo rows
constexpr int SR_CK = 16;                            // input channels per K slice (one k16 MMA step per tap)

enum { SRM_STORE_F16 = 0,      // dst_h[c0..c0+N) = act(acc + b)
       SRM_TRUNK = 1,          // dst_f = (acc + b) * scale + add_f                  (conv5: x5*0.2 + x)
       SRM_ADD_STORE_F16 = 2,  // dst_h = fp16((acc + b) + add_f)                    (conv_body + feat)
       SRM_STORE_F32F16 = 3,   // dst_f = acc + b (fp32, 64 ch) and dst_h = fp16     (conv_first: trunk + feat)
       SRM_OUT_NCHW = 4,       // out_nchw[c][y][x] = acc + b, c < n_valid          (conv_last)
       // conv3x3_ws_kernel only: the SFT layer(s) that follow the convolution run in its epilogue (see epilogue_sft)
       SRM_STORE_F16_SFT = 5,  // dst_h = fp16(sft(lrelu(acc + b)))                          (conv4 -> sft1)
       SRM_TRUNK_SFT = 6,      // t = (acc + b) * scale [+ add_f]; dst_f (, dst_f2) = t; dst_h2 = fp16(sft(t))   (conv_first, conv5 of rdb1/2 -> next sft0)
       SRM_TRUNK_SFT2 = 7 };   // t as above; u = sft(t) * scale2 + add_f2; dst_f = u; dst_h2 = fp16(sft2(u))    (conv5 of rdb3 -> RRDB tail -> next sft0 / sftbody)

struct ConvParams {
    const __half* src; int src_cstride; int src_c0; int cin;       // cin: multiple of 32 (zero padded weights beyond the real Cin)
    int H, W; int upsample;                                        // output size; upsample: src is (H/2) x (W/2), nearest
    const unsigned char* wpack; const float* bias;
    int mode; float lrelu; float scale;
    __half* dst_h; int dst_cstride; int dst_c0;
    float* dst_f; const float* add_f;                              // fp32 [P,64]
    float* out_nchw; int n_valid;
    int use_tma;                                                   // conv3x3_ws_kernel: halo by TMA tensor copies (not with upsample)
    // conv3x3_ws_kernel only -- sub-pixel form of "nearest x2 + 3x3 conv": the convolution iterates over the SOURCE
    // grid with `ntaps` (4) of the nine halo offsets and phase-combined weights, and writes output pixel
    // (y*out_s + out_oy, x*out_s + out_ox) of an (H*out_s) x (W*out_s) destination.  Defaults: 9 taps, out_s = 1.
    int ntaps; unsigned char tap_dy[9], tap_dx[9];
    int out_s, out_oy, out_ox;
    // rows [y_lo, y_hi) of the iteration grid computed by this launch (all kernels; y_hi == 0 means all H rows): a unit
    // of the multi-GPU decoder only needs, per layer, the rows inside the remaining receptive field of its kept block
    int y_lo, y_hi;
    float* dst_f2;                                                 // SRM_STORE_F32F16: second fp32 copy (the initial trunk)
    // SRM_OUT_NCHW: output pixel (y, x) of channel c goes to out_nchw[c*out_ps + (y-crop_y0)*out_rs + (x-crop_x0)] when it lies
    // in the crop window [crop_y0,crop_y1) x [crop_x0,crop_x1) (the kept block of a tile, written straight into the frame)
    long long out_ps, out_rs; int crop_y0, crop_y1, crop_x0, crop_x1;
    // ... and at the same offset into out_extra[0 .. n_out_extra): the same window of the other ranks' frames (peer-mapped,
    // k4_srnet_forward_roi_peers) -- the multi-GPU exchange as NVLink stores of the kernel that produces the pixels
    int n_out_extra; float* out_extra[K4_MAX_PEERS - 1];
    // fused SFT epilogues (SRM_*_SFT*): fp16 condition map [P,32], the fragment-ordered operand blocks of the SFT layer(s)
    // (sft_frag_layout), the fp16 destination of the (last) modulated result, the RRDB input for the block tail
    const __half* cond16; const unsigned char* sftw; const unsigned char* sftw2; int sft_n;
    __half* dst_h2; int dst2_cstride, dst2_c0; const float* add_f2; float scale2;
    // SRM_STORE_F16 with lrelu == 0 (LPIPS's VGG16, k4_conv3x3_relu_split): relu = max(x, 0); split > 0 also stores
    // lo = fp16(x - hi) at channel + split and hi again at channel + 2 split, the input layout of the next such layer
    int relu, split;
};

__device__ __forceinline__ void sr_store_out(const ConvParams& p, long long idx, float v) {
    p.out_nchw[idx] = v;
#pragma unroll 1
    for (int e = 0; e < p.n_out_extra; ++e) p.out_extra[e][idx] = v;
}

// SFT operands for the in-epilogue mma.sync evaluation: fp16 weights W0 [64][32] (scale_conv0 rows then shift_conv0 rows),
// W1s [n][32], W1h [n][32] with 40-half row pitch (conflict-free fragment loads), then fp32 biases b0 [64], b1s + 1 [n], b1h [n].
constexpr int SFTF_PITCH = 40;
struct SftFrag { int off_w0, off_w1s, off_w1h, off_b0, off_b1s, off_b1h, total; };
__host__ __device__ inline SftFrag sft_frag_layout(int n) {
    SftFrag L; int o = 0;
    L.off_w0 = o; o += 64 * SFTF_PITCH * 2;
    L.off_w1s = o; o += n * SFTF_PITCH * 2;
    L.off_w1h = o; o += n * SFTF_PITCH * 2;
    L.off_b0 = o; o += 64 * 4;
    L.off_b1s = o; o += n * 4;
    L.off_b1h = o; o += n * 4;
    L.total = (o + 15) & ~15;
    return L;
}
constexpr int SFTF_MAX = 2 * (3 * 64 * SFTF_PITCH * 2 + 3 * 64 * 4);      // two 64-channel layers: 32,256 B

// Hidden layer of one SFT layer for 16 pixels: cond fragments `ca` (m16 x k32) x W0 (64 outputs) -> LeakyReLU -> the A
// fragments of the two second GEMMs (scale branch: hidden 0..31, shift branch: hidden 32..63).  The accumulator fragment
// of two adjacent n8 blocks IS the A fragment of one k16 step (rows g / g+8, columns 2t..2t+1 / +8).
__device__ __forceinline__ void sft_hidden(const unsigned char* fw, const SftFrag& L, const uint32_t (&ca)[2][4], int g, int tq,
                                           uint32_t (&as)[2][4], uint32_t (&ah)[2][4]) {
    const __half* W0 = reinterpret_cast<const __half*>(fw + L.off_w0);
    const float* b0 = reinterpret_cast<const float*>(fw + L.off_b0);
#pragma unroll
    for (int j = 0; j < 8; ++j) {
        float c[4];
        c[0] = c[2] = b0[8 * j + 2 * tq]; c[1] = c[3] = b0[8 * j + 2 * tq + 1];
#pragma unroll
        for (int ks = 0; ks < 2; ++ks) {
            const __half* wr = W0 + (8 * j + g) * SFTF_PITCH + 16 * ks + 2 * tq;
            mma_16816(c, ca[ks], *reinterpret_cast<const uint32_t*>(wr), *reinterpret_cast<const uint32_t*>(wr + 8));
        }
#pragma unroll
        for (int e = 0; e < 4; ++e) c[e] = fmaxf(c[e], 0.2f * c[e]);
        uint32_t (&dst)[2][4] = (j < 4) ? as : ah;
        const int jj = j & 3;
        dst[jj >> 1][(jj & 1) * 2 + 0] = h2_sat(c[0], c[1]);          // row g
        dst[jj >> 1][(jj & 1) * 2 + 1] = h2_sat(c[2], c[3]);          // row g + 8
    }
}
// scale + 1 and shift of output channels 8j .. 8j+7 for the 16 pixels (accumulator fragment layout)
__device__ __forceinline__ void sft_scale_shift(const unsigned char* fw, const SftFrag& L, const uint32_t (&as)[2][4], const uint32_t (&ah)[2][4],
                                                int j, int g, int tq, float (&sc)[4], float (&sh)[4]) {
    const __half* W1s = reinterpret_cast<const __half*>(fw + L.off_w1s);
    const __half* W1h = reinterpret_cast<const __half*>(fw + L.off_w1h);
    const float* b1s = reinterpret_cast<const float*>(fw + L.off_b1s);
    const float* b1h = reinterpret_cast<const float*>(fw + L.off_b1h);
    sc[0] = sc[2] = b1s[8 * j + 2 * tq]; sc[1] = sc[3] = b1s[8 * j + 2 * tq + 1];
    sh[0] = sh[2] = b1h[8 * j + 2 * tq]; sh[1] = sh[3] = b1h[8 * j + 2 * tq + 1];
#pragma unroll
    for (int ks = 0; ks < 2; ++ks) {
        const __half* ws = W1s + (8 * j + g) * SFTF_PITCH + 16 * ks + 2 * tq;
        const __half* wh = W1h + (8 * j + g) * SFTF_PITCH + 16 * ks + 2 * tq;
        mma_16816(sc, as[ks], *reinterpret_cast<const uint32_t*>(ws), *reinterpret_cast<const uint32_t*>(ws + 8));
        mma_16816(sh, ah[ks], *reinterpret_cast<const uint32_t*>(wh), *reinterpret_cast<const uint32_t*>(wh + 8));
    }
}
// ---------------------------------------------------------------------------------------------
// conv3x3_ws_kernel<N>: every 3x3 convolution as an im2col-free implicit GEMM on Hopper warpgroup MMAs --
// ONE persistent CTA per SM, warp specialised, fed through a deep shared-memory ring:
//   warpgroup 2  producers: either one thread issuing TMA tensor copies of the (16+2)x(32+2) halo of a 16-channel
//                slice (two 8-channel planes; out-of-range coordinates are zero filled = the conv's padding) plus a
//                bulk copy of that slice's [N][16] weight tiles, or -- with nearest-x2 source addressing or without
//                tensor maps -- all 128 threads with cp.async, a stage published (mbarrier FULL) two stages behind
//                the issue point;
//   warpgroups 0, 1  consumers: each owns two of the tile's four 16x8-pixel M tiles (= four m64 halves) and issues
//                its wgmma.m64nNk16 straight from the ring -- the halo planes ARE the no-swizzle K-major operand layout
//                (core matrix = 8 horizontally adjacent pixels, SBO = halo row pitch, LBO = plane pitch), so the taps
//                are descriptors that differ only in their start address; the fp32 accumulators stay in registers for
//                the whole K loop, a stage is handed back (mbarrier EMPTY) as soon as the MMAs that read it retire,
//                and the epilogue (bias / LeakyReLU / residual / stores, or the fused SFT layers) runs on the
//                accumulator fragments in registers.
// Tiles (16 rows x 32 columns of output pixels) are dealt round-robin to the CTAs; dense-block concatenation is free
// (a conv reads channels [0,Cin) of the block's NHWC buffer and writes its growth channels behind them); "nearest x2
// then conv" runs in its sub-pixel form (run_conv_up2x).
// ---------------------------------------------------------------------------------------------
constexpr int WS_TM = 4;
constexpr int WS_TX = 8 * WS_TM, WS_HX = WS_TX + 2;            // 32 / 34
constexpr int WS_ROW = WS_HX * 16;                             // 544 B
constexpr int WS_PLANE = (SR_HY * WS_ROW + 127) / 128 * 128;   // 9856 B: 9792 B of pixels, padded so every plane is a 128-B aligned TMA destination
constexpr int WS_A_STAGE = (SR_CK / 8) * WS_PLANE;             // 19712 B
constexpr int WS_HALO = SR_HY * WS_HX * (SR_CK / 8);           // 1224 16-byte copies per stage
constexpr int WS_HALO_PER_THREAD = (WS_HALO + 127) / 128;      // 10
constexpr int WS_LAG = 2;
constexpr int WS_THREADS = 384;                                // warpgroups 0-1 MMA + epilogue, warpgroup 2 producers

template <int N> struct WsCfg {
    static constexpr int B_TAP = N * SR_CK * 2;
    static constexpr int B_STAGE = 9 * B_TAP;
    static constexpr int STAGE = WS_A_STAGE + B_STAGE;
    static constexpr int NST = (N >= 64) ? 5 : 6;
    static constexpr int SMEM = NST * STAGE + 512;              // + barriers (256 B) + bias (256 B)
};

// ---------------------------------------------------------------------------------------------
// Epilogue of one 16-pixel block with the following SFT layer(s) folded in (SRM_*_SFT* modes).  The 36 SFT layers of the
// decoder are 0.2 % of its FLOPs but cost a memory pass each as separate kernels; here they cost none.  Per 16 pixels a
// warp evaluates the layer's two small MLPs with mma.sync straight from registers -- cond row fragments (fp16, [P,32]) x
// W0 -> LeakyReLU -> re-used as A fragments -> W1s / W1h -- and the convolution's accumulator fragment has the SAME layout,
// so scale, shift and the value they modulate meet in registers with no shuffle.
// Rows of a thread: pixels (pyA, px) and (pyA + 1, px); channels 8j+2t, +1 of accumulator registers 4j .. 4j+3.
// ---------------------------------------------------------------------------------------------
template <int N>
__device__ __forceinline__ void epilogue_sft(const ConvParams& p, const unsigned char* fw, const float* sbias, const float (&acc)[N / 2],
                                             int pyA, int px, int lane) {
    constexpr int NB = N / 8;
    const int g = lane >> 2, tq = lane & 3;
    const SftFrag L1 = sft_frag_layout(p.sft_n);
    const SftFrag L2 = sft_frag_layout(64);
    const unsigned char* fw2 = fw + L1.total;
    const bool two = (N == 64) && p.mode == SRM_TRUNK_SFT2;
    const bool trunk = p.mode != SRM_STORE_F16_SFT;
    const bool inA = (pyA < p.y_hi) & (px < p.W), inB = (pyA + 1 < p.y_hi) & (px < p.W);
    const size_t pixA = (size_t)pyA * p.W + px, pixB = pixA + p.W;
    uint32_t ca[2][4];
    {
        const __half* cA = p.cond16 + (inA ? pixA : 0) * 32 + 2 * tq;
        const __half* cB = p.cond16 + (inB ? pixB : 0) * 32 + 2 * tq;
#pragma unroll
        for (int ks = 0; ks < 2; ++ks) {
            ca[ks][0] = __ldg(reinterpret_cast<const unsigned int*>(cA + 16 * ks));
            ca[ks][1] = __ldg(reinterpret_cast<const unsigned int*>(cB + 16 * ks));
            ca[ks][2] = __ldg(reinterpret_cast<const unsigned int*>(cA + 16 * ks + 8));
            ca[ks][3] = __ldg(reinterpret_cast<const unsigned int*>(cB + 16 * ks + 8));
        }
    }
    // residual rows (fp32 trunk, and the RRDB input for the block tail) travel through a rolling window of PF channel
    // blocks: block j+PF is requested when block j is consumed -- enough bytes in flight to cover the memory latency
    // without holding the whole 256-byte rows in registers
    constexpr int PF = (NB < 4) ? NB : 4;
    float2 rA[PF], rB[PF], xA[PF], xB[PF];
    auto load_res = [&](int j, int slot) {
        rA[slot] = rB[slot] = make_float2(0.f, 0.f);
        if (p.add_f) {
            if (inA) rA[slot] = __ldg(reinterpret_cast<const float2*>(p.add_f + pixA * 64 + 8 * j + 2 * tq));
            if (inB) rB[slot] = __ldg(reinterpret_cast<const float2*>(p.add_f + pixB * 64 + 8 * j + 2 * tq));
        }
        if (two) {
            xA[slot] = xB[slot] = make_float2(0.f, 0.f);
            if (inA) xA[slot] = __ldg(reinterpret_cast<const float2*>(p.add_f2 + pixA * 64 + 8 * j + 2 * tq));
            if (inB) xB[slot] = __ldg(reinterpret_cast<const float2*>(p.add_f2 + pixB * 64 + 8 * j + 2 * tq));
        }
    };
    if (trunk) {
#pragma unroll
        for (int j = 0; j < PF; ++j) load_res(j, j);
    }
    uint32_t as[2][4], ah[2][4], as2[2][4], ah2[2][4];
    sft_hidden(fw, L1, ca, g, tq, as, ah);
    if (two) sft_hidden(fw2, L2, ca, g, tq, as2, ah2);
#pragma unroll
    for (int j = 0; j < NB; ++j) {
        const int sl = j % PF;
        float sc[4], sh[4];
        sft_scale_shift(fw, L1, as, ah, j, g, tq, sc, sh);
        const int ch = 8 * j + 2 * tq;
        float v[4];
#pragma unroll
        for (int e = 0; e < 4; ++e) v[e] = acc[4 * j + e] + sbias[ch + (e & 1)];
        if (!trunk) {                       // SRM_STORE_F16_SFT
#pragma unroll
            for (int e = 0; e < 4; ++e) { const float a = p.lrelu > 0.f ? fmaxf(v[e], p.lrelu * v[e]) : v[e]; v[e] = fmaf(a, sc[e], sh[e]); }
            if (inA) *reinterpret_cast<uint32_t*>(p.dst_h + pixA * p.dst_cstride + p.dst_c0 + ch) = h2_sat(v[0], v[1]);
            if (inB) *reinterpret_cast<uint32_t*>(p.dst_h + pixB * p.dst_cstride + p.dst_c0 + ch) = h2_sat(v[2], v[3]);
            continue;
        }
        float t[4] = {fmaf(v[0], p.scale, rA[sl].x), fmaf(v[1], p.scale, rA[sl].y), fmaf(v[2], p.scale, rB[sl].x), fmaf(v[3], p.scale, rB[sl].y)};
        const float2 xa = xA[sl], xb = xB[sl];
        if (j + PF < NB) load_res(j + PF, sl);
        if (!two) {                         // SRM_TRUNK_SFT
            if (inA) {
                *reinterpret_cast<float2*>(p.dst_f + pixA * 64 + ch) = make_float2(t[0], t[1]);
                if (p.dst_f2) *reinterpret_cast<float2*>(p.dst_f2 + pixA * 64 + ch) = make_float2(t[0], t[1]);
            }
            if (inB) {
                *reinterpret_cast<float2*>(p.dst_f + pixB * 64 + ch) = make_float2(t[2], t[3]);
                if (p.dst_f2) *reinterpret_cast<float2*>(p.dst_f2 + pixB * 64 + ch) = make_float2(t[2], t[3]);
            }
#pragma unroll
            for (int e = 0; e < 4; ++e) t[e] = fmaf(t[e], sc[e], sh[e]);
        } else {                            // SRM_TRUNK_SFT2: u = sft(t) * scale2 + x_in -> trunk; then the next layer on u
            t[0] = fmaf(fmaf(t[0], sc[0], sh[0]), p.scale2, xa.x); t[1] = fmaf(fmaf(t[1], sc[1], sh[1]), p.scale2, xa.y);
            t[2] = fmaf(fmaf(t[2], sc[2], sh[2]), p.scale2, xb.x); t[3] = fmaf(fmaf(t[3], sc[3], sh[3]), p.scale2, xb.y);
            if (inA) *reinterpret_cast<float2*>(p.dst_f + pixA * 64 + ch) = make_float2(t[0], t[1]);
            if (inB) *reinterpret_cast<float2*>(p.dst_f + pixB * 64 + ch) = make_float2(t[2], t[3]);
            sft_scale_shift(fw2, L2, as2, ah2, j, g, tq, sc, sh);
#pragma unroll
            for (int e = 0; e < 4; ++e) t[e] = fmaf(t[e], sc[e], sh[e]);
        }
        if (inA) *reinterpret_cast<uint32_t*>(p.dst_h2 + pixA * p.dst2_cstride + p.dst2_c0 + ch) = h2_sat(t[0], t[1]);
        if (inB) *reinterpret_cast<uint32_t*>(p.dst_h2 + pixB * p.dst2_cstride + p.dst2_c0 + ch) = h2_sat(t[2], t[3]);
    }
}

// Epilogue of one 16-pixel block for the plain modes: pixels (py, px) and (py + 1, px) of the iteration grid, channels
// 8j+2t, +1 of accumulator registers 4j .. 4j+3.  SPLIT: the kernel honours ConvParams::split (conv3x3_ws_kernel only).
template <int N, bool SPLIT>
__device__ __forceinline__ void epilogue_plain(const ConvParams& p, const float* sbias, const float (&acc)[N / 2], int pyA, int px, int tq) {
#pragma unroll
    for (int r = 0; r < 2; ++r) {
        const int py = pyA + r;
        if (!((py < p.y_hi) & (px < p.W))) continue;
        const int oy = py * p.out_s + p.out_oy, ox = px * p.out_s + p.out_ox;
        const size_t pix = (size_t)oy * ((size_t)p.W * p.out_s) + (size_t)ox;
        const bool crop = oy >= p.crop_y0 && oy < p.crop_y1 && ox >= p.crop_x0 && ox < p.crop_x1;
#pragma unroll
        for (int j = 0; j < N / 8; ++j) {
            const int ch = 8 * j + 2 * tq;
            float o0 = acc[4 * j + 2 * r] + sbias[ch], o1 = acc[4 * j + 2 * r + 1] + sbias[ch + 1];
            if (p.mode == SRM_STORE_F16) {
                if (p.lrelu > 0.f) { o0 = o0 > 0.f ? o0 : o0 * p.lrelu; o1 = o1 > 0.f ? o1 : o1 * p.lrelu; }
                else if (p.relu) { o0 = fmaxf(o0, 0.f); o1 = fmaxf(o1, 0.f); }
                __half* d = p.dst_h + pix * p.dst_cstride + p.dst_c0 + ch;
                const uint32_t hi = h2_sat(o0, o1);
                *reinterpret_cast<uint32_t*>(d) = hi;
                if (SPLIT && p.split) {
                    const float2 f = __half22float2(*reinterpret_cast<const __half2*>(&hi));
                    *reinterpret_cast<uint32_t*>(d + p.split) = h2_sat(o0 - f.x, o1 - f.y);
                    *reinterpret_cast<uint32_t*>(d + 2 * p.split) = hi;
                }
            } else if (p.mode == SRM_TRUNK) {
                const float2 a = __ldg(reinterpret_cast<const float2*>(p.add_f + pix * 64 + ch));
                *reinterpret_cast<float2*>(p.dst_f + pix * 64 + ch) = make_float2(o0 * p.scale + a.x, o1 * p.scale + a.y);
            } else if (p.mode == SRM_ADD_STORE_F16) {
                const float2 a = __ldg(reinterpret_cast<const float2*>(p.add_f + pix * 64 + ch));
                *reinterpret_cast<uint32_t*>(p.dst_h + pix * p.dst_cstride + p.dst_c0 + ch) = h2_sat(o0 + a.x, o1 + a.y);
            } else if (p.mode == SRM_STORE_F32F16) {
                *reinterpret_cast<float2*>(p.dst_f + pix * 64 + ch) = make_float2(o0, o1);
                if (p.dst_f2) *reinterpret_cast<float2*>(p.dst_f2 + pix * 64 + ch) = make_float2(o0, o1);
            } else if (crop) {              // SRM_OUT_NCHW
                const long long o = (long long)(oy - p.crop_y0) * p.out_rs + (ox - p.crop_x0);
                if (ch < p.n_valid) sr_store_out(p, (long long)ch * p.out_ps + o, o0);
                if (ch + 1 < p.n_valid) sr_store_out(p, (long long)(ch + 1) * p.out_ps + o, o1);
            }
        }
    }
}

template <int N>
__global__ void __launch_bounds__(WS_THREADS, 1) conv3x3_ws_kernel(const __grid_constant__ ConvParams p, const __grid_constant__ CUtensorMap tmap) {
    using C = WsCfg<N>;
    extern __shared__ __align__(1024) unsigned char smem[];
    uint64_t* full = reinterpret_cast<uint64_t*>(smem + C::NST * C::STAGE);     // [NST] count 1 + tx (TMA) or 128 (cp.async)
    uint64_t* empty = full + C::NST;                                             // [NST] count 8: lane 0 of every consumer warp
    float* sbias = reinterpret_cast<float*>(smem + C::NST * C::STAGE + 256);    // [64]
    unsigned char* sftw_s = smem + C::NST * C::STAGE + 512;                      // SFT operand block(s) of the fused epilogue modes
    const int tid = threadIdx.x, warp = tid >> 5, wg = tid >> 7;
    if (tid < 64) sbias[tid] = p.bias[tid];
    if (p.mode >= SRM_STORE_F16_SFT) {                                           // constants: may be staged before the PDL wait
        const int n1 = sft_frag_layout(p.sft_n).total;
        for (int i = tid; i < n1 / 16; i += WS_THREADS) reinterpret_cast<uint4*>(sftw_s)[i] = __ldg(reinterpret_cast<const uint4*>(p.sftw) + i);
        if (p.mode == SRM_TRUNK_SFT2) {
            const int n2 = sft_frag_layout(64).total;
            for (int i = tid; i < n2 / 16; i += WS_THREADS) reinterpret_cast<uint4*>(sftw_s + n1)[i] = __ldg(reinterpret_cast<const uint4*>(p.sftw2) + i);
        }
    }
    const int tiles_x = (p.W + WS_TX - 1) / WS_TX, tiles_y = (p.y_hi - p.y_lo + SR_TY - 1) / SR_TY;
    const int n_tiles = tiles_x * tiles_y;
    const int nchunks = p.cin / SR_CK;

    if (tid == 0) {
        for (int i = 0; i < C::NST; ++i) { mbar_init(full + i, p.use_tma ? 1 : 128); mbar_init(empty + i, 8); }
        mbar_init_fence();
    }
    __syncthreads();
    pdl_wait_and_release();

    if (wg == 2) {
        setmaxnreg_dec<56>();
        if (p.use_tma) {
            // ------------------------------ producer (TMA): one thread, three bulk copies per stage ------------------------------
            // The activation buffer is a 3-D tensor (channel, x, y); a box of (8 channels, 34, 18) lands in shared
            // memory as [hy][hx] x 16 B = one plane of the operand layout.
            if (tid == 256) {
                unsigned g = 0;
                const uint64_t tm = reinterpret_cast<uint64_t>(&tmap);
                for (int tile = blockIdx.x; tile < n_tiles; tile += gridDim.x) {
                    const int ty = tile / tiles_x, tx = tile - ty * tiles_x;
                    const int y0 = p.y_lo + ty * SR_TY - 1, x0 = tx * WS_TX - 1;
                    for (int c = 0; c < nchunks; ++c, ++g) {
                        const unsigned slot = g % C::NST;
                        if (g >= (unsigned)C::NST) mbar_wait(empty + slot, ((g / C::NST) - 1) & 1);
                        uint64_t* bar = full + slot;
                        unsigned char* A = smem + slot * C::STAGE;
                        const uint32_t bbytes = (uint32_t)p.ntaps * C::B_TAP;
                        mbar_arrive_expect_tx(bar, (uint32_t)((SR_CK / 8) * SR_HY * WS_ROW) + bbytes);
#pragma unroll
                        for (int pl = 0; pl < SR_CK / 8; ++pl) tensor_g2s_3d(A + pl * WS_PLANE, tm, bar, c * SR_CK + pl * 8, x0, y0);
                        bulk_g2s(A + WS_A_STAGE, p.wpack + (size_t)c * bbytes, bbytes, bar);
                    }
                }
            }
        } else {
            // ------------------------------ producers (cp.async; nearest-x2 source addressing) ------------------------------
            const int pt = tid - 256;
            const int sW = p.upsample ? (p.W >> 1) : p.W;
            unsigned g = 0;
            auto publish = [&](unsigned gi) {
                fence_proxy_async();
                mbar_arrive(full + gi % C::NST);
            };
            for (int tile = blockIdx.x; tile < n_tiles; tile += gridDim.x) {
                const int ty = tile / tiles_x, tx = tile - ty * tiles_x;
                const int y0 = p.y_lo + ty * SR_TY, x0 = tx * WS_TX;
                for (int c = 0; c < nchunks; ++c, ++g) {
                    const unsigned slot = g % C::NST;
                    if (g >= (unsigned)C::NST) mbar_wait(empty + slot, ((g / C::NST) - 1) & 1);
                    unsigned char* A = smem + slot * C::STAGE;
#pragma unroll 1
                    for (int j = 0; j < WS_HALO_PER_THREAD; ++j) {
                        const int i = pt + j * 128;
                        if (i < WS_HALO) {
                            const int plane = i & 1, pix = i >> 1;
                            const int hy = pix / WS_HX, hx = pix - hy * WS_HX;
                            const int gy = y0 - 1 + hy, gx = x0 - 1 + hx;
                            const bool in = (gy >= 0) & (gy < p.H) & (gx >= 0) & (gx < p.W);
                            const int sy = p.upsample ? (gy >> 1) : gy, sx = p.upsample ? (gx >> 1) : gx;
                            const __half* src = in ? p.src + ((long long)sy * sW + sx) * p.src_cstride + p.src_c0 + plane * 8 + c * SR_CK : p.src;
                            cp_async16(A + plane * WS_PLANE + hy * WS_ROW + hx * 16, src, in ? 16 : 0);
                        }
                    }
                    const int bbytes = p.ntaps * C::B_TAP;
                    const unsigned char* wsrc = p.wpack + (size_t)c * bbytes;
                    unsigned char* B = A + WS_A_STAGE;
                    for (int i = pt; i < bbytes / 16; i += 128) cp_async16(B + i * 16, wsrc + i * 16, 16);
                    cp_async_commit();
                    if (g >= (unsigned)WS_LAG) {
                        cp_async_wait<WS_LAG>();
                        publish(g - WS_LAG);
                    }
                }
            }
            // drain: the last WS_LAG stages
            if (g >= 2) { cp_async_wait<1>(); publish(g - 2); }
            if (g >= 1) { cp_async_wait<0>(); publish(g - 1); }
        }
    } else {
        // ------------------------------ consumers: MMAs + epilogue of M tiles 2*wg, 2*wg+1 ------------------------------
        setmaxnreg_inc<224>();
        const int lane = tid & 31, wq = warp & 3, g8 = lane >> 2, tq = lane & 3;
        const uint32_t smem_s = smem_u32(smem);
        unsigned g = 0;
        for (int tile = blockIdx.x; tile < n_tiles; tile += gridDim.x) {
            const int ty = tile / tiles_x, tx = tile - ty * tiles_x;
            const int y0 = p.y_lo + ty * SR_TY, x0 = tx * WS_TX;
            float acc[2][2][N / 2];                                  // [M tile of this group][m64 half][fragment]
            for (int c = 0; c < nchunks; ++c, ++g) {
                const unsigned slot = g % C::NST;
                mbar_wait(full + slot, (g / C::NST) & 1);
                const uint32_t a0 = smem_s + slot * C::STAGE, b0 = a0 + WS_A_STAGE;
                wg_fence();
#pragma unroll
                for (int t = 0; t < 9; ++t) {
                    if (t < p.ntaps) {
                        const uint32_t aoff = (uint32_t)(p.tap_dy[t] * WS_ROW + p.tap_dx[t] * 16);
                        const uint64_t bd = wg_desc(b0 + t * C::B_TAP, 128, (SR_CK / 8) * 128);
#pragma unroll
                        for (int ml = 0; ml < 2; ++ml)
#pragma unroll
                            for (int mh = 0; mh < 2; ++mh)
                                wgmma_ss(acc[ml][mh], wg_desc(a0 + aoff + (2 * wg + ml) * 8 * 16 + mh * 8 * WS_ROW, WS_PLANE, WS_ROW), bd,
                                         (c | t) != 0);
                    }
                }
                wg_commit();
                // the previous stage's MMAs have retired once at most this stage's group is pending
                wg_wait<1>();
                if (c > 0 && lane == 0) mbar_arrive(empty + (g - 1) % C::NST);
            }
            wg_wait<0>();
            if (lane == 0) mbar_arrive(empty + (g - 1) % C::NST);
#pragma unroll
            for (int ml = 0; ml < 2; ++ml)
#pragma unroll
                for (int mh = 0; mh < 2; ++mh) {
                    wg_fence_acc(acc[ml][mh]);
                    // rows 16*wq + g8 (+8) of m64 half mh = image rows 8*mh + 2*wq (+1), column g8 of the 16x8 M tile
                    const int pyA = y0 + 8 * mh + 2 * wq, px = x0 + (2 * wg + ml) * 8 + g8;
                    if (p.mode >= SRM_STORE_F16_SFT) {
                        if constexpr (N >= 32) epilogue_sft<N>(p, sftw_s, sbias, acc[ml][mh], pyA, px, lane);
                    } else {
                        epilogue_plain<N, true>(p, sbias, acc[ml][mh], pyA, px, tq);
                    }
                }
        }
    }
}

// ---------------------------------------------------------------------------------------------
// conv3x3_k64_kernel<N>: the 64-input-channel convolutions (conv_body, conv_up1/2 phases, conv_hr, conv_last -- every
// layer after the dense blocks, i.e. all the high-resolution work) with 128-BYTE shared-memory rows.  conv3x3_ws_kernel
// moves a 16-channel slice as 612 rows of 16 B per plane; here a pixel's 64 channels are ONE 128-byte row in the
// SWIZZLE_128B K-major layout: the whole (16+2) x (24+2) halo of a tile is a single TMA tensor copy of 468 rows, the
// taps are wgmma descriptors that differ only in their start address (+ (dy*26 + dx) * 128 B), a k16 step is +32 B
// inside the row, and -- because Cin = 64 is a single K slice -- the layer's weights ([tap][n][64] fp16, 74 KB for
// N = 64) are loaded ONCE per persistent CTA and stay resident.  Roles as in conv3x3_ws_kernel: warpgroup 2 is the TMA
// producer, warpgroups 0 and 1 issue the MMAs of three of the tile's six m64 halves each and run their epilogues.
// ---------------------------------------------------------------------------------------------
constexpr int K64_TM = 3;                                       // 16 x 24 output pixels per tile
constexpr int K64_TX = 8 * K64_TM, K64_HX = K64_TX + 2;         // 24 / 26
constexpr int K64_ROWB = 128;                                   // bytes per pixel row (64 fp16)
constexpr int K64_A_BYTES = SR_HY * K64_HX * K64_ROWB;          // 59904: what one TMA copy delivers
constexpr int K64_A_STAGE = (K64_A_BYTES + 1023) / 1024 * 1024; // 60416
constexpr int K64_THREADS = 384;

template <int N> struct K64Cfg {
    static constexpr int B_TAP = N * K64_ROWB;                   // 8192 / 2048 (1024-aligned)
    static constexpr int B_BYTES = 9 * B_TAP;
    static constexpr int NST = (N >= 64) ? 2 : 3;
    static constexpr int SMEM = 1024 + B_BYTES + NST * K64_A_STAGE + 512;   // alignment slack + B + ring + barriers/bias
};

// SWIZZLE_128B K-major operand: SBO = distance between 8-row groups, LBO unused (1), layout type 1 = 128-byte swizzle.
// The swizzle is a function of the shared-memory address bits, as the TMA copy wrote it, so start addresses that are
// whole 128-byte rows (taps) or 32-byte k16 steps off a 1024-byte boundary address the same data.
__device__ __forceinline__ uint64_t k64_desc(uint32_t saddr, uint32_t sbo_bytes) {
    return (uint64_t)((saddr >> 4) & 0x3FFF) | ((uint64_t)1 << 16) | ((uint64_t)((sbo_bytes >> 4) & 0x3FFF) << 32) | (1ull << 62);
}

template <int N>
__global__ void __launch_bounds__(K64_THREADS, 1) conv3x3_k64_kernel(const __grid_constant__ ConvParams p, const __grid_constant__ CUtensorMap tmap_a,
                                                                      const __grid_constant__ CUtensorMap tmap_b) {
    using C = K64Cfg<N>;
    extern __shared__ unsigned char smem_raw[];
    unsigned char* smem = reinterpret_cast<unsigned char*>(((uintptr_t)smem_raw + 1023) & ~(uintptr_t)1023);
    unsigned char* Bw = smem;                                                    // [9][N][128 B] swizzled
    unsigned char* Ar = smem + C::B_BYTES;                                       // ring of NST halo stages
    uint64_t* full = reinterpret_cast<uint64_t*>(Ar + C::NST * K64_A_STAGE);    // [NST] count 1 + tx
    uint64_t* empty = full + C::NST;                                             // [NST] count 8: lane 0 of every consumer warp
    uint64_t* wbar = empty + C::NST;                                             // weights landed
    float* sbias = reinterpret_cast<float*>(Ar + C::NST * K64_A_STAGE + 256);   // [64]
    const int tid = threadIdx.x, warp = tid >> 5, wg = tid >> 7;
    if (tid < 64) sbias[tid] = p.bias[tid];
    const int tiles_x = (p.W + K64_TX - 1) / K64_TX, tiles_y = (p.y_hi - p.y_lo + SR_TY - 1) / SR_TY;
    const int n_tiles = tiles_x * tiles_y;

    if (tid == 0) {
        for (int i = 0; i < C::NST; ++i) { mbar_init(full + i, 1); mbar_init(empty + i, 8); }
        mbar_init(wbar, 1);
        mbar_init_fence();
    }
    __syncthreads();

    if (wg == 2) {
        // ------------------------------ producer: weights once, then one tensor copy per tile ------------------------------
        if (tid == 256) {
            const uint64_t ta = reinterpret_cast<uint64_t>(&tmap_a), tb = reinterpret_cast<uint64_t>(&tmap_b);
            mbar_arrive_expect_tx(wbar, (uint32_t)p.ntaps * C::B_TAP);
            for (int t = 0; t < p.ntaps; ++t) tensor_g2s_2d(Bw + t * C::B_TAP, tb, wbar, 0, t * N);
            pdl_wait_and_release();                               // the weights above are constants; the activations are not
            unsigned g = 0;
            for (int tile = blockIdx.x; tile < n_tiles; tile += gridDim.x, ++g) {
                const int ty = tile / tiles_x, tx = tile - ty * tiles_x;
                const unsigned slot = g % C::NST;
                if (g >= (unsigned)C::NST) mbar_wait(empty + slot, ((g / C::NST) - 1) & 1);
                mbar_arrive_expect_tx(full + slot, (uint32_t)K64_A_BYTES);
                tensor_g2s_3d(Ar + slot * K64_A_STAGE, ta, full + slot, 0, tx * K64_TX - 1, p.y_lo + ty * SR_TY - 1);
            }
        }
    } else {
        // ------------------------------ consumers: m64 halves 3*wg .. 3*wg+2 (M tile j/2, image rows 8*(j%2) ..) ------------------------------
        pdl_wait_and_release();                                   // residual reads / output writes touch earlier kernels' buffers
        const int lane = tid & 31, wq = warp & 3, g8 = lane >> 2, tq = lane & 3;
        mbar_wait(wbar, 0);
        const uint32_t bw = smem_u32(Bw);
        unsigned g = 0;
        for (int tile = blockIdx.x; tile < n_tiles; tile += gridDim.x, ++g) {
            const int ty = tile / tiles_x, tx = tile - ty * tiles_x;
            const int y0 = p.y_lo + ty * SR_TY, x0 = tx * K64_TX;
            const unsigned slot = g % C::NST;
            mbar_wait(full + slot, (g / C::NST) & 1);
            const uint32_t a0 = smem_u32(Ar + slot * K64_A_STAGE);
            float acc[3][N / 2];
            wg_fence();
#pragma unroll
            for (int t = 0; t < 9; ++t) {
                if (t < p.ntaps) {
                    const uint32_t aoff = (uint32_t)((p.tap_dy[t] * K64_HX + p.tap_dx[t]) * K64_ROWB);
#pragma unroll
                    for (int ks = 0; ks < 4; ++ks) {
                        const uint64_t bd = k64_desc(bw + t * C::B_TAP + ks * 32, 1024);
#pragma unroll
                        for (int h = 0; h < 3; ++h) {
                            const int j = 3 * wg + h, m = j >> 1, mh = j & 1;
                            wgmma_ss(acc[h], k64_desc(a0 + aoff + (8 * mh * K64_HX + 8 * m) * K64_ROWB + ks * 32, K64_HX * K64_ROWB), bd,
                                     (t | ks) != 0);
                        }
                    }
                }
            }
            wg_commit();
            wg_wait<0>();
            if (lane == 0) mbar_arrive(empty + slot);
#pragma unroll
            for (int h = 0; h < 3; ++h) {
                wg_fence_acc(acc[h]);
                const int j = 3 * wg + h, m = j >> 1, mh = j & 1;
                epilogue_plain<N, false>(p, sbias, acc[h], y0 + 8 * mh + 2 * wq, x0 + 8 * m + g8, tq);
            }
        }
    }
}

// ---------------------------------------------------------------------------------------------
// SFT layer: scale = C1s(lrelu(C0s(cond))), shift = C1h(lrelu(C0h(cond))), y = x*(scale+1)+shift
// ---------------------------------------------------------------------------------------------
struct SftParams {
    const float* cond;               // [P,32] fp32
    const float* w;                  // packed: s0 [32][32], s0b[32], h0 [32][32], h0b[32], s1 [COUT][32], s1b, h1 [COUT][32], h1b
    const float* x_f; const __half* x_h; int xh_cstride, xh_c0;     // input: fp32 [P,64] or fp16 channel range
    __half* dst_h; int dst_cstride, dst_c0;                          // fp16 output (or nullptr)
    float* dst_f; const float* res_f; float res_scale;               // fp32 output: y*res_scale + res_f (RRDB tail) when dst_f != nullptr
    long long P;                                                     // pixels processed ...
    long long p0;                                                    // ... starting at this pixel (row window of a decoder unit)
};

template <int COUT>
__global__ void __launch_bounds__(128) sft_kernel(const __grid_constant__ SftParams p) {
    constexpr int NW = 2 * (32 * 32 + 32) + 2 * (COUT * 32 + COUT);
    extern __shared__ __align__(16) float sw[];
    for (int i = threadIdx.x; i < NW; i += blockDim.x) sw[i] = __ldg(p.w + i);
    __syncthreads();
    const float* s0 = sw;             const float* s0b = s0 + 1024;
    const float* h0 = s0b + 32;       const float* h0b = h0 + 1024;
    const float* s1 = h0b + 32;       const float* s1b = s1 + COUT * 32;
    const float* h1 = s1b + COUT;     const float* h1b = h1 + COUT * 32;
    const long long lp = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (lp >= p.P) return;
    const long long pix = p.p0 + lp;
    float c[32], ts[32], th[32];
    const float4* cp = reinterpret_cast<const float4*>(p.cond + pix * 32);
#pragma unroll
    for (int q = 0; q < 8; ++q) { const float4 v = __ldg(cp + q); c[4 * q] = v.x; c[4 * q + 1] = v.y; c[4 * q + 2] = v.z; c[4 * q + 3] = v.w; }
#pragma unroll 4
    for (int o = 0; o < 32; ++o) {
        float a = s0b[o], b = h0b[o];
#pragma unroll
        for (int k = 0; k < 32; ++k) { a = fmaf(s0[o * 32 + k], c[k], a); b = fmaf(h0[o * 32 + k], c[k], b); }
        ts[o] = a > 0.f ? a : 0.2f * a;
        th[o] = b > 0.f ? b : 0.2f * b;
    }
#pragma unroll 1
    for (int o0 = 0; o0 < COUT; o0 += 8) {
        float y[8];
#pragma unroll
        for (int j = 0; j < 8; ++j) {
            const int o = o0 + j;
            float sc = s1b[o], sh = h1b[o];
#pragma unroll
            for (int k = 0; k < 32; ++k) { sc = fmaf(s1[o * 32 + k], ts[k], sc); sh = fmaf(h1[o * 32 + k], th[k], sh); }
            float x;
            if (p.x_f) x = __ldg(p.x_f + pix * 64 + o);
            else x = __half2float(p.x_h[pix * p.xh_cstride + p.xh_c0 + o]);
            y[j] = x * (sc + 1.f) + sh;
        }
        if (p.dst_f) {
#pragma unroll
            for (int j = 0; j < 8; ++j) p.dst_f[pix * 64 + o0 + j] = y[j] * p.res_scale + __ldg(p.res_f + pix * 64 + o0 + j);
        } else {
            uint32_t h[4];
#pragma unroll
            for (int j = 0; j < 4; ++j) h[j] = h2_sat(y[2 * j], y[2 * j + 1]);
            *reinterpret_cast<uint4*>(p.dst_h + pix * p.dst_cstride + p.dst_c0 + o0) = *reinterpret_cast<uint4*>(h);
        }
    }
}


// ---------------------------------------------------------------------------------------------
// SFT layer as its own pass (K4_SR_FUSE_SFT=0): the same fragment-level evaluation as the fused epilogues (sft_hidden,
// sft_scale_shift), with the modulated value read from memory.  A warp takes 16 pixels at a time: rows g and g+8 of
// the mma.sync fragments, channels 8j+2t, +1.  The layer's operand block (sft_frag_layout) is staged once per CTA.
// ---------------------------------------------------------------------------------------------
template <int COUT>
__global__ void __launch_bounds__(128) sft_mma_kernel(const __grid_constant__ SftParams p, const unsigned char* __restrict__ frag) {
    extern __shared__ __align__(16) unsigned char fw[];
    const SftFrag L = sft_frag_layout(COUT);
    for (int i = threadIdx.x; i < L.total / 16; i += blockDim.x) reinterpret_cast<uint4*>(fw)[i] = __ldg(reinterpret_cast<const uint4*>(frag) + i);
    __syncthreads();
    pdl_wait_and_release();
    const int lane = threadIdx.x & 31, g = lane >> 2, tq = lane & 3;
    const long long nblk = (p.P + 15) / 16;
    for (long long blk = (long long)blockIdx.x * 4 + (threadIdx.x >> 5); blk < nblk; blk += (long long)gridDim.x * 4) {
        const long long iA = blk * 16 + g, iB = iA + 8;
        const bool inA = iA < p.P, inB = iB < p.P;
        const long long pixA = p.p0 + (inA ? iA : 0), pixB = p.p0 + (inB ? iB : 0);
        uint32_t ca[2][4];
#pragma unroll
        for (int ks = 0; ks < 2; ++ks) {
            const float2 a0 = __ldg(reinterpret_cast<const float2*>(p.cond + pixA * 32 + 16 * ks + 2 * tq));
            const float2 b0 = __ldg(reinterpret_cast<const float2*>(p.cond + pixB * 32 + 16 * ks + 2 * tq));
            const float2 a1 = __ldg(reinterpret_cast<const float2*>(p.cond + pixA * 32 + 16 * ks + 8 + 2 * tq));
            const float2 b1 = __ldg(reinterpret_cast<const float2*>(p.cond + pixB * 32 + 16 * ks + 8 + 2 * tq));
            ca[ks][0] = h2_sat(a0.x, a0.y); ca[ks][1] = h2_sat(b0.x, b0.y);
            ca[ks][2] = h2_sat(a1.x, a1.y); ca[ks][3] = h2_sat(b1.x, b1.y);
        }
        uint32_t as[2][4], ah[2][4];
        sft_hidden(fw, L, ca, g, tq, as, ah);
#pragma unroll 2
        for (int j = 0; j < COUT / 8; ++j) {
            const int ch = 8 * j + 2 * tq;
            float sc[4], sh[4];
            sft_scale_shift(fw, L, as, ah, j, g, tq, sc, sh);
            float x[4];
            if (p.x_f) {
                const float2 xa = __ldg(reinterpret_cast<const float2*>(p.x_f + pixA * 64 + ch));
                const float2 xb = __ldg(reinterpret_cast<const float2*>(p.x_f + pixB * 64 + ch));
                x[0] = xa.x; x[1] = xa.y; x[2] = xb.x; x[3] = xb.y;
            } else {
                const float2 xa = __half22float2(*reinterpret_cast<const __half2*>(p.x_h + pixA * p.xh_cstride + p.xh_c0 + ch));
                const float2 xb = __half22float2(*reinterpret_cast<const __half2*>(p.x_h + pixB * p.xh_cstride + p.xh_c0 + ch));
                x[0] = xa.x; x[1] = xa.y; x[2] = xb.x; x[3] = xb.y;
            }
            float y[4];
#pragma unroll
            for (int e = 0; e < 4; ++e) y[e] = fmaf(x[e], sc[e], sh[e]);       // sc already holds scale + 1
            if (p.dst_f) {
                if (inA) {
                    const float2 r = __ldg(reinterpret_cast<const float2*>(p.res_f + pixA * 64 + ch));
                    *reinterpret_cast<float2*>(p.dst_f + pixA * 64 + ch) = make_float2(y[0] * p.res_scale + r.x, y[1] * p.res_scale + r.y);
                }
                if (inB) {
                    const float2 r = __ldg(reinterpret_cast<const float2*>(p.res_f + pixB * 64 + ch));
                    *reinterpret_cast<float2*>(p.dst_f + pixB * 64 + ch) = make_float2(y[2] * p.res_scale + r.x, y[3] * p.res_scale + r.y);
                }
            } else {
                if (inA) *reinterpret_cast<uint32_t*>(p.dst_h + pixA * p.dst_cstride + p.dst_c0 + ch) = h2_sat(y[0], y[1]);
                if (inB) *reinterpret_cast<uint32_t*>(p.dst_h + pixB * p.dst_cstride + p.dst_c0 + ch) = h2_sat(y[2], y[3]);
            }
        }
    }
}

// fp32 SFT weights (sft_kernel packing order) -> fragment-ordered block of the fused epilogues (sft_frag_layout)
__global__ void pack_sft_frag_kernel(const float* __restrict__ w, unsigned char* __restrict__ dst, int cout) {
    const SftFrag L = sft_frag_layout(cout);
    const float* s0 = w; const float* s0b = s0 + 1024; const float* h0 = s0b + 32; const float* h0b = h0 + 1024;
    const float* s1 = h0b + 32; const float* s1b = s1 + cout * 32; const float* h1 = s1b + cout; const float* h1b = h1 + cout * 32;
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i < 64 * 32) {
        const int n = i >> 5, k = i & 31;
        reinterpret_cast<__half*>(dst + L.off_w0)[n * SFTF_PITCH + k] = __float2half_rn(n < 32 ? s0[n * 32 + k] : h0[(n - 32) * 32 + k]);
    }
    if (i < cout * 32) {
        const int n = i >> 5, k = i & 31;
        reinterpret_cast<__half*>(dst + L.off_w1s)[n * SFTF_PITCH + k] = __float2half_rn(s1[n * 32 + k]);
        reinterpret_cast<__half*>(dst + L.off_w1h)[n * SFTF_PITCH + k] = __float2half_rn(h1[n * 32 + k]);
    }
    if (i < 64) reinterpret_cast<float*>(dst + L.off_b0)[i] = i < 32 ? s0b[i] : h0b[i - 32];
    if (i < cout) { reinterpret_cast<float*>(dst + L.off_b1s)[i] = s1b[i] + 1.f; reinterpret_cast<float*>(dst + L.off_b1h)[i] = h1b[i]; }
}

// CondNet: conv3x3(num_cond->64) lrelu, 1x1 64->64 lrelu, 1x1 64->64 lrelu, 1x1 64->32   (lib/sr_esrnet.py:440-444)
// cond_in: planar fp32 [nc][H][W].  w: c0 [64][nc][9], b0[64], c2 [64][64], b2, c4 [64][64], b4, c6 [32][64], b6
struct CondParams { const float* cond_in; const float* w; float* cond_out; int H, W; int y_lo, y_hi; __half* cond16; int nc; };

// WIDE (nc > 1, the view-conditioned decoder): layer 0 runs channel by channel with its weights read from global memory
// (64 x nc x 9 floats, 147 KB at nc = 64); shared memory holds the 1x1 layers and every bias at the offsets of nc = 1.
template <bool WIDE>
__global__ void __launch_bounds__(128) condnet_kernel(const __grid_constant__ CondParams p) {
    constexpr int NW = 64 * 9 + 64 + 2 * (64 * 64 + 64) + 32 * 64 + 32;
    extern __shared__ __align__(16) float sw[];
    const long long wskip = WIDE ? 576LL * (p.nc - 1) : 0;            // block offset of b0 minus that of nc = 1
    for (int i = threadIdx.x + (WIDE ? 576 : 0); i < NW; i += blockDim.x) sw[i] = __ldg(p.w + wskip + i);
    __syncthreads();
    const float* c0 = sw; const float* b0 = c0 + 576; const float* c2 = b0 + 64; const float* b2 = c2 + 4096;
    const float* c4 = b2 + 64; const float* b4 = c4 + 4096; const float* c6 = b4 + 64; const float* b6 = c6 + 2048;
    pdl_wait_and_release();
    const long long pix = (long long)p.y_lo * p.W + (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (pix >= (long long)p.y_hi * p.W) return;
    const int y = (int)(pix / p.W), x = (int)(pix - (long long)y * p.W);
    float a[64], b[64];
    if constexpr (WIDE) {
        // same FMA order per output as below: from the bias, channel by channel, taps in row-major order
#pragma unroll
        for (int o = 0; o < 64; ++o) a[o] = b0[o];
        const long long plane = (long long)p.H * p.W;
#pragma unroll 1
        for (int ci = 0; ci < p.nc; ++ci) {
            float n[9];
#pragma unroll
            for (int dy = 0; dy < 3; ++dy)
#pragma unroll
                for (int dx = 0; dx < 3; ++dx) {
                    const int yy = y + dy - 1, xx = x + dx - 1;
                    n[dy * 3 + dx] = (yy >= 0 && yy < p.H && xx >= 0 && xx < p.W) ? __ldg(p.cond_in + ci * plane + (size_t)yy * p.W + xx) : 0.f;
                }
            const float* w0 = p.w + ci * 9;
#pragma unroll
            for (int o = 0; o < 64; ++o)
#pragma unroll
                for (int k = 0; k < 9; ++k) a[o] = fmaf(__ldg(w0 + (size_t)o * p.nc * 9 + k), n[k], a[o]);
        }
#pragma unroll
        for (int o = 0; o < 64; ++o) a[o] = a[o] > 0.f ? a[o] : 0.2f * a[o];
    } else {
        float n[9];
#pragma unroll
        for (int dy = 0; dy < 3; ++dy)
#pragma unroll
            for (int dx = 0; dx < 3; ++dx) {
                const int yy = y + dy - 1, xx = x + dx - 1;
                n[dy * 3 + dx] = (yy >= 0 && yy < p.H && xx >= 0 && xx < p.W) ? __ldg(p.cond_in + (size_t)yy * p.W + xx) : 0.f;
            }
#pragma unroll 4
        for (int o = 0; o < 64; ++o) {
            float v = b0[o];
#pragma unroll
            for (int k = 0; k < 9; ++k) v = fmaf(c0[o * 9 + k], n[k], v);
            a[o] = v > 0.f ? v : 0.2f * v;
        }
    }
#pragma unroll 2
    for (int o = 0; o < 64; ++o) {
        float v = b2[o];
#pragma unroll
        for (int k = 0; k < 64; ++k) v = fmaf(c2[o * 64 + k], a[k], v);
        b[o] = v > 0.f ? v : 0.2f * v;
    }
#pragma unroll 2
    for (int o = 0; o < 64; ++o) {
        float v = b4[o];
#pragma unroll
        for (int k = 0; k < 64; ++k) v = fmaf(c4[o * 64 + k], b[k], v);
        a[o] = v > 0.f ? v : 0.2f * v;
    }
#pragma unroll 2
    for (int o = 0; o < 32; ++o) {
        float v = b6[o];
#pragma unroll
        for (int k = 0; k < 64; ++k) v = fmaf(c6[o * 64 + k], a[k], v);
        p.cond_out[pix * 32 + o] = v;
        if (p.cond16) p.cond16[pix * 32 + o] = __ushort_as_half((unsigned short)h2_sat(v, 0.f));   // operand of the fused SFT epilogues
    }
}

// ---------------------------------------------------------------------------------------------
// CondNet on the tensor cores (round 2): the 1x1 layers (64->64, 64->64, 64->32) as mma.sync GEMMs on 16-pixel row
// blocks, fp32-class through a 3-term fp16 split (a = ah + al, W = Wh + Wl; ah*Wh + al*Wh + ah*Wl, fp32 accumulate:
// the dropped al*Wl term is ~2^-22 relative), the 3x3 layer (9 MACs per output) in fp32 FFMA computed directly in the
// A-fragment layout.  The condition map feeds every SFT layer, so it is kept at fp32 accuracy; the fp32 FFMA kernel
// above (254 us per 520x520 tile, 4 % of the decoder) stays as the reference (K4_CONDNET_FP32=1).
// ---------------------------------------------------------------------------------------------
constexpr int CNM_PITCH = 72;                                   // halfs per weight row (64 + 8: conflict-free fragment loads)
struct CnmLayout { int w1h, w1l, w2h, w2l, w3h, w3l, w0, b0, b1, b2, b3, total; };
__host__ __device__ inline CnmLayout cnm_layout() {
    CnmLayout L; int o = 0;
    L.w1h = o; o += 64 * CNM_PITCH * 2; L.w1l = o; o += 64 * CNM_PITCH * 2;
    L.w2h = o; o += 64 * CNM_PITCH * 2; L.w2l = o; o += 64 * CNM_PITCH * 2;
    L.w3h = o; o += 32 * CNM_PITCH * 2; L.w3l = o; o += 32 * CNM_PITCH * 2;
    L.w0 = o; o += 64 * 9 * 4; L.b0 = o; o += 64 * 4; L.b1 = o; o += 64 * 4; L.b2 = o; o += 64 * 4; L.b3 = o; o += 32 * 4;
    L.total = (o + 15) & ~15;
    return L;
}
// w: c0 [64][nc][9], b0[64], c2 [64][64], b2, c4 [64][64], b4, c6 [32][64], b6  (the fp32 kernel's packing).  The fp32
// layer-0 weights w0 are packed at nc = 1 only; a wide layer 0 is packed by pack_condnet_wide_kernel.
__global__ void pack_condnet_mma_kernel(const float* __restrict__ w, int nc, unsigned char* __restrict__ dst) {
    const CnmLayout L = cnm_layout();
    const float* c0 = w; const float* b0 = c0 + 576 * nc; const float* c2 = b0 + 64; const float* b2 = c2 + 4096;
    const float* c4 = b2 + 64; const float* b4 = c4 + 4096; const float* c6 = b4 + 64; const float* b6 = c6 + 2048;
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    auto split = [&](int offh, int offl, int n, int k, float v) {
        const __half hi = __float2half_rn(v);
        reinterpret_cast<__half*>(dst + offh)[n * CNM_PITCH + k] = hi;
        reinterpret_cast<__half*>(dst + offl)[n * CNM_PITCH + k] = __float2half_rn(v - __half2float(hi));
    };
    if (i < 4096) { split(L.w1h, L.w1l, i >> 6, i & 63, c2[i]); split(L.w2h, L.w2l, i >> 6, i & 63, c4[i]); }
    if (i < 2048) split(L.w3h, L.w3l, i >> 6, i & 63, c6[i]);
    if (i < 576 && nc == 1) reinterpret_cast<float*>(dst + L.w0)[i] = c0[i];
    if (i < 64) { reinterpret_cast<float*>(dst + L.b0)[i] = b0[i]; reinterpret_cast<float*>(dst + L.b1)[i] = b2[i]; reinterpret_cast<float*>(dst + L.b2)[i] = b4[i]; }
    if (i < 32) reinterpret_cast<float*>(dst + L.b3)[i] = b6[i];
}

// Wide layer 0 (1 < nc <= 64): an implicit GEMM with K = 9 taps x 64 channels, tap-major.  Its weights follow the
// cnm_layout block as hi / lo fp16 rows [n][tap * 64 + c], CNW_PITCH halfs apart (584 = 4 words mod 32 banks: the eight
// rows g and four column pairs tq of a B-fragment load hit 32 different banks).  Channels c >= nc are zero.
constexpr int CNW_PITCH = 9 * 64 + 8;
__host__ __device__ inline int cnw_bytes() { return cnm_layout().total + 2 * 64 * CNW_PITCH * 2; }

// c0: CondNet.0 [64][nc][3][3] fp32 -> the hi / lo rows behind the cnm_layout block of dst (zeroed beforehand)
__global__ void pack_condnet_wide_kernel(const float* __restrict__ c0, int nc, unsigned char* __restrict__ dst) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= 64 * 9 * nc) return;
    const int n = i / (9 * nc), r = i - n * 9 * nc, c = r / 9, t = r - c * 9;
    __half* wh = reinterpret_cast<__half*>(dst + cnm_layout().total);
    __half* wl = wh + 64 * CNW_PITCH;
    const __half hi = __float2half_rn(c0[i]);
    wh[n * CNW_PITCH + t * 64 + c] = hi;
    wl[n * CNW_PITCH + t * 64 + c] = __float2half_rn(c0[i] - __half2float(hi));
}

// cond_in: planar fp32 [nc][H][W]; wblk: the cnm_layout block (+ the wide layer-0 rows when nc > 1)
struct CondMmaParams { const float* cond_in; const unsigned char* wblk; float* cond_out; __half* cond16; int H, W, y_lo, y_hi, nc; };

// accumulator fragments of 2 adjacent n8 blocks -> hi / lo A fragments of one k16 step.  Both halves saturate: beyond
// the fp16 range hi = +-65504 and lo = x - hi, itself clamped, so an activation of 65520 or more stays finite (a
// rounding to inf would make lo = -inf and the next MMA NaN).
__device__ __forceinline__ void cnm_split_frag(const float (&c0)[4], const float (&c1)[4], uint32_t (&ah)[4], uint32_t (&al)[4]) {
    auto pk = [](float x, float y, uint32_t& hi, uint32_t& lo) {
        hi = h2_sat(x, y);
        const float2 hf = __half22float2(*reinterpret_cast<const __half2*>(&hi));
        lo = h2_sat(x - hf.x, y - hf.y);
    };
    pk(c0[0], c0[1], ah[0], al[0]); pk(c0[2], c0[3], ah[1], al[1]);
    pk(c1[0], c1[1], ah[2], al[2]); pk(c1[2], c1[3], ah[3], al[3]);
}
// one 64-input layer for 16 pixels: NBLK n8 blocks of outputs, 3-term split products
template <int NBLK>
__device__ __forceinline__ void cnm_layer(const unsigned char* sm, int offh, int offl, int offb, const uint32_t (&ah)[4][4], const uint32_t (&al)[4][4],
                                          int g, int tq, float (&c)[NBLK][4]) {
    const __half* Wh = reinterpret_cast<const __half*>(sm + offh);
    const __half* Wl = reinterpret_cast<const __half*>(sm + offl);
    const float* b = reinterpret_cast<const float*>(sm + offb);
#pragma unroll
    for (int j = 0; j < NBLK; ++j) {
        c[j][0] = c[j][2] = b[8 * j + 2 * tq]; c[j][1] = c[j][3] = b[8 * j + 2 * tq + 1];
#pragma unroll
        for (int ks = 0; ks < 4; ++ks) {
            const __half* wh = Wh + (8 * j + g) * CNM_PITCH + 16 * ks + 2 * tq;
            const __half* wl = Wl + (8 * j + g) * CNM_PITCH + 16 * ks + 2 * tq;
            const uint32_t bh0 = *reinterpret_cast<const uint32_t*>(wh), bh1 = *reinterpret_cast<const uint32_t*>(wh + 8);
            mma_16816(c[j], al[ks], bh0, bh1);                     // small terms first
            mma_16816(c[j], ah[ks], *reinterpret_cast<const uint32_t*>(wl), *reinterpret_cast<const uint32_t*>(wl + 8));
            mma_16816(c[j], ah[ks], bh0, bh1);
        }
    }
}

// CondNet's 1x1 layers (64 -> 64, 64 -> 64, 64 -> 32) on layer 0's split LeakyReLU output, and the cond_out / cond16
// stores of the block's two pixel rows
__device__ __forceinline__ void cnm_tail(const unsigned char* csm, const CnmLayout& L, uint32_t (&ah)[4][4], uint32_t (&al)[4][4],
                                         int g, int tq, const CondMmaParams& p, long long pixA, long long pixB, bool inA, bool inB) {
    float c[8][4];
    cnm_layer<8>(csm, L.w1h, L.w1l, L.b1, ah, al, g, tq, c);
#pragma unroll
    for (int j = 0; j < 8; ++j)
#pragma unroll
        for (int e = 0; e < 4; ++e) c[j][e] = fmaxf(c[j][e], 0.2f * c[j][e]);
#pragma unroll
    for (int ks = 0; ks < 4; ++ks) cnm_split_frag(c[2 * ks], c[2 * ks + 1], ah[ks], al[ks]);
    cnm_layer<8>(csm, L.w2h, L.w2l, L.b2, ah, al, g, tq, c);
#pragma unroll
    for (int j = 0; j < 8; ++j)
#pragma unroll
        for (int e = 0; e < 4; ++e) c[j][e] = fmaxf(c[j][e], 0.2f * c[j][e]);
#pragma unroll
    for (int ks = 0; ks < 4; ++ks) cnm_split_frag(c[2 * ks], c[2 * ks + 1], ah[ks], al[ks]);
    float o[4][4];
    cnm_layer<4>(csm, L.w3h, L.w3l, L.b3, ah, al, g, tq, o);
#pragma unroll
    for (int j = 0; j < 4; ++j) {
        const int ch = 8 * j + 2 * tq;
        if (inA) {
            *reinterpret_cast<float2*>(p.cond_out + pixA * 32 + ch) = make_float2(o[j][0], o[j][1]);
            if (p.cond16) *reinterpret_cast<uint32_t*>(p.cond16 + pixA * 32 + ch) = h2_sat(o[j][0], o[j][1]);
        }
        if (inB) {
            *reinterpret_cast<float2*>(p.cond_out + pixB * 32 + ch) = make_float2(o[j][2], o[j][3]);
            if (p.cond16) *reinterpret_cast<uint32_t*>(p.cond16 + pixB * 32 + ch) = h2_sat(o[j][2], o[j][3]);
        }
    }
}

__global__ void __launch_bounds__(128) condnet_mma_kernel(const __grid_constant__ CondMmaParams p) {
    extern __shared__ __align__(16) unsigned char csm[];
    const CnmLayout L = cnm_layout();
    for (int i = threadIdx.x; i < L.total / 16; i += blockDim.x) reinterpret_cast<uint4*>(csm)[i] = __ldg(reinterpret_cast<const uint4*>(p.wblk) + i);
    __syncthreads();
    pdl_wait_and_release();
    const int lane = threadIdx.x & 31, g = lane >> 2, tq = lane & 3;
    const long long p0 = (long long)p.y_lo * p.W, pend = (long long)p.y_hi * p.W;
    const long long nblk = (pend - p0 + 15) / 16;
    const float* W0 = reinterpret_cast<const float*>(csm + L.w0);
    const float* B0 = reinterpret_cast<const float*>(csm + L.b0);
    for (long long blk = (long long)blockIdx.x * 4 + (threadIdx.x >> 5); blk < nblk; blk += (long long)gridDim.x * 4) {
        const long long pixA = p0 + blk * 16 + g, pixB = pixA + 8;
        const bool inA = pixA < pend, inB = pixB < pend;
        // 3x3 neighbourhoods of the two pixels (zero padding at the tile border, as the reference's conv)
        float nA[9], nB[9];
        {
            const long long pa = inA ? pixA : p0, pb = inB ? pixB : p0;
            const int ya = (int)(pa / p.W), xa = (int)(pa - (long long)ya * p.W), yb = (int)(pb / p.W), xb = (int)(pb - (long long)yb * p.W);
#pragma unroll
            for (int dy = 0; dy < 3; ++dy)
#pragma unroll
                for (int dx = 0; dx < 3; ++dx) {
                    const int y1 = ya + dy - 1, x1 = xa + dx - 1, y2 = yb + dy - 1, x2 = xb + dx - 1;
                    nA[dy * 3 + dx] = (y1 >= 0 && y1 < p.H && x1 >= 0 && x1 < p.W) ? __ldg(p.cond_in + (size_t)y1 * p.W + x1) : 0.f;
                    nB[dy * 3 + dx] = (y2 >= 0 && y2 < p.H && x2 >= 0 && x2 < p.W) ? __ldg(p.cond_in + (size_t)y2 * p.W + x2) : 0.f;
                }
        }
        // layer 0 (3x3, 1 -> 64) in fp32, each thread the 16 channels of its A-fragment slots: k-step ks holds channels
        // 16ks + 2tq, +1 (regs 0 / 1: pixel A / B) and 16ks + 8 + 2tq, +1 (regs 2 / 3)
        uint32_t ah[4][4], al[4][4];
#pragma unroll
        for (int ks = 0; ks < 4; ++ks) {
            float va[4], vb[4];
#pragma unroll
            for (int e = 0; e < 4; ++e) {
                const int ch = 16 * ks + (e >> 1) * 8 + 2 * tq + (e & 1);
                float a = B0[ch], b = B0[ch];
#pragma unroll
                for (int k = 0; k < 9; ++k) { a = fmaf(W0[ch * 9 + k], nA[k], a); b = fmaf(W0[ch * 9 + k], nB[k], b); }
                va[e] = fmaxf(a, 0.2f * a); vb[e] = fmaxf(b, 0.2f * b);
            }
            const float c0[4] = {va[0], va[1], vb[0], vb[1]}, c1[4] = {va[2], va[3], vb[2], vb[3]};
            cnm_split_frag(c0, c1, ah[ks], al[ks]);
        }
        cnm_tail(csm, L, ah, al, g, tq, p, pixA, pixB, inA, inB);
    }
}

// CondNet with a wide condition (1 < nc <= 64, NKS = ceil(nc / 16) k16 steps per tap): layer 0 as an implicit GEMM on
// the tensor cores, 16-pixel row blocks (M) x 9 taps x 16 NKS channels (K) x 64 outputs (N), with the 3-term split of
// the 1x1 layers on both operands: the condition is read straight from its planar fp32 map (L1 serves the nine taps'
// reuse) and split to hi / lo in registers, the weights come pre-split from shared memory.  Channels >= nc and taps
// outside the map are zero A operands.  The LeakyReLU output feeds the same 1x1 chain as condnet_mma_kernel.
// Shared memory: the cnm_layout block + 146 KB of layer-0 rows (cnw_bytes, 194 KB): one CTA of 8 warps per SM.
template <int NKS>
__global__ void __launch_bounds__(256, 1) condnet_wide_mma_kernel(const __grid_constant__ CondMmaParams p) {
    extern __shared__ __align__(16) unsigned char csm[];
    const CnmLayout L = cnm_layout();
    for (int i = threadIdx.x; i < cnw_bytes() / 16; i += blockDim.x) reinterpret_cast<uint4*>(csm)[i] = __ldg(reinterpret_cast<const uint4*>(p.wblk) + i);
    __syncthreads();
    pdl_wait_and_release();
    const int lane = threadIdx.x & 31, g = lane >> 2, tq = lane & 3, nwarps = blockDim.x >> 5;
    const long long p0 = (long long)p.y_lo * p.W, pend = (long long)p.y_hi * p.W;
    const long long nblk = (pend - p0 + 15) / 16, plane = (long long)p.H * p.W;
    const __half* W0h = reinterpret_cast<const __half*>(csm + L.total);
    const __half* W0l = W0h + 64 * CNW_PITCH;
    const float* B0 = reinterpret_cast<const float*>(csm + L.b0);
    for (long long blk = (long long)blockIdx.x * nwarps + (threadIdx.x >> 5); blk < nblk; blk += (long long)gridDim.x * nwarps) {
        const long long pixA = p0 + blk * 16 + g, pixB = pixA + 8;
        const bool inA = pixA < pend, inB = pixB < pend;
        const long long pa = inA ? pixA : p0, pb = inB ? pixB : p0;
        const int ya = (int)(pa / p.W), xa = (int)(pa - (long long)ya * p.W), yb = (int)(pb / p.W), xb = (int)(pb - (long long)yb * p.W);
        float c[8][4];
#pragma unroll
        for (int j = 0; j < 8; ++j) { c[j][0] = c[j][2] = B0[8 * j + 2 * tq]; c[j][1] = c[j][3] = B0[8 * j + 2 * tq + 1]; }
#pragma unroll 1
        for (int t = 0; t < 9; ++t) {
            const int y1 = ya + t / 3 - 1, x1 = xa + t % 3 - 1, y2 = yb + t / 3 - 1, x2 = xb + t % 3 - 1;
            const bool okA = y1 >= 0 && y1 < p.H && x1 >= 0 && x1 < p.W, okB = y2 >= 0 && y2 < p.H && x2 >= 0 && x2 < p.W;
            const float* sA = p.cond_in + (okA ? (long long)y1 * p.W + x1 : 0);
            const float* sB = p.cond_in + (okB ? (long long)y2 * p.W + x2 : 0);
            // A operands of the tap's NKS k16 steps: channels 16ks + 2tq, +1 (regs 0 / 1: pixel A / B), +8, +9 (regs 2 / 3)
            float va[NKS][4], vb[NKS][4];
#pragma unroll
            for (int ks = 0; ks < NKS; ++ks)
#pragma unroll
                for (int e = 0; e < 4; ++e) {
                    const int ch = 16 * ks + (e >> 1) * 8 + 2 * tq + (e & 1);
                    va[ks][e] = (okA && ch < p.nc) ? __ldg(sA + ch * plane) : 0.f;
                    vb[ks][e] = (okB && ch < p.nc) ? __ldg(sB + ch * plane) : 0.f;
                }
#pragma unroll
            for (int ks = 0; ks < NKS; ++ks) {
                uint32_t ah[4], al[4];
                const float f0[4] = {va[ks][0], va[ks][1], vb[ks][0], vb[ks][1]}, f1[4] = {va[ks][2], va[ks][3], vb[ks][2], vb[ks][3]};
                cnm_split_frag(f0, f1, ah, al);
                const int k0 = t * 64 + 16 * ks + 2 * tq;
#pragma unroll
                for (int j = 0; j < 8; ++j) {
                    const __half* wh = W0h + (8 * j + g) * CNW_PITCH + k0;
                    const __half* wl = W0l + (8 * j + g) * CNW_PITCH + k0;
                    const uint32_t bh0 = *reinterpret_cast<const uint32_t*>(wh), bh1 = *reinterpret_cast<const uint32_t*>(wh + 8);
                    mma_16816(c[j], al, bh0, bh1);                  // small terms first
                    mma_16816(c[j], ah, *reinterpret_cast<const uint32_t*>(wl), *reinterpret_cast<const uint32_t*>(wl + 8));
                    mma_16816(c[j], ah, bh0, bh1);
                }
            }
        }
#pragma unroll
        for (int j = 0; j < 8; ++j)
#pragma unroll
            for (int e = 0; e < 4; ++e) c[j][e] = fmaxf(c[j][e], 0.2f * c[j][e]);
        uint32_t ah[4][4], al[4][4];
#pragma unroll
        for (int ks = 0; ks < 4; ++ks) cnm_split_frag(c[2 * ks], c[2 * ks + 1], ah[ks], al[ks]);
        cnm_tail(csm, L, ah, al, g, tq, p, pixA, pixB, inA, inB);
    }
}

// planar fp32 [C,H,W] -> NHWC fp16 [H,W,32] (zero padded)
__global__ void nchw_to_nhwc32_kernel(const float* __restrict__ src, __half* __restrict__ dst, int C, long long P) {
    pdl_wait_and_release();
    const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= P * 32) return;
    const long long pix = i >> 5;
    const int c = (int)(i & 31);
    dst[i] = __float2half_rn(c < C ? src[(size_t)c * P + pix] : 0.f);
}

// conv weight [Cout][Cin][3][3] fp32 -> [cin_slice][tap][NPAD][SR_CK] canonical K-major fp16 tiles
__global__ void pack_conv3x3_kernel(const float* __restrict__ W, unsigned char* __restrict__ dst,
                                    int cout, int cin, int npad, int nslices) {
    const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    const long long total = (long long)nslices * 9 * npad * SR_CK;
    if (i >= total) return;
    const int k = (int)(i % SR_CK);
    long long r = i / SR_CK;
    const int n = (int)(r % npad); r /= npad;
    const int t = (int)(r % 9);
    const int sl = (int)(r / 9);
    const int ci = sl * SR_CK + k;
    const float w = (n < cout && ci < cin) ? W[((size_t)n * cin + ci) * 9 + t] : 0.f;
    const size_t off = ((size_t)sl * 9 + t) * (npad * SR_CK * 2) + tc_canon_off(n, k >> 3, SR_CK / 8) + (k & 7) * 2;
    *reinterpret_cast<__half*>(dst + off) = __float2half_rn(w);
}

// Sub-pixel weights of "nearest x2 upsample, then 3x3 conv": output pixel (2Y+py, 2X+px) only sees the 2x2
// source pixels (Y+py-1..Y+py, X+px-1..X+px); each of them collects the kernel rows / columns that land on it
// after upsampling: phase 0: {-1: k0, 0: k1+k2}, phase 1: {0: k0+k1, +1: k2}.  Packed as [slice][4 taps][NPAD][SR_CK]
// (tap = 2*iy + ix); the sums are formed in fp32 and rounded to fp16 once.  4/9 of the MACs of the direct form.
__global__ void pack_conv_phase_kernel(const float* __restrict__ W, unsigned char* __restrict__ dst,
                                       int cout, int cin, int npad, int nslices, int py, int px) {
    const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    const long long total = (long long)nslices * 4 * npad * SR_CK;
    if (i >= total) return;
    const int k = (int)(i % SR_CK);
    long long r = i / SR_CK;
    const int n = (int)(r % npad); r /= npad;
    const int t = (int)(r % 4);
    const int sl = (int)(r / 4);
    const int ci = sl * SR_CK + k;
    const int iy = t >> 1, ix = t & 1;
    // kernel index range collected by source offset (phase + i - 1)
    const int ky0 = (py == 0) ? (iy == 0 ? 0 : 1) : (iy == 0 ? 0 : 2), ky1 = (py == 0) ? (iy == 0 ? 0 : 2) : (iy == 0 ? 1 : 2);
    const int kx0 = (px == 0) ? (ix == 0 ? 0 : 1) : (ix == 0 ? 0 : 2), kx1 = (px == 0) ? (ix == 0 ? 0 : 2) : (ix == 0 ? 1 : 2);
    float w = 0.f;
    if (n < cout && ci < cin)
        for (int ky = ky0; ky <= ky1; ++ky)
            for (int kx = kx0; kx <= kx1; ++kx) w += W[((size_t)n * cin + ci) * 9 + ky * 3 + kx];
    const size_t off = ((size_t)sl * 4 + t) * (npad * SR_CK * 2) + tc_canon_off(n, k >> 3, SR_CK / 8) + (k & 7) * 2;
    *reinterpret_cast<__half*>(dst + off) = __float2half_rn(w);
}

// Weights for conv3x3_k64_kernel: plain [tap][NPAD][64] fp16 rows (the TMA copy applies the 128-byte swizzle).
// phase < 0: the nine taps of the direct 3x3 conv; phase 0..3: the four taps of that sub-pixel phase
// (same combination rule as pack_conv_phase_kernel).
__global__ void pack_conv_k64_kernel(const float* __restrict__ W, __half* __restrict__ dst, int cout, int cin, int npad, int phase) {
    const int ntaps = (phase < 0) ? 9 : 4;
    const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= (long long)ntaps * npad * 64) return;
    const int k = (int)(i % 64);
    const int n = (int)((i / 64) % npad);
    const int t = (int)(i / 64 / npad);
    float w = 0.f;
    if (n < cout && k < cin) {
        if (phase < 0) {
            w = W[((size_t)n * cin + k) * 9 + t];
        } else {
            const int py = phase >> 1, px = phase & 1, iy = t >> 1, ix = t & 1;
            const int ky0 = (py == 0) ? (iy == 0 ? 0 : 1) : (iy == 0 ? 0 : 2), ky1 = (py == 0) ? (iy == 0 ? 0 : 2) : (iy == 0 ? 1 : 2);
            const int kx0 = (px == 0) ? (ix == 0 ? 0 : 1) : (ix == 0 ? 0 : 2), kx1 = (px == 0) ? (ix == 0 ? 0 : 2) : (ix == 0 ? 1 : 2);
            for (int ky = ky0; ky <= ky1; ++ky)
                for (int kx = kx0; kx <= kx1; ++kx) w += W[((size_t)n * cin + k) * 9 + ky * 3 + kx];
        }
    }
    dst[i] = __float2half_rn(w);
}

}  // namespace

// ------------------------------------------------------------------------------------------------
// host side
// ------------------------------------------------------------------------------------------------
struct SrConv { unsigned char* wpack; float* bias; int cin_pad, cout, npad; unsigned char* wphase[4];
                __half* wk64; __half* wk64_phase[4]; };       // conv3x3_k64_kernel packs (Cin == 64 layers only)
struct SrSft { float* w; unsigned char* frag; int cout; };

struct k4_srnet {
    int num_feat, num_block, num_grow, num_cond, n_in, scale;
    SrConv conv_first, conv_body, conv_up1, conv_up2, conv_hr, conv_last;
    SrConv rdb_conv[32][3][5];
    SrSft rdb_sft[32][3][2];
    SrSft rrdb_sft[32];
    SrSft sftbody;
    float* condnet_w;
    unsigned char* condnet_mma;                 // cnm_layout block of condnet_mma_kernel
    void* allocs[1024];
    int n_allocs;
    size_t bytes;
};

namespace {

int sr_alloc(k4_srnet* n, void** p, size_t bytes) {
    if (n->n_allocs >= 1024) return K4_ERR_INVALID_ARG;
    K4_CUDA_TRY(cudaMalloc(p, bytes ? bytes : 16));
    n->allocs[n->n_allocs++] = *p;
    n->bytes += bytes;
    return K4_OK;
}

int make_conv(k4_srnet* n, SrConv& c, const float* w, const float* b, int cout, int cin, cudaStream_t s) {
    c.cout = cout;
    c.npad = cout <= 16 ? 16 : (cout <= 32 ? 32 : 64);
    c.cin_pad = (cin + 31) / 32 * 32;              // activations are stored in multiples of 32 channels
    const int nsl = c.cin_pad / SR_CK;
    const size_t bytes = (size_t)nsl * 9 * c.npad * SR_CK * 2;
    int st = sr_alloc(n, (void**)&c.wpack, bytes);
    if (st) return st;
    st = sr_alloc(n, (void**)&c.bias, 64 * 4);
    if (st) return st;
    K4_CUDA_TRY(cudaMemsetAsync(c.bias, 0, 64 * 4, s));
    K4_CUDA_TRY(cudaMemcpyAsync(c.bias, b, (size_t)cout * 4, cudaMemcpyDeviceToDevice, s));
    const long long total = (long long)nsl * 9 * c.npad * SR_CK;
    pack_conv3x3_kernel<<<(unsigned)((total + 255) / 256), 256, 0, s>>>(w, c.wpack, cout, cin, c.npad, nsl);
    K4_CUDA_TRY(cudaGetLastError());
    return K4_OK;
}

// the four sub-pixel weight packs of a conv that follows a nearest-x2 upsampling (conv_up1 / conv_up2)
int make_conv_phases(k4_srnet* n, SrConv& c, const float* w, int cout, int cin, cudaStream_t s) {
    const int nsl = c.cin_pad / SR_CK;
    const size_t bytes = (size_t)nsl * 4 * c.npad * SR_CK * 2;
    const long long total = (long long)nsl * 4 * c.npad * SR_CK;
    for (int ph = 0; ph < 4; ++ph) {
        int st = sr_alloc(n, (void**)&c.wphase[ph], bytes);
        if (st) return st;
        pack_conv_phase_kernel<<<(unsigned)((total + 255) / 256), 256, 0, s>>>(w, c.wphase[ph], cout, cin, c.npad, nsl, ph >> 1, ph & 1);
        K4_CUDA_TRY(cudaGetLastError());
    }
    return K4_OK;
}

// [tap][npad][64] packs for conv3x3_k64_kernel (direct 9 taps, and the 4 phases when `phases`)
int make_conv_k64(k4_srnet* n, SrConv& c, const float* w, int cout, int cin, bool phases, cudaStream_t s) {
    if (cin != 64 || (c.npad != 64 && c.npad != 16)) return K4_OK;
    {
        const long long total = 9LL * c.npad * 64;
        int st = sr_alloc(n, (void**)&c.wk64, (size_t)total * 2);
        if (st) return st;
        pack_conv_k64_kernel<<<(unsigned)((total + 255) / 256), 256, 0, s>>>(w, c.wk64, cout, cin, c.npad, -1);
        K4_CUDA_TRY(cudaGetLastError());
    }
    for (int ph = 0; phases && ph < 4; ++ph) {
        const long long total = 4LL * c.npad * 64;
        int st = sr_alloc(n, (void**)&c.wk64_phase[ph], (size_t)total * 2);
        if (st) return st;
        pack_conv_k64_kernel<<<(unsigned)((total + 255) / 256), 256, 0, s>>>(w, c.wk64_phase[ph], cout, cin, c.npad, ph);
        K4_CUDA_TRY(cudaGetLastError());
    }
    return K4_OK;
}

// SFT weights: 4 convs in the order scale0, scale1, shift0, shift1 (weight, bias each) -> packed s0,s0b,h0,h0b,s1,s1b,h1,h1b
int make_sft(k4_srnet* n, SrSft& f, const float* const* pw, int cout, cudaStream_t s) {
    f.cout = cout;
    const size_t nw = 2 * (1024 + 32) + 2 * ((size_t)cout * 32 + cout);
    int st = sr_alloc(n, (void**)&f.w, nw * 4);
    if (st) return st;
    float* d = f.w;
    auto cp = [&](const float* src, size_t cnt) { cudaMemcpyAsync(d, src, cnt * 4, cudaMemcpyDeviceToDevice, s); d += cnt; };
    cp(pw[0], 1024); cp(pw[1], 32);                 // scale_conv0 w, b
    cp(pw[4], 1024); cp(pw[5], 32);                 // shift_conv0 w, b
    cp(pw[2], (size_t)cout * 32); cp(pw[3], cout);  // scale_conv1 w, b
    cp(pw[6], (size_t)cout * 32); cp(pw[7], cout);  // shift_conv1 w, b
    K4_CUDA_TRY(cudaGetLastError());
    const SftFrag FL = sft_frag_layout(cout);
    st = sr_alloc(n, (void**)&f.frag, (size_t)FL.total);
    if (st) return st;
    K4_CUDA_TRY(cudaMemsetAsync(f.frag, 0, FL.total, s));
    pack_sft_frag_kernel<<<8, 256, 0, s>>>(f.w, f.frag, cout);
    K4_CUDA_TRY(cudaGetLastError());
    return K4_OK;
}

// CondNet weights: the 8 tensors of CondNet.0 (64 x nc x 3x3), .2 (64x64), .4 (64x64), .6 (32x64) and their biases -> the
// fp32 block of condnet_kernel and the cnm_layout block of condnet_mma_kernel, followed at nc > 1 by the wide layer-0
// rows of condnet_wide_mma_kernel
int make_condnet(k4_srnet* n, const float* const* pw, int nc, cudaStream_t s) {
    const size_t cnt[8] = {576 * (size_t)nc, 64, 4096, 64, 4096, 64, 2048, 32};
    size_t nw = 0;
    for (int q = 0; q < 8; ++q) nw += cnt[q];
    int st = sr_alloc(n, (void**)&n->condnet_w, nw * 4);
    if (st) return st;
    float* dd = n->condnet_w;
    for (int q = 0; q < 8; ++q) { cudaMemcpyAsync(dd, pw[q], cnt[q] * 4, cudaMemcpyDeviceToDevice, s); dd += cnt[q]; }
    const int bytes = nc == 1 ? cnm_layout().total : cnw_bytes();
    st = sr_alloc(n, (void**)&n->condnet_mma, (size_t)bytes);
    if (st) return st;
    K4_CUDA_TRY(cudaMemsetAsync(n->condnet_mma, 0, bytes, s));
    pack_condnet_mma_kernel<<<16, 256, 0, s>>>(n->condnet_w, nc, n->condnet_mma);
    if (nc > 1) pack_condnet_wide_kernel<<<(64 * 9 * nc + 255) / 256, 256, 0, s>>>(n->condnet_w, nc, n->condnet_mma);
    K4_CUDA_TRY(cudaGetLastError());
    return K4_OK;
}

// K4_SR_PDL=0 launches the decoder kernels without programmatic dependent launch (A/B switch)
static bool sr_use_pdl() {
    static int v = -1;
    if (v < 0) { const char* e = getenv("K4_SR_PDL"); v = (e && e[0] == '0') ? 0 : 1; }
    return v == 1;
}

template <typename... KArgs, typename... Args>
cudaError_t sr_launch(void (*kern)(KArgs...), unsigned grid, unsigned block, size_t smem, cudaStream_t s, Args&&... args) {
    cudaLaunchConfig_t cfg = {};
    cfg.gridDim = dim3(grid); cfg.blockDim = dim3(block); cfg.dynamicSmemBytes = smem; cfg.stream = s;
    cudaLaunchAttribute at[1];
    at[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
    at[0].val.programmaticStreamSerializationAllowed = 1;
    cfg.attrs = at; cfg.numAttrs = sr_use_pdl() ? 1 : 0;
    return cudaLaunchKernelEx(&cfg, kern, static_cast<KArgs>(args)...);
}

// per-device caches of the launchers (function attributes are per device; ADVICE r1)
struct SrDevInfo { int sms; unsigned attr_mask; };
static SrDevInfo* sr_dev() {
    static SrDevInfo info[64];
    int dev = 0;
    if (cudaGetDevice(&dev) != cudaSuccess || dev < 0 || dev >= 64) dev = 0;
    if (info[dev].sms == 0) cudaDeviceGetAttribute(&info[dev].sms, cudaDevAttrMultiProcessorCount, dev);
    return &info[dev];
}
template <typename F>
int sr_set_smem(F kern, int bit, int bytes) {
    SrDevInfo* d = sr_dev();
    if (!(d->attr_mask & (1u << bit))) {
        K4_CUDA_TRY(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, bytes));
        d->attr_mask |= (1u << bit);
    }
    return K4_OK;
}
constexpr int sr_bit_n(int n) { return n == 64 ? 0 : (n == 32 ? 1 : 2); }

typedef CUresult (*k4_encode_tiled_fn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*, const cuuint64_t*,
                                       const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave, CUtensorMapSwizzle,
                                       CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

// cuTensorMapEncodeTiled through the runtime's driver entry point (no link-time dependency on libcuda)
static k4_encode_tiled_fn sr_encode_tiled() {
    static k4_encode_tiled_fn fn = nullptr;
    static bool tried = false;
    if (!tried) {
        tried = true;
        void* ptr = nullptr;
        cudaDriverEntryPointQueryResult q;
        if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &ptr, cudaEnableDefault, &q) == cudaSuccess && q == cudaDriverEntryPointSuccess)
            fn = reinterpret_cast<k4_encode_tiled_fn>(ptr);
        else
            cudaGetLastError();
    }
    return fn;
}

// Tensor map of a rank-2 or rank-3 fp16 tensor at `base`: dense boxes (unit element strides), no interleave, 128-byte
// L2 promotion, and zeros for the elements of a box that lie outside the tensor (the convolutions' padding).  False when
// the driver has no cuTensorMapEncodeTiled or rejects the map.
static bool encode_f16_tmap(CUtensorMap* map, const void* base, cuuint32_t rank, const cuuint64_t* gdim, const cuuint64_t* gstride,
                            const cuuint32_t* box, CUtensorMapSwizzle swizzle) {
    k4_encode_tiled_fn enc = sr_encode_tiled();
    const cuuint32_t estr[3] = {1, 1, 1};
    return enc && enc(map, CU_TENSOR_MAP_DATA_TYPE_FLOAT16, rank, const_cast<void*>(base), gdim, gstride, box, estr,
                      CU_TENSOR_MAP_INTERLEAVE_NONE, swizzle, CU_TENSOR_MAP_L2_PROMOTION_L2_128B,
                      CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE) == CUDA_SUCCESS;
}

// (channel, x, y) view of the NHWC fp16 source starting at channel src_c0; box = one 8-channel halo plane
static bool sr_make_tmap(const ConvParams& p, CUtensorMap* tm) {
    const cuuint64_t gdim[3] = {(cuuint64_t)p.cin, (cuuint64_t)p.W, (cuuint64_t)p.H};
    const cuuint64_t gstride[2] = {(cuuint64_t)p.src_cstride * 2, (cuuint64_t)p.W * p.src_cstride * 2};
    const cuuint32_t box[3] = {8, (cuuint32_t)WS_HX, (cuuint32_t)SR_HY};
    const __half* base = p.src + p.src_c0;
    if (((uintptr_t)base & 15) || (gstride[0] & 15)) return false;
    return encode_f16_tmap(tm, base, 3, gdim, gstride, box, CU_TENSOR_MAP_SWIZZLE_NONE);
}

static bool sr_no_tma() {
    static int v = -1;
    if (v < 0) { const char* e = getenv("K4_CONV_NO_TMA"); v = (e && e[0] == '1') ? 1 : 0; }
    return v == 1;
}

// Which convolution kernel runs a layer (the K4_CONV_KERNEL_* values of k4_testing_conv3x3).  SRK_AUTO is the decoder's
// own choice, env switches included; a forced kernel either runs or the launch returns K4_ERR_UNSUPPORTED.
enum SrKernel { SRK_AUTO = 0, SRK_WS_TMA = 1, SRK_WS_CPASYNC = 2, SRK_K64 = 3 };

template <int N>
int launch_conv_ws(ConvParams p, cudaStream_t s, int sel, int* used) {
    using C = WsCfg<N>;
    if (int st = sr_set_smem(conv3x3_ws_kernel<N>, 3 + sr_bit_n(N), C::SMEM + SFTF_MAX)) return st;
    const int sms = sr_dev()->sms;
    alignas(64) CUtensorMap tm;
    memset(&tm, 0, sizeof(tm));
    const bool want_tma = (sel == SRK_AUTO) ? !sr_no_tma() : sel == SRK_WS_TMA;
    p.use_tma = (!p.upsample && want_tma && sr_make_tmap(p, &tm)) ? 1 : 0;
    if (sel == SRK_WS_TMA && !p.use_tma) return K4_ERR_UNSUPPORTED;
    const int tiles = ((p.W + WS_TX - 1) / WS_TX) * ((p.y_hi - p.y_lo + SR_TY - 1) / SR_TY);
    if (tiles <= 0) return K4_OK;
    size_t smem = C::SMEM;
    if (p.mode >= SRM_STORE_F16_SFT) {
        if (N < 32 || !p.cond16 || !p.sftw) return K4_ERR_UNSUPPORTED;     // the SFT layers follow 32- and 64-channel convolutions only
        smem += sft_frag_layout(p.sft_n).total + (p.mode == SRM_TRUNK_SFT2 ? sft_frag_layout(64).total : 0);
    }
    K4_CUDA_TRY(sr_launch(conv3x3_ws_kernel<N>, (unsigned)(tiles < sms ? tiles : sms), WS_THREADS, smem, s, p, tm));
    if (used) *used = p.use_tma ? SRK_WS_TMA : SRK_WS_CPASYNC;
    return K4_OK;
}

// conv3x3_k64_kernel launch: tensor maps for the activation (channel, x, y; box 64 x 26 x 18) and the weight rows
template <int N>
int launch_conv_k64(ConvParams p, const __half* wrows, cudaStream_t s) {
    using C = K64Cfg<N>;
    if (!sr_encode_tiled()) return K4_ERR_UNSUPPORTED;
    if (int st = sr_set_smem(conv3x3_k64_kernel<N>, 6 + sr_bit_n(N), C::SMEM)) return st;
    const int sms = sr_dev()->sms;
    alignas(64) CUtensorMap ta, tb;
    {
        const cuuint64_t gdim[3] = {64, (cuuint64_t)p.W, (cuuint64_t)p.H};
        const cuuint64_t gstr[2] = {(cuuint64_t)p.src_cstride * 2, (cuuint64_t)p.W * p.src_cstride * 2};
        const cuuint32_t box[3] = {64, (cuuint32_t)K64_HX, (cuuint32_t)SR_HY};
        if (!encode_f16_tmap(&ta, p.src + p.src_c0, 3, gdim, gstr, box, CU_TENSOR_MAP_SWIZZLE_128B)) return K4_ERR_UNSUPPORTED;
    }
    {
        const cuuint64_t gdim[2] = {64, (cuuint64_t)p.ntaps * N};
        const cuuint64_t gstr[1] = {128};
        const cuuint32_t box[2] = {64, (cuuint32_t)N};
        if (!encode_f16_tmap(&tb, wrows, 2, gdim, gstr, box, CU_TENSOR_MAP_SWIZZLE_128B)) return K4_ERR_UNSUPPORTED;
    }
    const int tiles = ((p.W + K64_TX - 1) / K64_TX) * ((p.y_hi - p.y_lo + SR_TY - 1) / SR_TY);
    if (tiles <= 0) return K4_OK;
    K4_CUDA_TRY(sr_launch(conv3x3_k64_kernel<N>, (unsigned)(tiles < sms ? tiles : sms), K64_THREADS, C::SMEM, s, p, ta, tb));
    return K4_OK;
}

// The 64-input-channel layers go to conv3x3_k64_kernel; K4_CONV_K64=0 keeps them on conv3x3_ws_kernel (A/B switch).
static bool sr_use_k64() {
    static int v = -1;
    if (v < 0) { const char* e = getenv("K4_CONV_K64"); v = (e && e[0] == '0') ? 0 : 1; }
    return v == 1;
}

// sel: SrKernel; *used (if given) receives the kernel that ran.
int run_conv(const SrConv& c, ConvParams p, cudaStream_t s, const __half* wk64_override = nullptr, int sel = SRK_AUTO,
             int* used = nullptr) {
    const __half* wk64 = wk64_override ? wk64_override : ((p.ntaps == 0 || p.ntaps == 9) ? c.wk64 : nullptr);
    if (!p.wpack) p.wpack = c.wpack;
    p.bias = c.bias; p.cin = c.cin_pad;
    if (p.ntaps == 0) {
        p.ntaps = 9;
        for (int t = 0; t < 9; ++t) { p.tap_dy[t] = (unsigned char)(t / 3); p.tap_dx[t] = (unsigned char)(t % 3); }
    }
    if (p.out_s == 0) p.out_s = 1;
    if (p.y_hi == 0) { p.y_lo = 0; p.y_hi = p.H; }
    if (p.y_lo < 0) p.y_lo = 0;
    if (p.y_hi > p.H) p.y_hi = p.H;
    if (p.y_hi <= p.y_lo) return K4_OK;
    const bool k64_ok = wk64 && p.cin == 64 && !p.upsample && !p.split && (p.src_cstride % 8) == 0 && (p.src_c0 % 8) == 0 &&
                        (p.mode == SRM_STORE_F16 || p.mode == SRM_ADD_STORE_F16 || p.mode == SRM_OUT_NCHW);
    if (sel == SRK_K64 || (sel == SRK_AUTO && sr_use_k64() && k64_ok)) {
        const int st = !k64_ok ? K4_ERR_UNSUPPORTED : (c.npad == 64) ? launch_conv_k64<64>(p, wk64, s)
                     : (c.npad == 16) ? launch_conv_k64<16>(p, wk64, s) : K4_ERR_UNSUPPORTED;
        if (st == K4_OK && used) *used = SRK_K64;
        if (st != K4_ERR_UNSUPPORTED || sel == SRK_K64) return st;
    }
    if (c.npad == 64) return launch_conv_ws<64>(p, s, sel, used);
    if (c.npad == 32) return launch_conv_ws<32>(p, s, sel, used);
    return launch_conv_ws<16>(p, s, sel, used);
}

// nearest-x2 + conv as four sub-pixel convolutions over the source grid (p.H x p.W = SOURCE size, dst is 2H x 2W)
int run_conv_up2x(const SrConv& c, ConvParams p, cudaStream_t s, int sel = SRK_AUTO, int* used = nullptr) {
    for (int ph = 0; ph < 4; ++ph) {
        const int py = ph >> 1, px = ph & 1;
        ConvParams q = p;
        q.upsample = 0; q.wpack = c.wphase[ph];
        q.ntaps = 4;
        for (int t = 0; t < 4; ++t) { q.tap_dy[t] = (unsigned char)(py + (t >> 1)); q.tap_dx[t] = (unsigned char)(px + (t & 1)); }
        q.out_s = 2; q.out_oy = py; q.out_ox = px;
        const int st = run_conv(c, q, s, c.wk64_phase[ph], sel, used);
        if (st != K4_OK) return st;
    }
    return K4_OK;
}

template <int COUT>
int launch_sft(const SftParams& p, cudaStream_t s) {
    constexpr int NW = 2 * (32 * 32 + 32) + 2 * (COUT * 32 + COUT);
    sft_kernel<COUT><<<(unsigned)((p.P + 127) / 128), 128, NW * 4, s>>>(p);
    K4_CUDA_TRY(cudaGetLastError());
    return K4_OK;
}

template <int COUT>
int launch_sft_mma(const SftParams& p, const unsigned char* frag, cudaStream_t s) {
    const int smem = sft_frag_layout(COUT).total;
    const long long nblk = (p.P + 15) / 16;
    if (nblk <= 0) return K4_OK;
    long long grid = (nblk + 3) / 4;
    const long long cap = (long long)sr_dev()->sms * 8;
    if (grid > cap) grid = cap;
    K4_CUDA_TRY(sr_launch(sft_mma_kernel<COUT>, (unsigned)grid, 128, (size_t)smem, s, p, frag));
    return K4_OK;
}

// Which kernel runs a CondNet or standalone SFT pass (the K4_SR_KERNEL_* values of k4_testing_condnet / k4_testing_sft).
// SRP_AUTO is the decoder's own choice, env switch included; both kernels run every shape, so a forced one always runs.
enum SrPixelKernel { SRP_AUTO = 0, SRP_MMA = 1, SRP_FP32 = 2 };

// sel: SrPixelKernel; *used (if given) receives the kernel that ran.
int run_sft(const SrSft& f, SftParams p, cudaStream_t s, int sel = SRP_AUTO, int* used = nullptr) {
    static const bool use_fp32 = getenv("K4_SFT_FP32") != nullptr;      // development switch: fp32 FFMA kernel
    const bool fp32 = (sel == SRP_AUTO) ? use_fp32 : sel == SRP_FP32;
    if (used) *used = fp32 ? SRP_FP32 : SRP_MMA;
    if (fp32) {
        p.w = f.w;
        return f.cout == 64 ? launch_sft<64>(p, s) : launch_sft<32>(p, s);
    }
    return f.cout == 64 ? launch_sft_mma<64>(p, f.frag, s) : launch_sft_mma<32>(p, f.frag, s);
}

template <int NKS>
int launch_condnet_wide(const CondMmaParams& cp, cudaStream_t s) {
    const int smem = cnw_bytes();
    if (int st = sr_set_smem(condnet_wide_mma_kernel<NKS>, 13 + NKS, smem)) return st;
    const long long nb = ((long long)(cp.y_hi - cp.y_lo) * cp.W + 15) / 16;
    long long grid = (nb + 7) / 8;
    const long long cap = (long long)sr_dev()->sms;                  // one CTA per SM fits its shared memory
    if (grid > cap) grid = cap;
    K4_CUDA_TRY(sr_launch(condnet_wide_mma_kernel<NKS>, (unsigned)(grid < 1 ? 1 : grid), 256, (size_t)smem, s, cp));
    return K4_OK;
}

// CondNet on rows [y_lo, y_hi) of an h x w condition map (planar fp32 [num_cond][h][w]): cond32 (fp32 [h*w][32]) and, if
// given, cond16 (the fp16 operand of the fused SFT epilogues) of those rows.  AUTO reads K4_CONDNET_FP32 per call (fp32
// FFMA kernel when it is "1").  num_cond 1 runs condnet_mma_kernel, a wider condition condnet_wide_mma_kernel.
int run_condnet(const k4_srnet* n, const float* cond_in, int h, int w, int y_lo, int y_hi, float* cond32, __half* cond16,
                cudaStream_t s, int sel = SRP_AUTO, int* used = nullptr) {
    bool fp32 = sel == SRP_FP32;
    if (sel == SRP_AUTO) { const char* cenv = getenv("K4_CONDNET_FP32"); fp32 = cenv && cenv[0] == '1'; }
    const int nc = n->num_cond;
    if (fp32) {
        CondParams cp{cond_in, n->condnet_w, cond32, h, w, y_lo, y_hi, cond16, nc};
        constexpr int NW = 64 * 9 + 64 + 2 * (64 * 64 + 64) + 32 * 64 + 32;
        const long long np = (long long)(y_hi - y_lo) * w;
        if (nc == 1) {
            if (int st = sr_set_smem(condnet_kernel<false>, 11, NW * 4)) return st;
            K4_CUDA_TRY(sr_launch(condnet_kernel<false>, (unsigned)((np + 127) / 128), 128, (size_t)NW * 4, s, cp));
        } else {
            if (int st = sr_set_smem(condnet_kernel<true>, 13, NW * 4)) return st;
            K4_CUDA_TRY(sr_launch(condnet_kernel<true>, (unsigned)((np + 127) / 128), 128, (size_t)NW * 4, s, cp));
        }
    } else if (nc > 1) {
        const CondMmaParams cp{cond_in, n->condnet_mma, cond32, cond16, h, w, y_lo, y_hi, nc};
        const int nks = (nc + 15) / 16;
        const int st = nks == 1 ? launch_condnet_wide<1>(cp, s) : nks == 2 ? launch_condnet_wide<2>(cp, s)
                     : nks == 3 ? launch_condnet_wide<3>(cp, s) : launch_condnet_wide<4>(cp, s);
        if (st) return st;
    } else {
        CondMmaParams cp{cond_in, n->condnet_mma, cond32, cond16, h, w, y_lo, y_hi, nc};
        const int smem = cnm_layout().total;
        if (int st = sr_set_smem(condnet_mma_kernel, 12, smem)) return st;
        const long long nb = ((long long)(y_hi - y_lo) * w + 15) / 16;
        long long grid = (nb + 3) / 4;
        const long long cap = (long long)sr_dev()->sms * 4;
        if (grid > cap) grid = cap;
        K4_CUDA_TRY(sr_launch(condnet_mma_kernel, (unsigned)(grid < 1 ? 1 : grid), 128, (size_t)smem, s, cp));
    }
    if (used) *used = fp32 ? SRP_FP32 : SRP_MMA;
    return K4_OK;
}

}  // namespace

extern "C" int k4_srnet_destroy(k4_srnet* n) {
    if (!n) return K4_OK;
    for (int i = 0; i < n->n_allocs; ++i) cudaFree(n->allocs[i]);
    delete n;
    return K4_OK;
}

extern "C" int k4_srnet_create(const k4_srnet_desc* d, k4_stream_t stream, k4_srnet** out) {
    if (!d || !out || !d->h_params) return K4_ERR_INVALID_ARG;
    *out = nullptr;
    if (d->num_cond < 1) return K4_ERR_INVALID_ARG;
    // the shipped configurations (run_sr.py:1353; x1 as in the 1x configs) with a condition of up to 64 channels (depth,
    // the view embedding, or both: run_sr.py:895-912); others are not built
    if (d->num_feat != 64 || d->num_grow_ch != 32 || d->num_cond > 64 || d->n_in_colors != 3 || (d->scale != 4 && d->scale != 1) ||
        d->num_block < 1 || d->num_block > 32)
        return K4_ERR_UNSUPPORTED;
    const bool up = d->scale == 4;          // x1 registers no conv_up1 / conv_up2 (lib/sr_esrnet.py:430-433)
    const int expect = 2 * (1 + 4 + d->num_block * (3 * 13 + 4) + 4 + (up ? 5 : 3));
    if (d->n_params != expect) return K4_ERR_INVALID_ARG;
    for (int i = 0; i < d->n_params; ++i) if (!d->h_params[i]) return K4_ERR_INVALID_ARG;
    int st = k4_device_check();
    if (st != K4_OK) return st;
    cudaStream_t s = (cudaStream_t)stream;
    k4_srnet* n = new (std::nothrow) k4_srnet();
    if (!n) return K4_ERR_INVALID_ARG;
    memset(n, 0, sizeof(*n));
    n->num_feat = 64; n->num_block = d->num_block; n->num_grow = 32; n->num_cond = d->num_cond; n->n_in = 3; n->scale = d->scale;
    const float* const* P = d->h_params;
    int k = 0;
#define SR_TRY(x) do { st = (x); if (st != K4_OK) { k4_srnet_destroy(n); return st; } } while (0)
    SR_TRY(make_conv(n, n->conv_first, P[k], P[k + 1], 64, 3, s)); k += 2;
    SR_TRY(make_condnet(n, P + k, n->num_cond, s)); k += 8;
    for (int i = 0; i < d->num_block; ++i) {
        for (int j = 0; j < 3; ++j) {
            for (int c = 0; c < 5; ++c) {
                const int cin = 64 + 32 * c, cout = (c == 4) ? 64 : 32;
                SR_TRY(make_conv(n, n->rdb_conv[i][j][c], P[k], P[k + 1], cout, cin, s)); k += 2;
            }
            SR_TRY(make_sft(n, n->rdb_sft[i][j][0], P + k, 64, s)); k += 8;
            SR_TRY(make_sft(n, n->rdb_sft[i][j][1], P + k, 32, s)); k += 8;
        }
        SR_TRY(make_sft(n, n->rrdb_sft[i], P + k, 64, s)); k += 8;
    }
    SR_TRY(make_sft(n, n->sftbody, P + k, 64, s)); k += 8;
    SR_TRY(make_conv(n, n->conv_body, P[k], P[k + 1], 64, 64, s)); SR_TRY(make_conv_k64(n, n->conv_body, P[k], 64, 64, false, s)); k += 2;
    if (up) {
        SR_TRY(make_conv(n, n->conv_up1, P[k], P[k + 1], 64, 64, s)); SR_TRY(make_conv_phases(n, n->conv_up1, P[k], 64, 64, s)); SR_TRY(make_conv_k64(n, n->conv_up1, P[k], 64, 64, true, s)); k += 2;
        SR_TRY(make_conv(n, n->conv_up2, P[k], P[k + 1], 64, 64, s)); SR_TRY(make_conv_phases(n, n->conv_up2, P[k], 64, 64, s)); SR_TRY(make_conv_k64(n, n->conv_up2, P[k], 64, 64, true, s)); k += 2;
    }
    SR_TRY(make_conv(n, n->conv_hr, P[k], P[k + 1], 64, 64, s)); SR_TRY(make_conv_k64(n, n->conv_hr, P[k], 64, 64, false, s)); k += 2;
    SR_TRY(make_conv(n, n->conv_last, P[k], P[k + 1], 3, 64, s)); SR_TRY(make_conv_k64(n, n->conv_last, P[k], 3, 64, false, s)); k += 2;
#undef SR_TRY
    *out = n;
    return K4_OK;
}

// workspace layout for an h x w tile (P = h*w LR pixels) of a x`scale` net: x1 has no up1 / up2, and hr is at LR
struct SrWs { size_t in16, cond32, cond16, feat, trunkA, trunkB, cat, cat2, sbody, bf, up1, up2, hr, total; };
static SrWs sr_ws(int h, int w, int scale) {
    const size_t P = (size_t)h * w;
    SrWs o; size_t off = 0;
    auto take = [&](size_t b) { size_t r = off; off += (b + 255) & ~(size_t)255; return r; };
    o.in16 = take(P * 32 * 2); o.cond32 = take(P * 32 * 4); o.feat = take(P * 64 * 4);
    o.trunkA = take(P * 64 * 4); o.trunkB = take(P * 64 * 4); o.cat = take(P * 192 * 2);
    o.cat2 = take(P * 192 * 2); o.cond16 = take(P * 32 * 2);         // fused SFT epilogues: dense blocks alternate between two concat buffers
    o.sbody = take(P * 64 * 2); o.bf = take(P * 64 * 2);
    o.up1 = o.up2 = 0;
    if (scale == 4) { o.up1 = take(P * 4 * 64 * 2); o.up2 = take(P * 16 * 64 * 2); }
    o.hr = take(P * scale * scale * 64 * 2);
    o.total = off;
    return o;
}

extern "C" size_t k4_srnet_workspace_bytes(const k4_srnet* n, int32_t h, int32_t w) {
    if (h <= 0 || w <= 0) return 0;
    return sr_ws(h, w, n ? n->scale : 4).total;          // no net: the x4 layout, the largest of the built scales
}

// Rows [lo, hi) of an h-row tile that a layer must produce when `r` more rows of receptive field follow it
// (keep rows [ky0, ky1)); clipped to the tile -- beyond it the convolutions see their zero padding.
struct SrRows { int lo, hi; };
static inline SrRows sr_rows(int ky0, int ky1, int r, int h) {
    SrRows o; o.lo = ky0 - r < 0 ? 0 : ky0 - r; o.hi = ky1 + r > h ? h : ky1 + r; return o;
}

// k4_testing_srnet_forward_upto: the steps of a forward are recorded, and it returns after stop_after of them.  The
// production forward passes no trace.
struct SrTrace { int stop_after, max_steps, n; k4_sr_step* steps; };
static inline bool sr_step(SrTrace* t, int kind, int i, int j, int c, int fused) {
    if (!t) return false;
    if (t->n < t->max_steps) t->steps[t->n] = k4_sr_step{kind, i, j, c, fused};
    return ++t->n >= t->stop_after;
}

static int srnet_forward_roi_impl(const k4_srnet* n, const float* d_x, const float* d_cond, int32_t h, int32_t w,
                                  int32_t keep_y0, int32_t keep_y1, int32_t keep_x0, int32_t keep_x1,
                                  float* d_out, int64_t out_plane_stride, int64_t out_row_stride,
                                  int32_t n_extra, float* const* h_extra,
                                  void* d_ws, size_t ws_bytes, k4_stream_t stream, SrTrace* tr = nullptr) {
    if (!n || !d_x || !d_cond || !d_out || h <= 0 || w <= 0) return K4_ERR_INVALID_ARG;
    if (n_extra < 0 || n_extra > K4_MAX_PEERS - 1 || (n_extra > 0 && !h_extra)) return K4_ERR_INVALID_ARG;
    for (int e = 0; e < n_extra; ++e) if (!h_extra[e]) return K4_ERR_INVALID_ARG;
    if (keep_y0 < 0 || keep_y1 > h || keep_y0 >= keep_y1 || keep_x0 < 0 || keep_x1 > w || keep_x0 >= keep_x1) return K4_ERR_INVALID_ARG;
    const int sc = n->scale;
    const SrWs L = sr_ws(h, w, sc);
    if (!d_ws || ws_bytes < L.total) return K4_ERR_WORKSPACE;
    cudaStream_t s = (cudaStream_t)stream;
    unsigned char* ws = (unsigned char*)d_ws;
    const long long P = (long long)h * w;
    __half* in16 = (__half*)(ws + L.in16); float* cond32 = (float*)(ws + L.cond32); float* feat = (float*)(ws + L.feat);
    float* tA = (float*)(ws + L.trunkA); float* tB = (float*)(ws + L.trunkB); __half* cat = (__half*)(ws + L.cat);
    __half* sbody = (__half*)(ws + L.sbody); __half* bf = (__half*)(ws + L.bf);
    __half* up1 = (__half*)(ws + L.up1); __half* up2 = (__half*)(ws + L.up2); __half* hr = (__half*)(ws + L.hr);
    __half* cat2 = (__half*)(ws + L.cat2); __half* cond16 = (__half*)(ws + L.cond16);
    // K4_SR_FUSE_SFT=0: every SFT layer as its own sft_mma_kernel pass (kept as the A/B reference of the fused epilogues)
    const char* fenv = getenv("K4_SR_FUSE_SFT");                   // read per call: tests compare both structures in one process
    const bool fuse = !(fenv && fenv[0] == '0') && !sr_no_tma();
    const int ky0 = keep_y0, ky1 = keep_y1;
    // Remaining receptive radius (LR rows) behind each layer, from the output backwards: at x4 conv_last / conv_hr / up2 / up1
    // need 1/4 + 1/4 + 1/4 + 1/2 LR rows (handled exactly in high-resolution rows below), at x1 conv_last / conv_hr run at LR
    // and need 1 + 1; either way conv_body's output bf is needed on rows(2), so what follows is the same for both scales:
    // conv_body 1, every 3x3 conv of a residual dense block 1 (SFT layers 0), conv_first 1: the trunk entering conv_body's SFT
    // is needed on rows(3), the output of the k-th dense block from the end on rows(3 + 5k), conv_first's on
    // rows(3 + 5 * 3 * num_block).
    const int nrdb = 3 * n->num_block;
    int st;
#define SR_DO(x, ...) do { st = (x); if (st != K4_OK) return st; if (sr_step(tr, __VA_ARGS__)) return K4_OK; } while (0)
    K4_CUDA_TRY(sr_launch(nchw_to_nhwc32_kernel, (unsigned)((P * 32 + 255) / 256), 256, 0, s, d_x, in16, 3, P));
    if (sr_step(tr, K4_SR_STEP_INPUT, -1, -1, -1, 0)) return K4_OK;
    {
        const SrRows rr = sr_rows(ky0, ky1, 3 + 5 * nrdb + 5, h);          // every SFT layer inside the window reads it
        SR_DO(run_condnet(n, d_cond, h, w, rr.lo, rr.hi, cond32, fuse ? cond16 : nullptr, s), K4_SR_STEP_CONDNET, -1, -1, -1, 0);
    }
    ConvParams c0{};
    c0.H = h; c0.W = w;
    auto rows = [&](ConvParams& p, int r) { const SrRows q = sr_rows(ky0, ky1, r, h); p.y_lo = q.lo; p.y_hi = q.hi; };
    auto win = [&](SftParams& sp, int r) { const SrRows q = sr_rows(ky0, ky1, r, h); sp.p0 = (long long)q.lo * w; sp.P = (long long)(q.hi - q.lo) * w; };
    if (fuse) {
        // Every SFT layer runs in the epilogue of the convolution that produces its input (epilogue_sft): conv_first -> sft0 of
        // the first dense block, conv4 -> sft1, conv5 -> sft0 of the next block (for the third block of an RRDB: the RRDB
        // tail first, then the next sft0 or sftbody).  A block's conv5 writes the NEXT block's first 64 concat channels while
        // other CTAs still read this block's, so the dense blocks alternate between two concat buffers.
        auto sft_of = [&](int r) -> const SrSft& {                 // sft0 of dense block r (global index), or sftbody after the last
            return r < nrdb ? n->rdb_sft[r / 3][r % 3][0] : n->sftbody;
        };
        auto next_dst = [&](ConvParams& p, int r) {                // where the fused sft0 / sftbody result goes
            if (r < nrdb) { p.dst_h2 = (r & 1) ? cat2 : cat; p.dst2_cstride = 192; p.dst2_c0 = 0; }
            else { p.dst_h2 = sbody; p.dst2_cstride = 64; p.dst2_c0 = 0; }
        };
        {   // feat = conv_first(x) -> feat, trunk A; xc0 = sft0(feat) -> cat[0:64]
            ConvParams p = c0; p.src = in16; p.src_cstride = 32; p.src_c0 = 0; p.mode = SRM_TRUNK_SFT; p.scale = 1.f;
            p.dst_f = feat; p.dst_f2 = tA; p.cond16 = cond16; p.sftw = sft_of(0).frag; p.sft_n = 64; next_dst(p, 0);
            rows(p, 3 + 5 * nrdb);
            SR_DO(run_conv(n->conv_first, p, s), K4_SR_STEP_CONV_FIRST, -1, -1, -1, 1);
        }
        for (int i = 0; i < n->num_block; ++i) {
            const float* cur = tA;
            for (int j = 0; j < 3; ++j) {
                const int r = 3 * i + j, k = nrdb - 1 - r, base = 3 + 5 * k;
                __half* cc = (r & 1) ? cat2 : cat;
                for (int c = 0; c < 4; ++c) {   // x{c+1} = lrelu(conv(cat[0:64+32c])) -> cat[64+32c : 96+32c]; conv4 also applies sft1
                    ConvParams p = c0; p.src = cc; p.src_cstride = 192; p.src_c0 = 0; p.mode = SRM_STORE_F16; p.lrelu = 0.2f;
                    p.dst_h = cc; p.dst_cstride = 192; p.dst_c0 = 64 + 32 * c;
                    if (c == 3) { p.mode = SRM_STORE_F16_SFT; p.cond16 = cond16; p.sftw = n->rdb_sft[i][j][1].frag; p.sft_n = 32; }
                    rows(p, base + 4 - c);
                    SR_DO(run_conv(n->rdb_conv[i][j][c], p, s), K4_SR_STEP_RDB_CONV, i, j, c, c == 3);
                }
                {   // x = conv5(cat) * 0.2 + x, then the SFT layer(s) that read it
                    ConvParams p = c0; p.src = cc; p.src_cstride = 192; p.src_c0 = 0; p.scale = 0.2f; p.add_f = cur;
                    p.cond16 = cond16; p.sft_n = 64;
                    if (j < 2) {
                        p.mode = SRM_TRUNK_SFT; p.dst_f = tB; p.sftw = sft_of(r + 1).frag;
                    } else {            // block tail: out = sft0(x) * 0.2 + x_in -> trunk A, then the next sft0 / sftbody of that
                        p.mode = SRM_TRUNK_SFT2; p.dst_f = tA; p.add_f2 = tA; p.scale2 = 0.2f;
                        p.sftw = n->rrdb_sft[i].frag; p.sftw2 = sft_of(r + 1).frag;
                    }
                    next_dst(p, r + 1);
                    rows(p, base);
                    SR_DO(run_conv(n->rdb_conv[i][j][4], p, s), K4_SR_STEP_RDB_CONV, i, j, 4, 1);
                    cur = tB;
                }
            }
        }
        {   // body_feat = conv_body(sftbody(trunk)) + feat   (sbody was written by the last conv5)
            ConvParams p = c0; p.src = sbody; p.src_cstride = 64; p.mode = SRM_ADD_STORE_F16; p.add_f = feat; p.dst_h = bf; p.dst_cstride = 64;
            rows(p, 2);
            SR_DO(run_conv(n->conv_body, p, s), K4_SR_STEP_CONV_BODY, -1, -1, -1, 0);
        }
    } else {
        {   // feat = conv_first(x): fp32 into `feat` and into trunk A (the initial trunk)
            ConvParams p = c0; p.src = in16; p.src_cstride = 32; p.src_c0 = 0; p.mode = SRM_STORE_F32F16; p.dst_f = feat; p.dst_f2 = tA;
            rows(p, 3 + 5 * nrdb);
            SR_DO(run_conv(n->conv_first, p, s), K4_SR_STEP_CONV_FIRST, -1, -1, -1, 0);
        }
        for (int i = 0; i < n->num_block; ++i) {
            // RRDB_SFT.forward: trunk A holds x (kept for the block's tail), RDBs update A -> B -> B -> B
            const float* cur = tA;
            for (int j = 0; j < 3; ++j) {
                const int k = nrdb - 1 - (3 * i + j);                              // dense blocks still to come
                const int base = 3 + 5 * k;                                        // rows(base): this block's output
                {   // xc0 = sft0(x) -> cat[0:64]
                    SftParams sp{}; sp.cond = cond32; sp.x_f = cur; sp.dst_h = cat; sp.dst_cstride = 192; sp.dst_c0 = 0;
                    win(sp, base + 5);
                    SR_DO(run_sft(n->rdb_sft[i][j][0], sp, s), K4_SR_STEP_SFT0, i, j, -1, 0);
                }
                for (int c = 0; c < 4; ++c) {   // x{c+1} = lrelu(conv(cat[0:64+32c])) -> cat[64+32c : 96+32c]
                    ConvParams p = c0; p.src = cat; p.src_cstride = 192; p.src_c0 = 0; p.mode = SRM_STORE_F16; p.lrelu = 0.2f;
                    p.dst_h = cat; p.dst_cstride = 192; p.dst_c0 = 64 + 32 * c;
                    rows(p, base + 4 - c);
                    SR_DO(run_conv(n->rdb_conv[i][j][c], p, s), K4_SR_STEP_RDB_CONV, i, j, c, 0);
                }
                {   // xc1 = sft1(x4) in place: cat[160:192]
                    SftParams sp{}; sp.cond = cond32; sp.x_h = cat; sp.xh_cstride = 192; sp.xh_c0 = 160;
                    sp.dst_h = cat; sp.dst_cstride = 192; sp.dst_c0 = 160;
                    win(sp, base + 1);
                    SR_DO(run_sft(n->rdb_sft[i][j][1], sp, s), K4_SR_STEP_SFT1, i, j, -1, 0);
                }
                {   // x = conv5(cat) * 0.2 + x
                    ConvParams p = c0; p.src = cat; p.src_cstride = 192; p.src_c0 = 0; p.mode = SRM_TRUNK; p.scale = 0.2f;
                    p.add_f = cur; p.dst_f = tB;
                    rows(p, base);
                    SR_DO(run_conv(n->rdb_conv[i][j][4], p, s), K4_SR_STEP_RDB_CONV, i, j, 4, 0);
                    cur = tB;
                }
            }
            {   // out = sft0(rdb3 out) * 0.2 + x_in  -> A
                SftParams sp{}; sp.cond = cond32; sp.x_f = tB; sp.dst_f = tA; sp.res_f = tA; sp.res_scale = 0.2f;
                win(sp, 3 + 5 * (nrdb - 3 * (i + 1)));
                SR_DO(run_sft(n->rrdb_sft[i], sp, s), K4_SR_STEP_SFT_RRDB, i, -1, -1, 0);
            }
        }
        {   // body_feat = conv_body(sftbody(trunk)) + feat
            SftParams sp{}; sp.cond = cond32; sp.x_f = tA; sp.dst_h = sbody; sp.dst_cstride = 64; sp.dst_c0 = 0;
            win(sp, 3);
            SR_DO(run_sft(n->sftbody, sp, s), K4_SR_STEP_SFT_BODY, -1, -1, -1, 0);
            ConvParams p = c0; p.src = sbody; p.src_cstride = 64; p.mode = SRM_ADD_STORE_F16; p.add_f = feat; p.dst_h = bf; p.dst_cstride = 64;
            rows(p, 2);
            SR_DO(run_conv(n->conv_body, p, s), K4_SR_STEP_CONV_BODY, -1, -1, -1, 0);
        }
    }
    {   // x4: upsample x2 (nearest) + conv + lrelu, twice; then conv_hr + lrelu and conv_last at the output resolution
        // (x4: 4h x 4w from up2; x1: h x w straight from bf), rows in the layer's own resolution
        ConvParams p = c0; p.src = bf; p.src_cstride = 64; p.mode = SRM_STORE_F16; p.lrelu = 0.2f; p.dst_cstride = 64;
        auto clip = [](int v, int hi) { return v < 0 ? 0 : (v > hi ? hi : v); };
        if (sc == 4) {
            p.upsample = 1; p.dst_h = up1;
            p.H = h; p.W = w;                                   // iterate over the SOURCE grid, write the 2x grid
            p.y_lo = clip(ky0 - 1, h); p.y_hi = clip(ky1 + 1, h);                    // -> up1 rows [2ky0-2, 2ky1+2)
            SR_DO(run_conv_up2x(n->conv_up1, p, s), K4_SR_STEP_UP1, -1, -1, -1, 0);
            p.H = 2 * h; p.W = 2 * w; p.src = up1; p.dst_h = up2;
            p.y_lo = clip(2 * ky0 - 1, 2 * h); p.y_hi = clip(2 * ky1 + 1, 2 * h);    // -> up2 rows [4ky0-2, 4ky1+2)
            SR_DO(run_conv_up2x(n->conv_up2, p, s), K4_SR_STEP_UP2, -1, -1, -1, 0);
            p.upsample = 0; p.src = up2;
        }
        p.H = sc * h; p.W = sc * w; p.dst_h = hr;
        p.y_lo = clip(sc * ky0 - 1, sc * h); p.y_hi = clip(sc * ky1 + 1, sc * h);
        SR_DO(run_conv(n->conv_hr, p, s), K4_SR_STEP_HR, -1, -1, -1, 0);
        ConvParams q = c0; q.H = sc * h; q.W = sc * w; q.src = hr; q.src_cstride = 64; q.mode = SRM_OUT_NCHW; q.out_nchw = d_out; q.n_valid = 3;
        q.y_lo = sc * ky0; q.y_hi = sc * ky1;
        q.out_ps = out_plane_stride; q.out_rs = out_row_stride;
        q.crop_y0 = sc * ky0; q.crop_y1 = sc * ky1; q.crop_x0 = sc * keep_x0; q.crop_x1 = sc * keep_x1;
        q.n_out_extra = n_extra;
        for (int e = 0; e < n_extra; ++e) q.out_extra[e] = h_extra[e];
        SR_DO(run_conv(n->conv_last, q, s), K4_SR_STEP_LAST, -1, -1, -1, 0);
    }
#undef SR_DO
    return K4_OK;
}

extern "C" int k4_srnet_forward_roi(const k4_srnet* n, const float* d_x, const float* d_cond, int32_t h, int32_t w,
                                    int32_t keep_y0, int32_t keep_y1, int32_t keep_x0, int32_t keep_x1,
                                    float* d_out, int64_t out_plane_stride, int64_t out_row_stride,
                                    void* d_ws, size_t ws_bytes, k4_stream_t stream) {
    return srnet_forward_roi_impl(n, d_x, d_cond, h, w, keep_y0, keep_y1, keep_x0, keep_x1, d_out, out_plane_stride,
                                  out_row_stride, 0, nullptr, d_ws, ws_bytes, stream);
}

extern "C" int k4_srnet_forward_roi_peers(const k4_srnet* n, const float* d_x, const float* d_cond, int32_t h, int32_t w,
                                          int32_t keep_y0, int32_t keep_y1, int32_t keep_x0, int32_t keep_x1,
                                          float* d_out, int64_t out_plane_stride, int64_t out_row_stride,
                                          int32_t n_extra, float* const* h_extra,
                                          void* d_ws, size_t ws_bytes, k4_stream_t stream) {
    return srnet_forward_roi_impl(n, d_x, d_cond, h, w, keep_y0, keep_y1, keep_x0, keep_x1, d_out, out_plane_stride,
                                  out_row_stride, n_extra, h_extra, d_ws, ws_bytes, stream);
}

extern "C" int k4_srnet_forward(const k4_srnet* n, const float* d_x, const float* d_cond, int32_t h, int32_t w,
                                float* d_out, void* d_ws, size_t ws_bytes, k4_stream_t stream) {
    if (!n) return K4_ERR_INVALID_ARG;
    const int64_t sc = n->scale;
    return k4_srnet_forward_roi(n, d_x, d_cond, h, w, 0, h, 0, w, d_out, sc * sc * h * w, sc * w, d_ws, ws_bytes, stream);
}

// The real forward, stopped after `stop_after` steps, for the test suite: the intermediate buffers stay in the workspace.
extern "C" int k4_testing_srnet_forward_upto(const k4_srnet* n, const float* d_x, const float* d_cond, int32_t h, int32_t w,
                                             int32_t keep_y0, int32_t keep_y1, int32_t keep_x0, int32_t keep_x1,
                                             float* d_out, int64_t out_plane_stride, int64_t out_row_stride,
                                             void* d_ws, size_t ws_bytes, int32_t stop_after,
                                             k4_sr_step* steps, int32_t max_steps, int32_t* n_steps, k4_sr_ws_layout* ws,
                                             k4_stream_t stream) {
    if (n_steps) *n_steps = 0;
    if (!n || !n_steps || !ws || stop_after < 1 || max_steps < 0 || (max_steps > 0 && !steps)) return K4_ERR_INVALID_ARG;
    if (h <= 0 || w <= 0) return K4_ERR_INVALID_ARG;
    const SrWs L = sr_ws(h, w, n->scale);
    *ws = k4_sr_ws_layout{L.in16, L.cond32, L.cond16, L.feat, L.trunkA, L.trunkB, L.cat, L.cat2, L.sbody, L.bf, L.up1, L.up2,
                          L.hr, L.total};
    SrTrace tr{stop_after, max_steps, 0, steps};
    const int st = srnet_forward_roi_impl(n, d_x, d_cond, h, w, keep_y0, keep_y1, keep_x0, keep_x1, d_out, out_plane_stride,
                                          out_row_stride, 0, nullptr, d_ws, ws_bytes, stream, &tr);
    *n_steps = tr.n;
    return st;
}

// One decoder layer for the test suite: a throw-away k4_srnet holds the packs (make_conv & co., as k4_srnet_create
// builds them), run_conv / run_conv_up2x run it with the requested kernel, k4_srnet_destroy frees it.
extern "C" int k4_testing_conv3x3(const k4_conv_test_args* a, int32_t* kernel_used, k4_stream_t stream) {
    if (kernel_used) *kernel_used = -1;
    if (!a || !a->d_weight || !a->d_bias || !a->d_src) return K4_ERR_INVALID_ARG;
    if (a->cout < 1 || a->cout > 64 || a->cin < 1 || a->cin > 192 || a->H < 1 || a->W < 1) return K4_ERR_INVALID_ARG;
    if (a->mode < SRM_STORE_F16 || a->mode > SRM_TRUNK_SFT2) return K4_ERR_INVALID_ARG;
    if (a->kernel < SRK_AUTO || a->kernel > SRK_K64) return K4_ERR_INVALID_ARG;
    if (a->y_lo < 0 || a->y_lo >= a->y_hi || a->y_hi > a->H) return K4_ERR_INVALID_ARG;
    const int cin_pad = (a->cin + 31) / 32 * 32, npad = a->cout <= 16 ? 16 : (a->cout <= 32 ? 32 : 64);
    if (a->src_c0 < 0 || a->src_c0 % 8 || a->src_cstride % 8 || a->src_c0 + cin_pad > a->src_cstride) return K4_ERR_INVALID_ARG;
    const int m = a->mode, oh = a->upsample2x ? 2 * a->H : a->H, ow = a->upsample2x ? 2 * a->W : a->W;
    const bool sft = m >= SRM_STORE_F16_SFT;
    if ((m == SRM_STORE_F16 || m == SRM_ADD_STORE_F16 || m == SRM_STORE_F16_SFT) &&
        (!a->d_dst_h || a->dst_c0 < 0 || a->dst_c0 % 2 || a->dst_cstride % 2 || a->dst_c0 + npad > a->dst_cstride))
        return K4_ERR_INVALID_ARG;
    if ((m == SRM_TRUNK || m == SRM_ADD_STORE_F16) && !a->d_add_f) return K4_ERR_INVALID_ARG;
    if ((m == SRM_TRUNK || m == SRM_STORE_F32F16 || m == SRM_TRUNK_SFT || m == SRM_TRUNK_SFT2) && !a->d_dst_f) return K4_ERR_INVALID_ARG;
    if (m == SRM_OUT_NCHW && (!a->d_out_nchw || a->n_valid < 1 || a->n_valid > npad || a->out_plane_stride < 1 || a->out_row_stride < 1 ||
                              a->crop_y0 < 0 || a->crop_y0 >= a->crop_y1 || a->crop_y1 > oh ||
                              a->crop_x0 < 0 || a->crop_x0 >= a->crop_x1 || a->crop_x1 > ow))
        return K4_ERR_INVALID_ARG;
    if (sft) {
        if (!a->d_cond16 || !a->h_sft || (m != SRM_STORE_F16_SFT && (!a->d_dst_h2 || a->dst2_c0 < 0 || a->dst2_c0 % 2 ||
                                                                     a->dst2_cstride % 2 || a->dst2_c0 + npad > a->dst2_cstride)))
            return K4_ERR_INVALID_ARG;
        if (m == SRM_TRUNK_SFT2 && (!a->d_add_f2 || !a->h_sft2)) return K4_ERR_INVALID_ARG;
        for (int i = 0; i < 8; ++i)
            if (!a->h_sft[i] || (m == SRM_TRUNK_SFT2 && !a->h_sft2[i])) return K4_ERR_INVALID_ARG;
    }
    // built combinations only: SFT layers of 32 / 64 channels behind a direct convolution, the two-layer tail at 64
    if (sft && (a->upsample2x || a->cout != npad || npad == 16 || (m == SRM_TRUNK_SFT2 && npad != 64))) return K4_ERR_UNSUPPORTED;
    int st = k4_device_check();
    if (st != K4_OK) return st;

    cudaStream_t s = (cudaStream_t)stream;
    k4_srnet* n = new (std::nothrow) k4_srnet();
    if (!n) return K4_ERR_INVALID_ARG;
    memset(n, 0, sizeof(*n));
    SrConv& c = n->conv_first;
    SrSft& f1 = n->sftbody;
    SrSft& f2 = n->rrdb_sft[0];
    st = make_conv(n, c, a->d_weight, a->d_bias, a->cout, a->cin, s);
    if (!st && a->upsample2x) st = make_conv_phases(n, c, a->d_weight, a->cout, a->cin, s);
    if (!st) st = make_conv_k64(n, c, a->d_weight, a->cout, a->cin, a->upsample2x != 0, s);
    if (!st && sft) st = make_sft(n, f1, a->h_sft, a->cout, s);
    if (!st && m == SRM_TRUNK_SFT2) st = make_sft(n, f2, a->h_sft2, 64, s);
    int used = -1;
    if (!st) {
        ConvParams p{};
        p.src = static_cast<const __half*>(a->d_src); p.src_cstride = a->src_cstride; p.src_c0 = a->src_c0;
        p.H = a->H; p.W = a->W; p.y_lo = a->y_lo; p.y_hi = a->y_hi;
        p.mode = m; p.lrelu = a->lrelu; p.scale = a->scale; p.scale2 = a->scale2;
        p.dst_h = static_cast<__half*>(a->d_dst_h); p.dst_cstride = a->dst_cstride; p.dst_c0 = a->dst_c0;
        p.dst_f = a->d_dst_f; p.dst_f2 = a->d_dst_f2; p.add_f = a->d_add_f; p.add_f2 = a->d_add_f2;
        p.dst_h2 = static_cast<__half*>(a->d_dst_h2); p.dst2_cstride = a->dst2_cstride; p.dst2_c0 = a->dst2_c0;
        p.out_nchw = a->d_out_nchw; p.n_valid = a->n_valid; p.out_ps = a->out_plane_stride; p.out_rs = a->out_row_stride;
        p.crop_y0 = a->crop_y0; p.crop_y1 = a->crop_y1; p.crop_x0 = a->crop_x0; p.crop_x1 = a->crop_x1;
        p.cond16 = static_cast<const __half*>(a->d_cond16);
        if (sft) { p.sftw = f1.frag; p.sft_n = a->cout; }
        if (m == SRM_TRUNK_SFT2) p.sftw2 = f2.frag;
        st = a->upsample2x ? run_conv_up2x(c, p, s, a->kernel, &used) : run_conv(c, p, s, nullptr, a->kernel, &used);
    }
    const cudaError_t e = cudaStreamSynchronize(s);       // the packs are freed below
    if (st == K4_OK && e != cudaSuccess) { k4_set_cuda_error(e, "k4_testing_conv3x3"); st = K4_ERR_CUDA; }
    k4_srnet_destroy(n);
    if (st == K4_OK && kernel_used) *kernel_used = used;
    return st;
}

// CondNet for the test suite: a throw-away k4_srnet holds the packs (make_condnet, as k4_srnet_create builds them),
// run_condnet runs them with the requested kernel and the decoder's grid, k4_srnet_destroy frees them.
extern "C" int k4_testing_condnet(const k4_condnet_test_args* a, int32_t* kernel_used, k4_stream_t stream) {
    if (kernel_used) *kernel_used = -1;
    if (!a || !a->h_condnet || !a->d_cond_in || !a->d_cond_out) return K4_ERR_INVALID_ARG;
    for (int i = 0; i < 8; ++i) if (!a->h_condnet[i]) return K4_ERR_INVALID_ARG;
    if (a->H < 1 || a->W < 1 || (long long)a->H * a->W > (1LL << 30)) return K4_ERR_INVALID_ARG;
    if (a->y_lo < 0 || a->y_lo >= a->y_hi || a->y_hi > a->H) return K4_ERR_INVALID_ARG;
    if (a->kernel < SRP_AUTO || a->kernel > SRP_FP32) return K4_ERR_INVALID_ARG;
    if (a->num_cond < 0 || a->num_cond > 64) return K4_ERR_INVALID_ARG;
    if (((uintptr_t)a->d_cond_in & 3) || ((uintptr_t)a->d_cond_out & 7) || ((uintptr_t)a->d_cond16 & 3)) return K4_ERR_INVALID_ARG;
    int st = k4_device_check();
    if (st != K4_OK) return st;

    cudaStream_t s = (cudaStream_t)stream;
    k4_srnet* n = new (std::nothrow) k4_srnet();
    if (!n) return K4_ERR_INVALID_ARG;
    memset(n, 0, sizeof(*n));
    n->num_cond = a->num_cond ? a->num_cond : 1;
    int used = -1;
    st = make_condnet(n, a->h_condnet, n->num_cond, s);
    if (!st) st = run_condnet(n, a->d_cond_in, a->H, a->W, a->y_lo, a->y_hi, a->d_cond_out, static_cast<__half*>(a->d_cond16), s,
                              a->kernel, &used);
    const cudaError_t e = cudaStreamSynchronize(s);       // the packs are freed below
    if (st == K4_OK && e != cudaSuccess) { k4_set_cuda_error(e, "k4_testing_condnet"); st = K4_ERR_CUDA; }
    k4_srnet_destroy(n);
    if (st == K4_OK && kernel_used) *kernel_used = used;
    return st;
}

// One SFT layer as its own pass for the test suite: make_sft packs it as k4_srnet_create does, run_sft runs it.
extern "C" int k4_testing_sft(const k4_sft_test_args* a, int32_t* kernel_used, k4_stream_t stream) {
    if (kernel_used) *kernel_used = -1;
    if (!a || !a->h_sft || !a->d_cond) return K4_ERR_INVALID_ARG;
    for (int i = 0; i < 8; ++i) if (!a->h_sft[i]) return K4_ERR_INVALID_ARG;
    if (a->cout != 32 && a->cout != 64) return K4_ERR_INVALID_ARG;
    if (a->kernel < SRP_AUTO || a->kernel > SRP_FP32) return K4_ERR_INVALID_ARG;
    if (a->p0 < 0 || a->P < 1 || a->P > (1LL << 30)) return K4_ERR_INVALID_ARG;
    if (!a->d_x_f == !a->d_x_h || !a->d_dst_h == !a->d_dst_f) return K4_ERR_INVALID_ARG;       // exactly one input, one output
    if (a->d_x_h && (a->xh_c0 < 0 || a->xh_c0 % 2 || a->xh_cstride % 2 || a->xh_c0 + a->cout > a->xh_cstride)) return K4_ERR_INVALID_ARG;
    if (a->d_dst_h && (a->dst_c0 < 0 || a->dst_c0 % 8 || a->dst_cstride % 8 || a->dst_c0 + a->cout > a->dst_cstride)) return K4_ERR_INVALID_ARG;
    if (a->d_dst_f && !a->d_res_f) return K4_ERR_INVALID_ARG;
    if (((uintptr_t)a->d_cond & 15) || ((uintptr_t)a->d_x_f & 7) || ((uintptr_t)a->d_x_h & 3) || ((uintptr_t)a->d_dst_h & 15) ||
        ((uintptr_t)a->d_dst_f & 7) || ((uintptr_t)a->d_res_f & 7))
        return K4_ERR_INVALID_ARG;
    int st = k4_device_check();
    if (st != K4_OK) return st;

    cudaStream_t s = (cudaStream_t)stream;
    k4_srnet* n = new (std::nothrow) k4_srnet();
    if (!n) return K4_ERR_INVALID_ARG;
    memset(n, 0, sizeof(*n));
    int used = -1;
    st = make_sft(n, n->sftbody, a->h_sft, a->cout, s);
    if (!st) {
        SftParams p{};
        p.cond = a->d_cond;
        p.x_f = a->d_x_f; p.x_h = static_cast<const __half*>(a->d_x_h); p.xh_cstride = a->xh_cstride; p.xh_c0 = a->xh_c0;
        p.dst_h = static_cast<__half*>(a->d_dst_h); p.dst_cstride = a->dst_cstride; p.dst_c0 = a->dst_c0;
        p.dst_f = a->d_dst_f; p.res_f = a->d_res_f; p.res_scale = a->res_scale;
        p.p0 = a->p0; p.P = a->P;
        st = run_sft(n->sftbody, p, s, a->kernel, &used);
    }
    const cudaError_t e = cudaStreamSynchronize(s);       // the packs are freed below
    if (st == K4_OK && e != cudaSuccess) { k4_set_cuda_error(e, "k4_testing_sft"); st = K4_ERR_CUDA; }
    k4_srnet_destroy(n);
    if (st == K4_OK && kernel_used) *kernel_used = used;
    return st;
}

// ------------------------------------------------------------------------------------------------
// The decoder's 3x3 convolutions for another network: LPIPS's VGG16 trunk (k4_lpips.cu), in fp32-class precision from
// fp16 operands.  A value x is carried as hi = fp16(x) and lo = fp16(x - hi) (both for activations and weights), and a
// layer is the one GEMM of K = 3 Cin over the activation channels [hi | lo | hi] and the weights [w_hi | w_hi | w_lo]:
// a_hi w_hi + a_lo w_hi + a_hi w_lo, only a_lo w_lo (2^-22 relative) dropped.  Cout is cut into blocks of 64 output
// channels, each packed as the decoder packs a 64-channel conv and run by run_conv as one N = 64 launch whose epilogue
// writes its channels of the three copies.
// ------------------------------------------------------------------------------------------------
namespace {
// w [cout][cin][3][3] -> [cout][3 cin][3][3]: w_hi, w_hi, w_lo as fp32 values (each exact in fp16)
__global__ void split_conv_weights_kernel(const float* __restrict__ w, float* __restrict__ dst, int cout, int cin) {
    const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= (long long)cout * 3 * cin * 9) return;
    const int t = (int)(i % 9);
    const long long r = i / 9;
    const int k = (int)(r % (3 * cin)), co = (int)(r / (3 * cin));
    const float v = w[((long long)co * cin + k % cin) * 9 + t];
    const float hi = __half2float(__float2half_rn(v));
    dst[i] = k < 2 * cin ? hi : __half2float(__float2half_rn(v - hi));
}
}  // namespace

int k4_conv3x3_pack(const float* w, const float* b, int cout, int cin, cudaStream_t s, K4Conv3x3Pack* c) {
    if (!w || !b || !c || cout < 64 || cout % 64 || cin < 1) return K4_ERR_INVALID_ARG;
    *c = K4Conv3x3Pack{};
    c->cout = cout;
    c->cin = cin;
    c->cin_pad = (3 * cin + 31) / 32 * 32;
    const int nsl = c->cin_pad / SR_CK, nblk = cout / 64;
    c->ws_bytes = (size_t)nsl * 9 * 64 * SR_CK * 2;                 // a multiple of 1024 B: every block stays aligned
    const size_t nsplit = (size_t)cout * 3 * cin * 9;
    K4_CUDA_TRY(cudaMalloc(&c->blob, nblk * c->ws_bytes + (size_t)cout * 4 + nsplit * 4));
    unsigned char* blob = static_cast<unsigned char*>(c->blob);
    c->wpack = blob;
    c->bias = reinterpret_cast<float*>(blob + nblk * c->ws_bytes);
    float* wsplit = c->bias + cout;                                  // staging of the split weights
    split_conv_weights_kernel<<<(unsigned)((nsplit + 255) / 256), 256, 0, s>>>(w, wsplit, cout, cin);
    for (int nb = 0; nb < nblk; ++nb) {
        const long long total = (long long)nsl * 9 * 64 * SR_CK;
        pack_conv3x3_kernel<<<(unsigned)((total + 255) / 256), 256, 0, s>>>(wsplit + (size_t)nb * 64 * 3 * cin * 9,
                                                                          c->wpack + nb * c->ws_bytes, 64, 3 * cin, 64, nsl);
    }
    K4_CUDA_TRY(cudaGetLastError());
    K4_CUDA_TRY(cudaMemcpyAsync(c->bias, b, (size_t)cout * 4, cudaMemcpyDeviceToDevice, s));
    return K4_OK;
}

void k4_conv3x3_free(K4Conv3x3Pack* c) {
    if (c && c->blob) cudaFree(c->blob);
    if (c) *c = K4Conv3x3Pack{};
}

int k4_conv3x3_relu_split(const K4Conv3x3Pack& c, const __half* src, int H, int W, __half* dst, cudaStream_t s) {
    for (int nb = 0; nb < c.cout / 64; ++nb) {
        SrConv sc{};
        sc.wpack = c.wpack + nb * c.ws_bytes;
        sc.bias = c.bias + 64 * nb;
        sc.cin_pad = c.cin_pad;
        sc.cout = sc.npad = 64;
        ConvParams p{};
        p.src = src; p.src_cstride = c.cin_pad; p.src_c0 = 0;
        p.H = H; p.W = W;
        p.mode = SRM_STORE_F16; p.relu = 1; p.split = c.cout;
        p.dst_h = dst; p.dst_cstride = 3 * c.cout; p.dst_c0 = 64 * nb;
        if (int st = run_conv(sc, p, s)) return st;
    }
    return K4_OK;
}
