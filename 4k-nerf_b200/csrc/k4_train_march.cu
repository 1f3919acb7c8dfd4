// k4_train_march.cu -- one scene-training step's render and loss in two kernels (include/k4nerf.h,
// k4_train_march_args): the training forward of DirectVoxGO / DirectMPIGO and run_sr.py's composite loss
// (run_sr.py:521-546 without nearclip), then its gradient.  The materialised path (k4nerf/train_forward.py) builds
// the flat sample list, compacts it three times with host syncs and runs autograd through a few dozen ops; here
//   tm_forward_kernel   one thread per ray marches it with the marchers' own device code (k4_march_ray.cuh:
//                       setup_ray, march_step<KIND, false>), so sample points, the alpha and weight thresholds, the
//                       double-precision transmittance and the T < 1e-3 stop are the materialised path's exactly;
//                       gathers k0 from the planar grid in grid_sample_fwd_kernel's corner order and FMA chain, runs
//                       the rgbnet in fp32 in the fp32 marcher mode's operation order, and writes rgb_marched,
//                       alphainv_last and the ray's totals (rgb_feature, sum w, sum w s, the distortion pair sum and
//                       sum w^2, the rgbper sum) to the workspace.
//   tm_loss_kernel      one CTA: the loss terms from the per-ray totals in a fixed order (fp64, no atomics), and the
//                       distortion divisor n = largest shaded ray id + 1.
//   tm_backward_kernel  re-marches every ray with the same code (every T_i and every threshold decision is bit-identical
//                       to the forward), recomputes each shaded sample's activations and backpropagates:
//                         dL/dw_i      g_rgbm . c_i + distortion term (its suffixes W>i, WM>i as total - prefix),
//                                      in fp64
//                         dL/dalpha_i  dL/dw_i T_i - B_i / (1 - alpha_i + 1e-10)  (Alphas2Weights.backward,
//                                      render_utils_kernel.cu:654-677), B_i = g_last T_last + sum_{j>i} dL/dw_j w_j
//                                      taken as the forward's total minus the running prefix, both in fp64 (TmRay)
//                         dL/dx_i      Raw2Alpha.backward's double product chain (render_utils_kernel.cu:507-530)
//                       and scatters dL/d density and dL/d k0 into the grid gradients with fp32 atomics, as
//                       grid_sample_bwd_kernel does.  Samples below the alpha threshold or past the stop get nothing;
//                       samples dropped by the weight threshold act through T only.
// rgbnet weight gradients are batched per warp: the warp marches its 32 rays step by step in lockstep, and at a step
// where any lane shades, every lane stages its sample's layer inputs and output deltas in shared memory (zeros for a lane
// without one); the warp forms dW = dY^T H over the 32 rows and adds it with one atomic per weight, never one per sample.
#include <cmath>
#include <cstring>
#include "k4_internal.cuh"
#include "k4_march_common.cuh"
#include "k4_march_ray.cuh"

namespace {

constexpr int TM_T = 32;                  // threads (rays) per CTA: one warp, so 4096 rays still fill 128 SMs
constexpr int TM_WARPS = TM_T / 32;
constexpr int TM_MAX_K0 = 32;
constexpr int TM_MAX_W = 128;
constexpr int TM_RED_T = 1024;

// Per-ray totals of the forward, read by the loss pass and the backward.  The totals the backward subtracts its
// running prefixes from are fp64: the suffix B_i = total - prefix is divided by fp32(1 - alpha_i) + 1e-10, which is
// 1e-10 for a near-opaque sample whose alpha rounds to 1, and an fp32 residual of the empty suffix behind the ray's last
// sample (a few ulp of the total) would come out of that division as a gradient.  In fp64 the residual is 2^-29 times
// smaller than any fp32 term of the gradient.
struct TmRay {
    double rgbf[3];                       // rgb_feature (sum w c)
    double w_sum, ws_sum;                 // sum w, sum w s over the shaded samples
    double pair;                          // sum_i w_i (s_i W<i - WM<i)
    double w2;                            // sum w^2
    float rgbm[3];                        // rgb_marched (the fp32 output)
    float T;                              // alphainv_last
    float per;                            // sum w |c - target|^2
    int n_shaded;
};
static_assert(sizeof(TmRay) == 80, "workspace layout");
struct TmHeader { long long n_dist; long long reserved; };

struct TmParams {
    K4Dev s;                              // geometry, mask, density, thresholds: what march_step reads
    K4RenderParams rp;
    long long N, nvox;
    const float *ro, *rd, *vd, *tgt, *bkgd;
    const float* k0;                      // planar [C, X, Y, Z]
    const float* W[3];
    const float* B[3];
    int n_in[3], n_out[3];
    float w_main, w_ent, w_dist, w_rp;
    float* rgbm;
    float* alphainv;
    float* loss;
    float* terms;
    float* g_den;
    float* g_k0;
    float* gW[3];
    float* gB[3];
    TmRay* tot;
    TmHeader* hdr;
    const float* g_loss;
    int ks;                               // row stride of the staged layer inputs (floats)
    int ds;                               // row stride of the staged output deltas
};

// ---------------------------------------------------------------------------------------------
// one sample's colour: k0 gather (grid_sample_fwd_kernel's order), rgbnet (mlp_fp32's order), sigmoid.  Keeps the
// layer inputs and pre-activations for the backward.
// ---------------------------------------------------------------------------------------------
struct Shade {
    float k0[TM_MAX_K0];
    float x[K4_MAX_DIM0];
    float z1[TM_MAX_W], h1[TM_MAX_W], z2[TM_MAX_W], h2[TM_MAX_W];
    float logit[3], c[3];
    int n_x;
};

template <int ACT>
__device__ __forceinline__ void tm_layer(const TmParams& p, int l, const float* in, float* z, float* h) {
    const int nin = p.n_in[l], nout = p.n_out[l];
    const float* __restrict__ W = p.W[l];
    const float* __restrict__ B = p.B[l];
    for (int j = 0; j < nout; ++j) {
        float acc = __ldg(B + j);
        const float* w = W + (size_t)j * nin;
        for (int k = 0; k < nin; ++k) acc = __fmaf_rn(in[k], __ldg(w + k), acc);
        if (z) z[j] = acc;
        h[j] = (l == 2) ? acc : RgbAct<ACT>::fp32(acc, p.s);
    }
}

template <int KIND, int ACT, bool KEEP>
__device__ __forceinline__ void tm_shade(const TmParams& p, const Cell& cell, const float cw[8], const int cidx[8],
                                         const float* vemb, int n_vemb, Shade& sh) {
    const int C = p.s.C;
    for (int c = 0; c < C; ++c) {
        const float* g = p.k0 + (long long)c * p.nvox;
        float acc = __fmul_rn(__ldg(g + cidx[0]), cw[0]);
#pragma unroll
        for (int k = 1; k < 8; ++k) acc = __fmaf_rn(__ldg(g + cidx[k]), cw[k], acc);
        sh.k0[c] = acc;
    }
    if (p.s.depth == 0) {
        for (int c = 0; c < 3; ++c) sh.logit[c] = sh.k0[c];
    } else {
        int n = 0;
        for (int c = p.s.k0_view_off; c < C; ++c) sh.x[n++] = sh.k0[c];
        if (KIND == K4_KIND_DMPIGO) {
            const float pe[3] = {cell.cz, cell.cy, cell.cx};      // .flip(-1), lib/dmpigo.py:338
            n += embed3(pe, p.s.spape, sh.x + n);
        }
        for (int c = 0; c < n_vemb; ++c) sh.x[n++] = vemb[c];
        sh.n_x = n;
        tm_layer<ACT>(p, 0, sh.x, KEEP ? sh.z1 : nullptr, sh.h1);          // pre-activations: the backward's only
        tm_layer<ACT>(p, 1, sh.h1, KEEP ? sh.z2 : nullptr, sh.h2);
        tm_layer<ACT>(p, 2, sh.h2, nullptr, sh.logit);
        if (KIND == K4_KIND_DVGO && !p.s.direct)
            for (int c = 0; c < 3; ++c) sh.logit[c] = __fadd_rn(sh.logit[c], sh.k0[c]);
    }
    for (int c = 0; c < 3; ++c) sh.c[c] = sigmoid_ref(sh.logit[c]);
}

// d act / d z times dh (torch's backward of relu / leaky_relu / exp(-x**2 / (2*a**2)))
template <int ACT>
__device__ __forceinline__ float act_bwd(float dh, float z, float h, const K4Dev& s) {
    if constexpr (ACT == K4_ACT_GAUSS) {
        return __fmul_rn(-__fdiv_rn(__fmul_rn(dh, h), s.act_den), __fmul_rn(2.f, z));
    } else if constexpr (ACT == K4_ACT_LKRELU) {
        return z > 0.f ? dh : __fmul_rn(dh, 0.01f);
    } else {
        return z > 0.f ? dh : 0.f;
    }
}

// alpha and exp(x) of an occupied sample: march_step's expression (Raw2Alpha, render_utils_kernel.cu:439-441) on the
// same corner weights, so the value is the one march_step compared with the threshold
template <int KIND>
__device__ __forceinline__ float sample_alpha(const K4Dev& s, const K4RenderParams& rp, const Cell& cell, const float cw[8],
                                              const int cidx[8], float& e) {
    float den = interp_density(s, cw, cidx);
    float shift = s.act_shift;
    if (KIND == K4_KIND_DMPIGO) {
        const int z0 = cell.z0, z1 = cell.z0 + 1;
        float a = 0.f;
        if (z0 >= 0 && z0 < s.mpi_depth) a = __fmul_rn(__ldg(s.act_grid + z0), cell.wz0);
        if (z1 >= 0 && z1 < s.mpi_depth) a = __fmaf_rn(__ldg(s.act_grid + z1), cell.wz1, a);
        den = __fadd_rn(den, a);
        shift = 0.f;
    }
    e = expf(__fadd_rn(den, shift));
    return __fsub_rn(1.f, powf(__fadd_rn(1.f, e), -rp.interval));
}

__device__ __forceinline__ float sample_s(const K4RenderParams& rp, int i) {
    return __fmul_rn(__fadd_rn((float)i, 0.5f), rp.inv_nsamples);       // (step_id + 0.5) / n_max
}

// ---------------------------------------------------------------------------------------------
// forward
// ---------------------------------------------------------------------------------------------
template <int KIND, int ACT>
__global__ void __launch_bounds__(TM_T) tm_forward_kernel(const __grid_constant__ TmParams p) {
    const long long r = (long long)blockIdx.x * TM_T + threadIdx.x;
    if (r >= p.N) return;
    const Ray ray = setup_ray<KIND>(p.s, p.rp, ld3(p.ro, r), ld3(p.rd, r));
    float vemb[3 + 6 * 10];
    int n_vemb = 0;
    if (p.s.depth > 0) {
        const Vec3 v = ld3(p.vd, r);
        const float vv[3] = {v.x, v.y, v.z};
        n_vemb = embed3(vv, p.s.viewpe, vemb);
    }
    const Vec3 t = ld3(p.tgt, r);
    MarchState<KIND> st(true);
    float acc[3] = {0.f, 0.f, 0.f}, per = 0.f;
    double accd[3] = {0.0, 0.0, 0.0}, wp = 0.0, wsp = 0.0, pair = 0.0, w2 = 0.0;
    int n_sh = 0;
    const float mpi_den = (float)(p.rp.n_samples - 1);
    Shade sh;
    for (int i = 0; !st.done && i < ray.n_steps; ++i) {
        float w = 0.f;
        Cell cell;
        float cw[8];
        int cidx[8];
        if (!march_step<KIND, false>(p.s, p.rp, ray, mpi_den, st, i, w, cell, cw, cidx)) continue;
        tm_shade<KIND, ACT, false>(p, cell, cw, cidx, vemb, n_vemb, sh);
        for (int c = 0; c < 3; ++c) {
            acc[c] = __fadd_rn(acc[c], __fmul_rn(w, sh.c[c]));
            accd[c] = fma((double)w, (double)sh.c[c], accd[c]);
        }
        ++n_sh;
        if (p.w_dist > 0.f) {
            const double s = sample_s(p.rp, i), wd = w;
            pair = fma(wd, s * wp - wsp, pair);
            w2 = fma(wd, wd, w2);
            wp += wd;
            wsp = fma(wd, s, wsp);
        }
        if (p.w_rp > 0.f) {
            const float d0 = __fsub_rn(sh.c[0], t.x), d1 = __fsub_rn(sh.c[1], t.y), d2 = __fsub_rn(sh.c[2], t.z);
            per = __fmaf_rn(w, __fmaf_rn(d2, d2, __fmaf_rn(d1, d1, __fmul_rn(d0, d0))), per);
        }
    }
    TmRay o;
    for (int c = 0; c < 3; ++c) {
        const float bg = p.bkgd ? __ldg(p.bkgd + 3 * r + c) : p.rp.bg;
        o.rgbf[c] = accd[c];
        o.rgbm[c] = __fadd_rn(acc[c], __fmul_rn(st.T, bg));            // rgb_feature + alphainv_last * bg
        p.rgbm[3 * r + c] = o.rgbm[c];
    }
    o.T = st.T;
    p.alphainv[r] = st.T;
    o.w_sum = wp; o.ws_sum = wsp; o.pair = pair; o.w2 = w2; o.per = per; o.n_shaded = n_sh;
    p.tot[r] = o;
}

// ---------------------------------------------------------------------------------------------
// the loss: one CTA, every thread a contiguous chunk of rays, fp64 sums, then a fixed-order CTA reduction
// ---------------------------------------------------------------------------------------------
template <typename T, typename Op>
__device__ __forceinline__ T cta_reduce(T v, T* sh, Op op) {
#pragma unroll
    for (int d = 16; d >= 1; d >>= 1) v = op(v, __shfl_down_sync(FULL, v, d));
    if ((threadIdx.x & 31) == 0) sh[threadIdx.x >> 5] = v;
    __syncthreads();
    if (threadIdx.x == 0)
        for (int i = 1; i < TM_RED_T / 32; ++i) v = op(v, sh[i]);
    __syncthreads();
    return v;                             // valid in thread 0
}

__device__ __forceinline__ double entropy_of(float T) {
    const double q = fmin(fmax((double)T, 1e-6), 1.0 - 1e-6);
    return -(q * log(q) + (1.0 - q) * log(1.0 - q));
}

__global__ void __launch_bounds__(TM_RED_T, 1) tm_loss_kernel(const __grid_constant__ TmParams p) {
    __shared__ double shd[TM_RED_T / 32];
    __shared__ long long shl[TM_RED_T / 32];
    const long long chunk = (p.N + TM_RED_T - 1) / TM_RED_T;
    const long long lo = min(p.N, (long long)threadIdx.x * chunk), hi = min(p.N, lo + chunk);
    double mse = 0.0, ent = 0.0, dist = 0.0, per = 0.0;
    long long rmax = -1;
    const double third = (double)p.rp.inv_nsamples / 3.0;
    for (long long r = lo; r < hi; ++r) {
        const TmRay& o = p.tot[r];
        for (int c = 0; c < 3; ++c) {
            const double d = (double)o.rgbm[c] - (double)__ldg(p.tgt + 3 * r + c);
            mse += d * d;
        }
        ent += entropy_of(o.T);
        dist += 2.0 * o.pair + third * o.w2;
        per += (double)o.per;
        if (o.n_shaded > 0) rmax = r;
    }
    const auto add = [](double a, double b) { return a + b; };
    mse = cta_reduce(mse, shd, add);
    ent = cta_reduce(ent, shd, add);
    dist = cta_reduce(dist, shd, add);
    per = cta_reduce(per, shd, add);
    rmax = cta_reduce(rmax, shl, [](long long a, long long b) { return a > b ? a : b; });
    if (threadIdx.x == 0) {
        const double N = (double)p.N;
        const double t0 = p.w_main > 0.f ? (double)p.w_main * mse / (3.0 * N) : 0.0;
        const double t1 = p.w_ent > 0.f ? (double)p.w_ent * ent / N : 0.0;
        const double t2 = (p.w_dist > 0.f && rmax >= 0) ? (double)p.w_dist * dist / (double)(rmax + 1) : 0.0;
        const double t3 = (p.w_rp > 0.f && rmax >= 0) ? (double)p.w_rp * per / N : 0.0;
        p.terms[0] = (float)t0; p.terms[1] = (float)t1; p.terms[2] = (float)t2; p.terms[3] = (float)t3;
        *p.loss = (float)(t0 + t1 + t2 + t3);
        p.hdr->n_dist = rmax + 1;
    }
}

// ---------------------------------------------------------------------------------------------
// backward
// ---------------------------------------------------------------------------------------------
// dW[o][k] += sum over the warp's 32 staged rows of D[row][o] * H[row][k]; dB[o] += sum D[row][o]
__device__ __forceinline__ void warp_dw(const float* Hs, int ks, const float* Ds, int ds, int nout, int nin, float* gW, float* gB,
                                        int lane) {
    if (gW) {
        for (int e = lane; e < nout * nin; e += 32) {
            const int o = e / nin, k = e - o * nin;
            float acc = 0.f;
#pragma unroll 8
            for (int row = 0; row < 32; ++row) acc = __fmaf_rn(Ds[row * ds + o], Hs[row * ks + k], acc);
            if (acc != 0.f) atomicAdd(gW + e, acc);
        }
    }
    if (gB) {
        for (int o = lane; o < nout; o += 32) {
            float acc = 0.f;
            for (int row = 0; row < 32; ++row) acc = __fadd_rn(acc, Ds[row * ds + o]);
            if (acc != 0.f) atomicAdd(gB + o, acc);
        }
    }
}

__device__ __forceinline__ void scatter8(float* g, const float cw[8], const int cidx[8], float v) {
    if (v == 0.f) return;
#pragma unroll
    for (int k = 0; k < 8; ++k)
        if (cw[k] != 0.f) atomicAdd(g + cidx[k], __fmul_rn(cw[k], v));
}

template <int KIND, int ACT>
__global__ void __launch_bounds__(TM_T) tm_backward_kernel(const __grid_constant__ TmParams p) {
    extern __shared__ __align__(16) float tm_smem[];
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    float* Hs = tm_smem + (size_t)warp * 32 * (p.ks + p.ds);
    float* Ds = Hs + 32 * p.ks;
    const long long r = (long long)blockIdx.x * TM_T + threadIdx.x;
    const bool have = r < p.N;
    const float gL = __ldg(p.g_loss);
    const bool mlp = p.s.depth > 0;

    Ray ray = no_ray();
    float vemb[3 + 6 * 10];
    int n_vemb = 0;
    TmRay o;
    memset(&o, 0, sizeof(o));
    float g_rgbm[3] = {0.f, 0.f, 0.f}, tg[3] = {0.f, 0.f, 0.f}, g_last = 0.f;
    double B_tot = 0.0, cd = 0.0;                 // sum over the ray of dL/dw_k w_k; the distortion gradient's g / n
    const double c23 = 2.0 * (double)p.rp.inv_nsamples / 3.0;
    if (have) {
        ray = setup_ray<KIND>(p.s, p.rp, ld3(p.ro, r), ld3(p.rd, r));
        if (mlp) {
            const Vec3 v = ld3(p.vd, r);
            const float vv[3] = {v.x, v.y, v.z};
            n_vemb = embed3(vv, p.s.viewpe, vemb);
        }
        o = p.tot[r];
        const float c_m = (float)((double)gL * 2.0 * (double)p.w_main / (3.0 * (double)p.N));
        for (int c = 0; c < 3; ++c) {
            tg[c] = __ldg(p.tgt + 3 * r + c);
            const float bg = p.bkgd ? __ldg(p.bkgd + 3 * r + c) : p.rp.bg;
            g_rgbm[c] = __fmul_rn(c_m, __fsub_rn(o.rgbm[c], tg[c]));
            g_last = __fmaf_rn(g_rgbm[c], bg, g_last);
            B_tot = fma((double)g_rgbm[c], o.rgbf[c], B_tot);
        }
        if (p.w_ent > 0.f && o.T >= 1e-6f && o.T <= 1.f - 1e-6f) {
            const float ce = (float)((double)gL * (double)p.w_ent / (double)p.N);
            g_last = __fmaf_rn(ce, __fsub_rn(logf(__fsub_rn(1.f, o.T)), logf(o.T)), g_last);
        }
        if (p.w_dist > 0.f && o.n_shaded > 0) {
            cd = (double)gL * (double)p.w_dist / (double)p.hdr->n_dist;
            // sum_i D_i w_i = 4 pair + 2/3 I sum w^2: the distortion part of the suffix total
            B_tot = fma(cd, fma(4.0, o.pair, c23 * o.w2), B_tot);
        }
    }
    const float c_rp = (float)((double)gL * 2.0 * (double)p.w_rp / (double)p.N);
    const float back0 = __fmul_rn(g_last, o.T);

    MarchState<KIND> st(have);
    double Bp = 0.0, wp = 0.0, wsp = 0.0;        // running prefixes (through the current sample for Bp)
    const float mpi_den = (float)(p.rp.n_samples - 1);
    Shade sh;
    float dz[TM_MAX_W];
    for (int i = 0;; ++i) {
        const bool active = !st.done && i < ray.n_steps;
        if (!__any_sync(FULL, active)) break;
        bool shade = false, live = false;
        float w = 0.f, T_prev = st.T, alpha = 0.f, e = 0.f;
        Cell cell;
        float cw[8];
        int cidx[8];
        if (active) {
            const int d0 = st.cnt_d;
            shade = march_step<KIND, false>(p.s, p.rp, ray, mpi_den, st, i, w, cell, cw, cidx);
            if (st.cnt_d != d0) {            // occupied: alpha as march_step computed it
                alpha = sample_alpha<KIND>(p.s, p.rp, cell, cw, cidx, e);
                live = !(p.s.thres > 0.f) || alpha > p.s.thres;
            }
        }
        double gw = 0.0;                             // dL/dw of the sample (0 unless shaded)
        if (shade) {
            tm_shade<KIND, ACT, true>(p, cell, cw, cidx, vemb, n_vemb, sh);
            gw = fma((double)g_rgbm[2], (double)sh.c[2], fma((double)g_rgbm[1], (double)sh.c[1], (double)g_rgbm[0] * sh.c[0]));
            if (p.w_dist > 0.f) {
                const double s = sample_s(p.rp, i), wd = w;
                const double wa = o.w_sum - wp - wd;                 // W>i  = total - W<=i
                const double wsa = o.ws_sum - wsp - wd * s;          // WM>i
                const double D = 2.0 * (s * (wp - wa) + (wsa - wsp)) + c23 * wd;
                gw = fma(cd, D, gw);
                wp += wd;
                wsp = fma(wd, s, wsp);
            }
            // dL/d rgb -> dL/d logit
            float dlog[3];
            for (int c = 0; c < 3; ++c) {
                float dc = __fmul_rn(w, g_rgbm[c]);
                if (p.w_rp > 0.f) dc = __fmaf_rn(__fmul_rn(c_rp, w), __fsub_rn(sh.c[c], tg[c]), dc);
                dlog[c] = __fmul_rn(__fmul_rn(dc, __fsub_rn(1.f, sh.c[c])), sh.c[c]);
            }
            float dk0[TM_MAX_K0];
            const int C = p.s.C;
            for (int c = 0; c < C; ++c) dk0[c] = 0.f;
            if (!mlp) {
                for (int c = 0; c < 3; ++c) dk0[c] = dlog[c];
            } else {
                const int W = p.n_out[0];
                // layer 3 -> h2
                for (int k = 0; k < W; ++k) {
                    float a = 0.f;
                    for (int oc = 0; oc < 3; ++oc) a = __fmaf_rn(dlog[oc], __ldg(p.W[2] + (size_t)oc * W + k), a);
                    dz[k] = act_bwd<ACT>(a, sh.z2[k], sh.h2[k], p.s);
                }
                // layer 2 -> h1 (dz becomes dL/dz1; the staged deltas need dz2, so stage layer 2's rows first)
                for (int k = 0; k < W; ++k) { Ds[lane * p.ds + k] = dz[k]; Hs[lane * p.ks + k] = sh.h1[k]; }
                float dz1[TM_MAX_W];
                for (int k = 0; k < W; ++k) {
                    float a = 0.f;
                    for (int oc = 0; oc < W; ++oc) a = __fmaf_rn(dz[oc], __ldg(p.W[1] + (size_t)oc * W + k), a);
                    dz1[k] = act_bwd<ACT>(a, sh.z1[k], sh.h1[k], p.s);
                }
                for (int k = 0; k < W; ++k) dz[k] = dz1[k];
                // layer 1 -> input: dL/d k0 of the channels fed to the MLP
                const int nk = C - p.s.k0_view_off, nx = p.n_in[0];
                for (int k = 0; k < nk; ++k) {
                    float a = 0.f;
                    for (int oc = 0; oc < W; ++oc) a = __fmaf_rn(dz[oc], __ldg(p.W[0] + (size_t)oc * nx + k), a);
                    dk0[p.s.k0_view_off + k] = a;
                }
                if (KIND == K4_KIND_DVGO && !p.s.direct)
                    for (int c = 0; c < 3; ++c) dk0[c] = dlog[c];
                sh.logit[0] = dlog[0]; sh.logit[1] = dlog[1]; sh.logit[2] = dlog[2];   // kept for layer 3's rows
            }
            if (p.g_k0)
                for (int c = 0; c < C; ++c) scatter8(p.g_k0 + (long long)c * p.nvox, cw, cidx, dk0[c]);
        }
        if (live) {
            // Alphas2Weights.backward, B_i = g_last T_last + (total - prefix through i)
            Bp = fma(gw, (double)w, Bp);
            const float back = (float)((double)back0 + (B_tot - Bp));
            const double den = (double)__fsub_rn(1.f, alpha) + 1e-10;
            const float ga = (float)((double)__fmul_rn((float)gw, T_prev) - (double)back / den);
            // Raw2Alpha.backward
            const double m = fmin((double)e, 1e10);
            const float pw = powf(__fadd_rn(1.f, e), __fsub_rn(-p.rp.interval, 1.f));
            const float gx = (float)(((m * (double)pw) * (double)p.rp.interval) * (double)ga);
            if (p.g_den) scatter8(p.g_den, cw, cidx, gx);
        }
        // the warp's rgbnet weight gradients for this step: layers 2 (staged above), 1 and 3
        if (mlp && __any_sync(FULL, shade)) {
            const int W = p.n_out[0], nx = p.n_in[0];
            if (!shade)
                for (int k = 0; k < W; ++k) { Ds[lane * p.ds + k] = 0.f; Hs[lane * p.ks + k] = 0.f; }
            __syncwarp();
            warp_dw(Hs, p.ks, Ds, p.ds, W, W, p.gW[1], p.gB[1], lane);
            __syncwarp();
            for (int k = 0; k < W; ++k) Ds[lane * p.ds + k] = shade ? dz[k] : 0.f;
            for (int k = 0; k < nx; ++k) Hs[lane * p.ks + k] = shade ? sh.x[k] : 0.f;
            __syncwarp();
            warp_dw(Hs, p.ks, Ds, p.ds, W, nx, p.gW[0], p.gB[0], lane);
            __syncwarp();
            for (int k = 0; k < 3; ++k) Ds[lane * p.ds + k] = shade ? sh.logit[k] : 0.f;
            for (int k = 0; k < W; ++k) Hs[lane * p.ks + k] = shade ? sh.h2[k] : 0.f;
            __syncwarp();
            warp_dw(Hs, p.ks, Ds, p.ds, 3, W, p.gW[2], p.gB[2], lane);
            __syncwarp();
        }
    }
}

// ---------------------------------------------------------------------------------------------
// host side
// ---------------------------------------------------------------------------------------------
inline size_t tm_ws_bytes(long long n) { return sizeof(TmHeader) + (size_t)n * sizeof(TmRay); }

int tm_check(const k4_train_march_args* a) {
    if (!a || a->n_rays < 1) return K4_ERR_INVALID_ARG;
    if (a->kind != K4_KIND_DVGO && a->kind != K4_KIND_DMPIGO && a->kind != K4_KIND_DCVGO) return K4_ERR_INVALID_ARG;
    if (a->rgbnet_act < K4_ACT_RELU || a->rgbnet_act > K4_ACT_LKRELU) return K4_ERR_INVALID_ARG;
    for (int i = 0; i < 3; ++i)
        if (a->world_size[i] < 1 || a->mask_size[i] < 1) return K4_ERR_INVALID_ARG;
    if (a->k0_dim < 3 || a->rgbnet_depth < 0 || a->viewbase_pe < 0 || a->spatial_pe < 0) return K4_ERR_INVALID_ARG;
    if (a->rgbnet_depth == 0 && a->k0_dim != 3) return K4_ERR_INVALID_ARG;
    if (a->rgbnet_depth > 0 && a->rgbnet_width < 1) return K4_ERR_INVALID_ARG;
    if (!(a->stepsize > 0.f) || !(a->interval > 0.f)) return K4_ERR_INVALID_ARG;
    if (a->w_main < 0.f || a->w_entropy < 0.f || a->w_distortion < 0.f || a->w_rgbper < 0.f) return K4_ERR_INVALID_ARG;
    if (!a->d_rays_o || !a->d_rays_d || !a->d_viewdirs || !a->d_target || !a->d_density || !a->d_k0 || !a->d_mask)
        return K4_ERR_INVALID_ARG;
    if (a->kind == K4_KIND_DMPIGO && (!a->d_act_shift_grid || a->mpi_depth < 2)) return K4_ERR_INVALID_ARG;
    if (a->kind == K4_KIND_DVGO && a->w_distortion > 0.f) return K4_ERR_INVALID_ARG;     // no s / n_max (lib/dvgo.py)
    if (a->kind == K4_KIND_DMPIGO && a->rgbnet_depth > 0 && a->rgbnet_act == K4_ACT_GAUSS &&
        !(std::isfinite(a->rgbnet_act_param) && a->rgbnet_act_param > 0.f))
        return K4_ERR_INVALID_ARG;                                                      // GaussianActivation.a: finite, > 0
    if (a->kind == K4_KIND_DCVGO) return K4_ERR_UNSUPPORTED;
    if (a->kind == K4_KIND_DVGO && a->rgbnet_act != K4_ACT_RELU) return K4_ERR_UNSUPPORTED;
    if (a->rgbnet_depth != 0 && a->rgbnet_depth != 3) return K4_ERR_UNSUPPORTED;
    if (a->k0_dim > TM_MAX_K0 || a->rgbnet_width > TM_MAX_W || a->viewbase_pe > 10 || a->spatial_pe > 10) return K4_ERR_UNSUPPORTED;
    if ((long long)a->world_size[0] * a->world_size[1] * a->world_size[2] >= (1ll << 31)) return K4_ERR_UNSUPPORTED;
    if (a->rgbnet_depth == 3) {
        const int off = (a->kind == K4_KIND_DVGO && !a->rgbnet_direct) ? 3 : 0;
        const int dim0 = a->k0_dim - off + 3 + 6 * a->viewbase_pe + (a->kind == K4_KIND_DMPIGO ? 3 + 6 * a->spatial_pe : 0);
        if (dim0 > K4_MAX_DIM0) return K4_ERR_UNSUPPORTED;
        for (int l = 0; l < 3; ++l)
            if (!a->d_rgbnet_weight[l] || !a->d_rgbnet_bias[l]) return K4_ERR_INVALID_ARG;
    }
    return K4_OK;
}

int tm_ws_check(const void* ws, size_t bytes, long long n) {
    if (!ws || (uintptr_t)ws % 16) return K4_ERR_INVALID_ARG;
    if (bytes < tm_ws_bytes(n)) return K4_ERR_WORKSPACE;
    return K4_OK;
}

void tm_params(TmParams& p, const k4_train_march_args* a, const void* ws) {
    memset(&p, 0, sizeof(p));
    K4Dev& v = p.s;
    v.kind = a->kind;
    v.X = a->world_size[0]; v.Y = a->world_size[1]; v.Z = a->world_size[2];
    v.C = a->k0_dim;
    v.mX = a->mask_size[0]; v.mY = a->mask_size[1]; v.mZ = a->mask_size[2];
    for (int i = 0; i < 3; ++i) {
        v.xyz_min[i] = a->xyz_min[i]; v.xyz_max[i] = a->xyz_max[i];
        v.xyz_len[i] = a->xyz_max[i] - a->xyz_min[i];                // fp32, as torch: (xyz_max - xyz_min)
        v.m_scale[i] = a->xyz2ijk_scale[i]; v.m_shift[i] = a->xyz2ijk_shift[i];
    }
    v.act_shift = a->kind == K4_KIND_DVGO ? a->act_shift : 0.f;
    v.thres = a->fast_color_thres;
    v.mpi_depth = a->mpi_depth;
    v.depth = a->rgbnet_depth;
    v.width = a->rgbnet_width;
    v.direct = a->rgbnet_direct;
    v.viewpe = a->rgbnet_depth ? a->viewbase_pe : 0;
    v.spape = a->rgbnet_depth ? a->spatial_pe : 0;
    v.k0_view_off = (a->kind == K4_KIND_DVGO && a->rgbnet_depth && !a->rgbnet_direct) ? 3 : 0;
    const float aa = a->rgbnet_act_param * a->rgbnet_act_param;
    v.act_den = 2.f * aa;                                             // torch: 2*self.a**2, in fp32
    v.density = a->d_density;
    v.mask = a->d_mask;
    v.act_grid = a->d_act_shift_grid;
    K4RenderParams& rp = p.rp;
    rp.near_ = a->near_;
    rp.bg = a->bg;
    rp.interval = a->interval;
    if (a->kind == K4_KIND_DVGO) {
        rp.far_ = 1e9f;                                               // lib/dvgo.py:307
        rp.stepdist = a->stepsize * a->voxel_size;                    // lib/dvgo.py:310 (fp32 product)
        rp.n_samples = (int)((float)(a->max_world_size - 1) / a->stepsize) + 1;
    } else {
        rp.far_ = 1.f;
        rp.n_samples = (int)((double)(a->mpi_depth - 1) / (double)a->stepsize) + 1;   // lib/dmpigo.py:278
    }
    rp.inv_nsamples = (float)(1.0 / (double)rp.n_samples);            // ATen: a / cpu_scalar == a * (1/b)
    p.N = a->n_rays;
    p.nvox = (long long)v.X * v.Y * v.Z;
    p.ro = a->d_rays_o; p.rd = a->d_rays_d; p.vd = a->d_viewdirs; p.tgt = a->d_target; p.bkgd = a->d_bkgd;
    p.k0 = a->d_k0;
    if (a->rgbnet_depth == 3) {
        const int dim0 = a->k0_dim - v.k0_view_off + 3 + 6 * v.viewpe + (a->kind == K4_KIND_DMPIGO ? 3 + 6 * v.spape : 0);
        const int nin[3] = {dim0, a->rgbnet_width, a->rgbnet_width}, nout[3] = {a->rgbnet_width, a->rgbnet_width, 3};
        for (int l = 0; l < 3; ++l) {
            p.W[l] = a->d_rgbnet_weight[l]; p.B[l] = a->d_rgbnet_bias[l];
            p.n_in[l] = nin[l]; p.n_out[l] = nout[l];
            p.gW[l] = a->d_grad_weight[l]; p.gB[l] = a->d_grad_bias[l];
        }
        v.dim0 = dim0;
        p.ks = (dim0 > a->rgbnet_width ? dim0 : a->rgbnet_width) + 1;    // +1: a lane's row write hits its own bank
        p.ds = a->rgbnet_width + 1;
    }
    p.w_main = a->w_main; p.w_ent = a->w_entropy; p.w_dist = a->w_distortion; p.w_rp = a->w_rgbper;
    p.rgbm = a->d_rgb_marched; p.alphainv = a->d_alphainv_last; p.loss = a->d_loss; p.terms = a->d_loss_terms;
    p.g_den = a->d_grad_density; p.g_k0 = a->d_grad_k0;
    p.hdr = (TmHeader*)ws;
    p.tot = (TmRay*)(p.hdr + 1);
}

template <int KIND, int ACT>
int tm_launch(const TmParams& p, bool backward, cudaStream_t s) {
    const unsigned blocks = (unsigned)((p.N + TM_T - 1) / TM_T);
    if (!backward) {
        tm_forward_kernel<KIND, ACT><<<blocks, TM_T, 0, s>>>(p);
        K4_CUDA_TRY(cudaGetLastError());
        tm_loss_kernel<<<1, TM_RED_T, 0, s>>>(p);
    } else {
        const size_t smem = p.s.depth ? (size_t)TM_WARPS * 32 * (p.ks + p.ds) * sizeof(float) : 0;
        auto kern = tm_backward_kernel<KIND, ACT>;
        if (smem > 48 * 1024) K4_CUDA_TRY(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
        kern<<<blocks, TM_T, smem, s>>>(p);
    }
    K4_CUDA_TRY(cudaGetLastError());
    return K4_OK;
}

int tm_dispatch(const TmParams& p, int act, bool backward, cudaStream_t s) {
    if (p.s.kind == K4_KIND_DVGO) return tm_launch<K4_KIND_DVGO, K4_ACT_RELU>(p, backward, s);
    if (act == K4_ACT_GAUSS) return tm_launch<K4_KIND_DMPIGO, K4_ACT_GAUSS>(p, backward, s);
    if (act == K4_ACT_LKRELU) return tm_launch<K4_KIND_DMPIGO, K4_ACT_LKRELU>(p, backward, s);
    return tm_launch<K4_KIND_DMPIGO, K4_ACT_RELU>(p, backward, s);
}

}  // namespace

extern "C" {

size_t k4_train_march_workspace_bytes(int64_t n_rays) {
    return n_rays < 1 ? 0 : tm_ws_bytes(n_rays);
}

int k4_train_march_forward(const k4_train_march_args* a, void* d_workspace, size_t workspace_bytes, k4_stream_t stream) {
    int st = tm_check(a);
    if (st != K4_OK) return st;
    if (!a->d_rgb_marched || !a->d_alphainv_last || !a->d_loss || !a->d_loss_terms) return K4_ERR_INVALID_ARG;
    st = tm_ws_check(d_workspace, workspace_bytes, a->n_rays);
    if (st != K4_OK) return st;
    TmParams p;
    tm_params(p, a, d_workspace);
    return tm_dispatch(p, a->rgbnet_act, false, (cudaStream_t)stream);
}

int k4_train_march_backward(const k4_train_march_args* a, const float* d_grad_loss, const void* d_workspace, size_t workspace_bytes,
                            k4_stream_t stream) {
    int st = tm_check(a);
    if (st != K4_OK) return st;
    if (!d_grad_loss) return K4_ERR_INVALID_ARG;
    st = tm_ws_check(d_workspace, workspace_bytes, a->n_rays);
    if (st != K4_OK) return st;
    TmParams p;
    tm_params(p, a, d_workspace);
    p.g_loss = d_grad_loss;
    return tm_dispatch(p, a->rgbnet_act, true, (cudaStream_t)stream);
}

}  // extern "C"
