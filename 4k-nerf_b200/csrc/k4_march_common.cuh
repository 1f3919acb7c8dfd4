// k4_march_common.cuh -- device helpers shared by the fused marcher and its tensor-core MLP context:
// grid coordinates and trilinear gathers that follow DenseGrid.forward / ATen grid_sampler_3d
// (lib/grid.py:117-128), the embeddings (lib/dvgo.py:387-388) and torch.sigmoid.
#pragma once
#include "k4_internal.cuh"
#include "k4_ptx.cuh"

namespace {

#define FULL 0xffffffffu

struct Vec3 { float x, y, z; };

__device__ __forceinline__ Vec3 ld3(const float* p, long long i) {
    Vec3 v;
    v.x = __ldg(p + 3 * i + 0);
    v.y = __ldg(p + 3 * i + 1);
    v.z = __ldg(p + 3 * i + 2);
    return v;
}

// ---------------------------------------------------------------------------------------------
// Grid coordinates of a world point, following DenseGrid.forward (lib/grid.py:123):
//   ind_norm = ((xyz - xyz_min) / (xyz_max - xyz_min)).flip(-1) * 2 - 1
// and ATen's grid_sampler_unnormalize(align_corners=True): ((c + 1) / 2) * (size - 1).
// Every torch op is a separate rounding, so no FMA here.
// ---------------------------------------------------------------------------------------------
struct Cell {
    float cx, cy, cz;      // ind_norm components of world x / y / z (before the flip)
    int x0, y0, z0;
    float wx1, wy1, wz1;   // fractional parts
    float wx0, wy0, wz0;
};

__device__ __forceinline__ float norm_coord(float p, float mn, float len) {
    float n = __fdiv_rn(__fsub_rn(p, mn), len);
    return __fsub_rn(__fmul_rn(n, 2.f), 1.f);
}

__device__ __forceinline__ float unnorm(float c, int size) {
    return __fmul_rn(__fmul_rn(__fadd_rn(c, 1.f), 0.5f), (float)(size - 1));
}

__device__ __forceinline__ void cell_axis(float g, int size, int& i0, float& w0, float& w1) {
    float f = floorf(g);
    i0 = (int)f;
    w1 = __fsub_rn(g, f);                         // ix - ix_tnw
    w0 = __fsub_rn(__fadd_rn(f, 1.f), g);         // ix_bse - ix  (== (float)(i0+1) - ix)
    (void)size;
}

__device__ __forceinline__ Cell make_cell(const K4Dev& s, float px, float py, float pz) {
    Cell c;
    c.cx = norm_coord(px, s.xyz_min[0], s.xyz_len[0]);
    c.cy = norm_coord(py, s.xyz_min[1], s.xyz_len[1]);
    c.cz = norm_coord(pz, s.xyz_min[2], s.xyz_len[2]);
    cell_axis(unnorm(c.cx, s.X), s.X, c.x0, c.wx0, c.wx1);
    cell_axis(unnorm(c.cy, s.Y), s.Y, c.y0, c.wy0, c.wy1);
    cell_axis(unnorm(c.cz, s.Z), s.Z, c.z0, c.wz0, c.wz1);
    return c;
}

// The 8 corner weights in ATen's order tnw,tne,tsw,tse,bnw,bne,bsw,bse where ATen's x is the
// W axis = world z, y = world y, z (top/bottom) = world x; each weight is ((a*b)*c) with
// a = z-factor, b = y-factor, c = x-factor (aten/src/ATen/native/cuda/GridSampler.cu).
__device__ __forceinline__ void corner_weights(const Cell& c, float w[8]) {
    float zy00 = __fmul_rn(c.wz0, c.wy0), zy10 = __fmul_rn(c.wz1, c.wy0);
    float zy01 = __fmul_rn(c.wz0, c.wy1), zy11 = __fmul_rn(c.wz1, c.wy1);
    w[0] = __fmul_rn(zy00, c.wx0); w[1] = __fmul_rn(zy10, c.wx0);
    w[2] = __fmul_rn(zy01, c.wx0); w[3] = __fmul_rn(zy11, c.wx0);
    w[4] = __fmul_rn(zy00, c.wx1); w[5] = __fmul_rn(zy10, c.wx1);
    w[6] = __fmul_rn(zy01, c.wx1); w[7] = __fmul_rn(zy11, c.wx1);
}

// Corner k of ATen's order: dz = k&1 (world z), dy = (k>>1)&1, dx = (k>>2)&1.
// Out-of-range corners are skipped by ATen (zero padding); in-box points only ever have the +1
// corner out of range, with weight exactly 0, so clamping the index and zeroing the weight is
// identical for finite grids.
__device__ __forceinline__ void corner_setup(const K4Dev& s, const Cell& c, float w[8], int idx[8]) {
    corner_weights(c, w);
    int x1 = c.x0 + 1, y1 = c.y0 + 1, z1 = c.z0 + 1;
    bool vx0 = (c.x0 >= 0) & (c.x0 < s.X), vx1 = (x1 >= 0) & (x1 < s.X);
    bool vy0 = (c.y0 >= 0) & (c.y0 < s.Y), vy1 = (y1 >= 0) & (y1 < s.Y);
    bool vz0 = (c.z0 >= 0) & (c.z0 < s.Z), vz1 = (z1 >= 0) & (z1 < s.Z);
    int cx0 = min(max(c.x0, 0), s.X - 1), cx1 = min(max(x1, 0), s.X - 1);
    int cy0 = min(max(c.y0, 0), s.Y - 1), cy1 = min(max(y1, 0), s.Y - 1);
    int cz0 = min(max(c.z0, 0), s.Z - 1), cz1 = min(max(z1, 0), s.Z - 1);
#pragma unroll
    for (int k = 0; k < 8; ++k) {
        bool v = ((k & 1) ? vz1 : vz0) & ((k & 2) ? vy1 : vy0) & ((k & 4) ? vx1 : vx0);
        int xx = (k & 4) ? cx1 : cx0, yy = (k & 2) ? cy1 : cy0, zz = (k & 1) ? cz1 : cz0;
        idx[k] = (xx * s.Y + yy) * s.Z + zz;
        if (!v) w[k] = 0.f;
    }
}

__device__ __forceinline__ float interp_density(const K4Dev& s, const float w[8], const int idx[8]) {
    float v[8];
#pragma unroll
    for (int k = 0; k < 8; ++k) v[k] = __ldg(s.density + idx[k]);
    float acc = __fmul_rn(v[0], w[0]);             // out_acc = 0 + v*w (the FMA with 0 is the product)
#pragma unroll
    for (int k = 1; k < 8; ++k) acc = __fmaf_rn(v[k], w[k], acc);
    return acc;
}

// k0 features, channel-last copy [X,Y,Z,Cpad]; 4 channels per pass keeps 8 float4 loads in flight.
template <int NQ>
__device__ __forceinline__ void interp_k0(const K4Dev& s, const float w[8], const int idx[8], float* out) {
    const float4* base = reinterpret_cast<const float4*>(s.k0cl);
    const int q = s.Cpad >> 2;
#pragma unroll
    for (int j = 0; j < NQ; ++j) {
        if (j < q) {
            float4 v[8];
#pragma unroll
            for (int k = 0; k < 8; ++k) v[k] = __ldg(base + (size_t)idx[k] * q + j);
            float4 a;
            a.x = __fmul_rn(v[0].x, w[0]); a.y = __fmul_rn(v[0].y, w[0]);
            a.z = __fmul_rn(v[0].z, w[0]); a.w = __fmul_rn(v[0].w, w[0]);
#pragma unroll
            for (int k = 1; k < 8; ++k) {
                a.x = __fmaf_rn(v[k].x, w[k], a.x); a.y = __fmaf_rn(v[k].y, w[k], a.y);
                a.z = __fmaf_rn(v[k].z, w[k], a.z); a.w = __fmaf_rn(v[k].w, w[k], a.w);
            }
            out[4 * j + 0] = a.x; out[4 * j + 1] = a.y; out[4 * j + 2] = a.z; out[4 * j + 3] = a.w;
        }
    }
}

// The same gather for a copy of exactly NQ channel quads per voxel (s.Cpad == 4 * NQ, the wgmma marcher's configs):
// no run-time channel count and no branch per quad, the corner rows addressed once with the quads at immediate offsets,
// loads issued KR corners (all their quads) at a time.  ptxas still interleaves the loads of later corners with the
// FMAs of earlier ones; what this saves is the per-quad branches and address arithmetic.  With 4 quads the unbranched
// loads raise the register pressure at the marchers' 128-register cap (config 4 would spill 76 bytes, not 28), so
// those configs keep the per-quad rounds of interp_k0.  Per channel the same products and FMA order as interp_k0.
template <int NQ, int KR = 2>
__device__ __forceinline__ void interp_k0_cfg(const K4Dev& s, const float w[8], const int idx[8], float* out) {
    static_assert(8 % KR == 0, "corners per round");
    if (NQ > 3) {
        interp_k0<NQ>(s, w, idx, out);
        return;
    }
    const float4* base = reinterpret_cast<const float4*>(s.k0cl);
    float4 a[NQ];
#pragma unroll
    for (int k0 = 0; k0 < 8; k0 += KR) {
        float4 v[KR][NQ];
#pragma unroll
        for (int k = 0; k < KR; ++k) {
            const float4* p = base + (size_t)idx[k0 + k] * NQ;
#pragma unroll
            for (int j = 0; j < NQ; ++j) v[k][j] = __ldg(p + j);
        }
#pragma unroll
        for (int j = 0; j < NQ; ++j)
#pragma unroll
            for (int k = 0; k < KR; ++k) {
                const float wk = w[k0 + k];
                if (k0 + k == 0) {                      // out_acc = 0 + v*w: the FMA with 0 is the product
                    a[j].x = __fmul_rn(v[k][j].x, wk); a[j].y = __fmul_rn(v[k][j].y, wk);
                    a[j].z = __fmul_rn(v[k][j].z, wk); a[j].w = __fmul_rn(v[k][j].w, wk);
                } else {
                    a[j].x = __fmaf_rn(v[k][j].x, wk, a[j].x); a[j].y = __fmaf_rn(v[k][j].y, wk, a[j].y);
                    a[j].z = __fmaf_rn(v[k][j].z, wk, a[j].z); a[j].w = __fmaf_rn(v[k][j].w, wk, a[j].w);
                }
            }
    }
#pragma unroll
    for (int j = 0; j < NQ; ++j) {
        out[4 * j + 0] = a[j].x; out[4 * j + 1] = a[j].y; out[4 * j + 2] = a[j].z; out[4 * j + 3] = a[j].w;
    }
}

// ---------------------------------------------------------------------------------------------
// Empty-space skipping (result preserving).  Called for a sample at step i that is inside the bounding box, maps to
// occupancy voxel (mi, mj, mk) and found it EMPTY.  s.skip holds, per cell of K4_SKIP_B^3 occupancy voxels, the
// Chebyshev distance d (in cells) to the nearest cell that contains an occupied voxel; d >= 1 means every voxel of the
// (2d-1)^3 cells around this one is empty.  Sample j of the ray sits at A + D*j (A = ray start, D = direction * step
// length).  The function returns n such that samples i+1 .. i+n
//   * lie inside that empty voxel region, whose faces are at half-integer voxel coordinates because the reference looks
//     up the NEAREST voxel (round(p*scale+shift), render_utils_kernel.cu:385-390), and
//   * lie inside the scene's bounding box (so each of them counts as an in-box sample, exactly as if it had been visited),
// both with a safety margin of 1e-3 voxel / 1e-3 step, three orders of magnitude above the rounding error of the sample
// position.  Such samples fail the occupancy test in the reference pipeline and contribute nothing; the caller adds n
// to its in-box counter and jumps.  n = 0 is always a correct answer.
// ---------------------------------------------------------------------------------------------
// one axis: false = the current sample is not safely inside the region on this axis (no skip at all)
__device__ __forceinline__ bool skip_axis(int c, int d, int msz, float shift, float iscale, float bmin, float bmax,
                                          float A, float D, float fi, float& s_exit) {
    // voxel index range of the empty region on this axis, clipped to the mask; world-space faces at -+0.5 voxel
    const int lo_v = max((c - d + 1) * K4_SKIP_B, 0), hi_v = min((c + d) * K4_SKIP_B - 1, msz - 1);
    const float eps = 1e-3f * iscale;
    const float lo = fmaxf(((float)lo_v - 0.5f - shift) * iscale, bmin) + eps;
    const float hi = fminf(((float)hi_v + 0.5f - shift) * iscale, bmax) - eps;
    const float cur = fmaf(D, fi, A);
    if (!(cur >= lo && cur <= hi)) return false;
    if (D > 0.f) s_exit = fminf(s_exit, __fdividef(hi - A, D));
    else if (D < 0.f) s_exit = fminf(s_exit, __fdividef(lo - A, D));
    return true;
}

__device__ __forceinline__ int skip_steps(const K4Dev& s, int mi, int mj, int mk, float ax, float ay, float az,
                                          float dx, float dy, float dz, int i, int n_steps) {
    const int ci = mi / K4_SKIP_B, cj = mj / K4_SKIP_B, ck = mk / K4_SKIP_B;
    const int d = __ldg(s.skip + ((size_t)ci * s.cY + cj) * s.cZ + ck);
    if (d == 0) return 0;
    const float fi = (float)i;
    float s_exit = 3.0e38f;
    if (!skip_axis(ci, d, s.mX, s.m_shift[0], s.m_iscale[0], s.xyz_min[0], s.xyz_max[0], ax, dx, fi, s_exit)) return 0;
    if (!skip_axis(cj, d, s.mY, s.m_shift[1], s.m_iscale[1], s.xyz_min[1], s.xyz_max[1], ay, dy, fi, s_exit)) return 0;
    if (!skip_axis(ck, d, s.mZ, s.m_shift[2], s.m_iscale[2], s.xyz_min[2], s.xyz_max[2], az, dz, fi, s_exit)) return 0;
    // samples with parameter j <= s_exit - 1e-3 are inside; never past the ray's last sample
    float jm = floorf(s_exit - 1e-3f);
    jm = fminf(jm, (float)(n_steps - 1));
    const int n = (int)(jm - fi);
    return n > 0 ? n : 0;
}

// torch.norm(dim=-1) of a 3-vector on CUDA: the reduction accumulates acc = fma(x, x, acc) in element
// order from 0, then sqrt (ATen norm_two ops compiled with fmad).
__device__ __forceinline__ float l2norm3_aten(float x, float y, float z) {
    float s = __fmul_rn(x, x);
    s = __fmaf_rn(y, y, s);
    s = __fmaf_rn(z, z, s);
    return __fsqrt_rn(s);
}

// torch.sigmoid on CUDA: 1 / (1 + exp(-x)) in fp32.
__device__ __forceinline__ float sigmoid_ref(float x) {
    return __fdiv_rn(1.f, __fadd_rn(1.f, expf(-x)));
}

// [v, sin(v*f_0..F-1) comp-major, cos(...)]  (lib/dvgo.py:387-388, lib/dmpigo.py:347-351)
__device__ __forceinline__ int embed3(const float v[3], int nfreq, float* out) {
    out[0] = v[0]; out[1] = v[1]; out[2] = v[2];
    int n = 3;
    for (int c = 0; c < 3; ++c)
        for (int f = 0; f < nfreq; ++f) out[n++] = sinf(__fmul_rn(v[c], (float)(1 << f)));
    for (int c = 0; c < 3; ++c)
        for (int f = 0; f < nfreq; ++f) out[n++] = cosf(__fmul_rn(v[c], (float)(1 << f)));
    return n;
}

// The rgbnet's hidden activation (K4_ACT_*, include/k4nerf.h), the one definition every MLP path uses.
//   fp32(x)  the fp32 mode: torch's own expression order, so that mode stays the exact cross-check
//            gauss:  -x**2 / (2*a**2) -> t = x*x; t = -t; expf(t / den) with den = 2*(a*a) rounded in fp32 on the host
//            lkrelu: ATen leaky_relu, x > 0 ? x : x * negval
//   tc(x)    the tensor-core modes, on the fp32 accumulator before the one rounding to fp16:
//            gauss:  ex2.approx(x*x*c), c = -log2(e) / (2 a^2) (k4_scene_create); +-inf and huge x give exactly 0
// relu is fmaxf(x, 0) in both (the wgmma repack fuses it into cvt.rn.relu, see mlp_act_h2 in k4_march_mlp.cuh).
template <int ACT>
struct RgbAct {
    static_assert(ACT == K4_ACT_RELU || ACT == K4_ACT_GAUSS || ACT == K4_ACT_LKRELU, "K4_ACT_*");
    __device__ __forceinline__ static float fp32(float x, const K4Dev& s) {
        if constexpr (ACT == K4_ACT_GAUSS) {
            const float t = -__fmul_rn(x, x);
            return expf(__fdiv_rn(t, s.act_den));
        } else if constexpr (ACT == K4_ACT_LKRELU) {
            return x > 0.f ? x : __fmul_rn(x, 0.01f);
        } else {
            return fmaxf(x, 0.f);
        }
    }
    __device__ __forceinline__ static float tc(float x, float c) {
        if constexpr (ACT == K4_ACT_GAUSS) {
            return ex2_approx_ftz(__fmul_rn(__fmul_rn(x, x), c));
        } else if constexpr (ACT == K4_ACT_LKRELU) {
            return x > 0.f ? x : __fmul_rn(x, 0.01f);
        } else {
            return fmaxf(x, 0.f);
        }
    }
};

// fp32 rgbnet: Linear-act-...-Linear, sequential FMA from the bias (exact mode).
template <int ACT>
__device__ __noinline__ void mlp_fp32(const K4Dev& s, const float* x, float rgb[3]) {
    float bufA[K4_MAX_WIDTH], bufB[K4_MAX_WIDTH];
    const float* in = x;
    float* out = bufA;
    for (int l = 0; l < s.depth; ++l) {
        const int nin = s.n_in[l], nout = s.n_out[l], ld = s.ldw[l];
        const float* __restrict__ W = s.wT[l];
        const float* __restrict__ B = s.bias[l];
        const bool last = (l == s.depth - 1);
        for (int j = 0; j < nout; j += 4) {
            float4 acc = __ldg(reinterpret_cast<const float4*>(B + j));
            for (int k = 0; k < nin; ++k) {
                const float xk = in[k];
                const float4 w4 = __ldg(reinterpret_cast<const float4*>(W + (size_t)k * ld + j));
                acc.x = __fmaf_rn(xk, w4.x, acc.x); acc.y = __fmaf_rn(xk, w4.y, acc.y);
                acc.z = __fmaf_rn(xk, w4.z, acc.z); acc.w = __fmaf_rn(xk, w4.w, acc.w);
            }
            if (last) {
                rgb[0] = acc.x; rgb[1] = acc.y; rgb[2] = acc.z;
            } else {
                out[j + 0] = RgbAct<ACT>::fp32(acc.x, s); out[j + 1] = RgbAct<ACT>::fp32(acc.y, s);
                out[j + 2] = RgbAct<ACT>::fp32(acc.z, s); out[j + 3] = RgbAct<ACT>::fp32(acc.w, s);
            }
        }
        in = out;
        out = (out == bufA) ? bufB : bufA;
    }
}

// One ray's results: into the caller's [N,3] / [N] arrays, or -- for a block-cyclic multi-GPU frame -- straight into the
// image-order frame of every rank (peer-mapped stores over NVLink; 20 bytes per ray and destination, issued while the
// other warps of the CTA march on, so the exchange costs no step of its own).
__device__ __forceinline__ void k4_store_ray(const K4RenderParams& rp, long long ray_i, float cr, float cg, float cb,
                                             float T, float depth) {
    if (rp.n_dst == 0) {
        rp.rgb[3 * ray_i + 0] = cr; rp.rgb[3 * ray_i + 1] = cg; rp.rgb[3 * ray_i + 2] = cb;
        rp.alphainv[ray_i] = T;
        if (rp.depth) rp.depth[ray_i] = depth;
        return;
    }
    const long long row = ray_i / rp.f_w;
    const long long col = ray_i - row * rp.f_w;
    const long long g = (((row >> 3) * rp.f_world + rp.f_rank) * 8 + (row & 7)) * rp.f_w + col;
#pragma unroll 1
    for (int p = 0; p < rp.n_dst; ++p) {
        float* f = rp.d_frame[p];
        f[3 * g + 0] = cr; f[3 * g + 1] = cg; f[3 * g + 2] = cb;
        if (rp.render_depth) f[3 * rp.f_nfull + g] = depth;
        f[4 * rp.f_nfull + g] = T;
    }
}

}  // namespace
