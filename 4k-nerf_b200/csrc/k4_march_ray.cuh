// k4_march_ray.cuh -- what one thread does for one ray in both fused marchers (k4_march.cu, k4_march_ws.cu),
// independent of how the surviving samples are shaded: the per-ray geometry, one marching step up to
// the shade / skip decision, and the per-ray and per-warp results.  The one copy of
//   sample_pts_on_rays / sample_ndc_pts_on_rays   lib/cuda/render_utils_kernel.cu:12-79,167-194,245-270
//   maskcache_lookup                               lib/cuda/render_utils_kernel.cu:373-392
//   raw2alpha                                      lib/cuda/render_utils_kernel.cu:431-443
//   alpha2weight (+ T < 1e-3 early-out)            lib/cuda/render_utils_kernel.cu:577-605
//   the three threshold compactions                lib/dvgo.py:353-369
//   background, depth                              lib/dvgo.py:415-446
//
// Floating-point shape: every `a*b+c` that nvcc contracts in the reference kernels is written as
// an explicit __fmaf_rn here, and everything else uses the _rn intrinsics, so that the geometric
// results (t_min/t_max, step counts, in-box and occupancy masks) are bit-identical to the
// reference's device code regardless of the including file's own compiler flags.
//
// Everything is __forceinline__ and takes the model kind as a template parameter: each kernel compiles the expressions
// below into its own loop, as if they were written there.
#pragma once
#include "k4_internal.cuh"
#include "k4_march_common.cuh"

namespace {

// ---------------------------------------------------------------------------------------------
// per-ray geometry
// ---------------------------------------------------------------------------------------------
struct Ray {
    float sx, sy, sz;      // DVGO: start point; MPI: origin; DCVGO: origin in the unit-sphere frame
    float dx, dy, dz;      // DVGO / DCVGO: unit direction; MPI: rays_d (un-normalised NDC direction)
    int n_steps;
    float t_min, t_max;    // DVGO only (0 otherwise)
};

template <int KIND>
__device__ __forceinline__ Ray setup_ray(const K4Dev& s, const K4RenderParams& rp, Vec3 o, Vec3 d) {
    Ray r;
    if (KIND == K4_KIND_DVGO) {
        // infer_t_minmax / infer_n_samples / infer_ray_start_dir (render_utils_kernel.cu:12-79).
        const float vx = (d.x == 0.f) ? 1e-6f : d.x;
        const float vy = (d.y == 0.f) ? 1e-6f : d.y;
        const float vz = (d.z == 0.f) ? 1e-6f : d.z;
        const float ax = __fdiv_rn(__fsub_rn(s.xyz_max[0], o.x), vx);
        const float ay = __fdiv_rn(__fsub_rn(s.xyz_max[1], o.y), vy);
        const float az = __fdiv_rn(__fsub_rn(s.xyz_max[2], o.z), vz);
        const float bx = __fdiv_rn(__fsub_rn(s.xyz_min[0], o.x), vx);
        const float by = __fdiv_rn(__fsub_rn(s.xyz_min[1], o.y), vy);
        const float bz = __fdiv_rn(__fsub_rn(s.xyz_min[2], o.z), vz);
        r.t_min = fmaxf(fminf(fmaxf(fmaxf(fminf(ax, bx), fminf(ay, by)), fminf(az, bz)), rp.far_), rp.near_);
        r.t_max = fmaxf(fminf(fminf(fminf(fmaxf(ax, bx), fmaxf(ay, by)), fmaxf(az, bz)), rp.far_), rp.near_);
        float nn = __fmul_rn(d.y, d.y);              // reference SASS: FMUL y,y ; FFMA x,x,. ; FFMA z,z,.
        nn = __fmaf_rn(d.x, d.x, nn);
        nn = __fmaf_rn(d.z, d.z, nn);
        const float rnorm = __fsqrt_rn(nn);
        const float ns = ceilf(__fdiv_rn(__fmul_rn(__fsub_rn(r.t_max, r.t_min), rnorm), rp.stepdist));
        r.n_steps = (ns > 1.f) ? ((ns >= 2147483520.f) ? 2147483647 : (int)ns) : 1;   // max(ceil(.), 1.)
        r.sx = __fmaf_rn(d.x, r.t_min, o.x);
        r.sy = __fmaf_rn(d.y, r.t_min, o.y);
        r.sz = __fmaf_rn(d.z, r.t_min, o.z);
        r.dx = __fdiv_rn(d.x, rnorm);
        r.dy = __fdiv_rn(d.y, rnorm);
        r.dz = __fdiv_rn(d.z, rnorm);
    } else if (KIND == K4_KIND_DCVGO) {
        // sample_ray, lib/dcvgo.py:237-238: o' = (o - center) / radius ; d' = d / ||d||  (torch ops)
        r.sx = __fdiv_rn(__fsub_rn(o.x, s.scene_center[0]), s.scene_radius[0]);
        r.sy = __fdiv_rn(__fsub_rn(o.y, s.scene_center[1]), s.scene_radius[1]);
        r.sz = __fdiv_rn(__fsub_rn(o.z, s.scene_center[2]), s.scene_radius[2]);
        const float dn = l2norm3_aten(d.x, d.y, d.z);
        r.dx = __fdiv_rn(d.x, dn); r.dy = __fdiv_rn(d.y, dn); r.dz = __fdiv_rn(d.z, dn);
        r.n_steps = rp.n_samples;
        r.t_min = r.t_max = 0.f;
    } else {
        r.sx = o.x; r.sy = o.y; r.sz = o.z; r.dx = d.x; r.dy = d.y; r.dz = d.z;
        r.n_steps = rp.n_samples;
        r.t_min = r.t_max = 0.f;
    }
    return r;
}

// the ray of a thread that has none (a pixel beyond the image edge): no steps
__device__ __forceinline__ Ray no_ray() {
    Ray r;
    r.n_steps = 0; r.t_min = r.t_max = 0.f;
    r.sx = r.sy = r.sz = r.dx = r.dy = r.dz = 0.f;
    return r;
}

// ---------------------------------------------------------------------------------------------
// per-ray marching state
// ---------------------------------------------------------------------------------------------
template <int KIND> struct Contraction {};
template <> struct Contraction<K4_KIND_DCVGO> {
    float cum_dist = 0.f;                   // cumdist_thres: distance accumulated since the last point kept by distance
    float qx = 0.f, qy = 0.f, qz = 0.f;     // previous contracted point
};

template <int KIND>
struct MarchState : Contraction<KIND> {
    float T = 1.f, acc_depth = 0.f;
    int cnt_m = 0, cnt_d = 0, cnt_c = 0;    // this ray's in-box samples, density queries, shaded samples (S_m, S_d, S_c)
    bool done;
    __device__ __forceinline__ explicit MarchState(bool have_ray) : done(!have_ray) {}
};

// ---------------------------------------------------------------------------------------------
// One marching step: the sample at step i of an active ray (!st.done && i < r.n_steps).  Returns whether the sample is
// to be shaded, with weight w_sample and the k0 gather prepared in cell / cw / cidx.  i is advanced by the steps skipped
// through empty space, not past the sample itself.  mpi_den = n_samples - 1 as a float (MPI's step denominator).
// SKIP: compile the empty-space skip in (it still needs a model with a skip field, s.skip).
// ---------------------------------------------------------------------------------------------
template <int KIND, bool SKIP>
__device__ __forceinline__ bool march_step(const K4Dev& s, const K4RenderParams& rp, const Ray& r, float mpi_den,
                                           MarchState<KIND>& st, int& i, float& w_sample, Cell& cell, float cw[8], int cidx[8]) {
    float px, py, pz;
    if (KIND == K4_KIND_DVGO) {
        const float dist = __fmul_rn(rp.stepdist, (float)i);
        px = __fmaf_rn(r.dx, dist, r.sx);
        py = __fmaf_rn(r.dy, dist, r.sy);
        pz = __fmaf_rn(r.dz, dist, r.sz);
    } else if (KIND == K4_KIND_DMPIGO) {
        const float dist = __fdiv_rn((float)i, mpi_den);
        px = __fmaf_rn(r.dx, dist, r.sx);
        py = __fmaf_rn(r.dy, dist, r.sy);
        pz = __fmaf_rn(r.dz, dist, r.sz);
    }
    bool outb;
    float t_i = 0.f;
    if constexpr (KIND == K4_KIND_DCVGO) {
        // lib/dcvgo.py:249-262: p = o' + d'*t (separate torch ops), inf-norm contraction of the outside
        t_i = __ldg(rp.t_list + i);
        px = __fadd_rn(r.sx, __fmul_rn(r.dx, t_i));
        py = __fadd_rn(r.sy, __fmul_rn(r.dy, t_i));
        pz = __fadd_rn(r.sz, __fmul_rn(r.dz, t_i));
        const float nrm = fmaxf(fabsf(px), fmaxf(fabsf(py), fabsf(pz)));
        const bool inner = nrm <= 1.f;
        if (!inner) {
            // ray_pts / norm * ((1+bg_len) - bg_len/norm); scalar/tensor is reciprocal()*scalar
            const float f = __fsub_rn(s.one_plus_bg, __fmul_rn(__fdiv_rn(1.f, nrm), s.bg_len));
            px = __fmul_rn(__fdiv_rn(px, nrm), f);
            py = __fmul_rn(__fdiv_rn(py, nrm), f);
            pz = __fmul_rn(__fdiv_rn(pz, nrm), f);
        }
        // lib/dcvgo.py:282-285 + ub360_utils_kernel.cu:12-32: keep inner points, and outer points
        // whenever the distance accumulated since the last kept-by-distance point exceeds thres
        bool over = false;
        if (i > 0) {
            st.cum_dist = __fadd_rn(st.cum_dist, l2norm3_aten(__fsub_rn(px, st.qx), __fsub_rn(py, st.qy), __fsub_rn(pz, st.qz)));
            over = st.cum_dist > rp.dist_thres;
            if (over) st.cum_dist = 0.f;
        }
        st.qx = px; st.qy = py; st.qz = pz;
        outb = !(inner | over);
    } else {
        outb = (s.xyz_min[0] > px) | (s.xyz_min[1] > py) | (s.xyz_min[2] > pz) |
               (s.xyz_max[0] < px) | (s.xyz_max[1] < py) | (s.xyz_max[2] < pz);
    }
    bool shade = false;
    if (!outb) {
        ++st.cnt_m;
        // MaskGrid.forward -> maskcache_lookup (render_utils_kernel.cu:385-390)
        const int mi = (int)roundf(__fmaf_rn(px, s.m_scale[0], s.m_shift[0]));
        const int mj = (int)roundf(__fmaf_rn(py, s.m_scale[1], s.m_shift[1]));
        const int mk = (int)roundf(__fmaf_rn(pz, s.m_scale[2], s.m_shift[2]));
        bool occ = false;
        const bool in_mask = (0 <= mi) & (mi < s.mX) & (0 <= mj) & (mj < s.mY) & (0 <= mk) & (mk < s.mZ);
        if (in_mask) occ = __ldg(s.mask + ((size_t)mi * s.mY + mj) * s.mZ + mk) != 0;
        if (SKIP && KIND != K4_KIND_DCVGO && !occ && in_mask && s.skip) {
            // empty-space skipping (k4_march_common.cuh): the next n samples are in-box and unoccupied
            const float h = (KIND == K4_KIND_DVGO) ? rp.stepdist : __fdiv_rn(1.f, mpi_den);
            const int n = skip_steps(s, mi, mj, mk, r.sx, r.sy, r.sz, r.dx * h, r.dy * h, r.dz * h, i, r.n_steps);
            st.cnt_m += n;
            i += n;
        }
        if (occ) {
            ++st.cnt_d;
            cell = make_cell(s, px, py, pz);
            corner_setup(s, cell, cw, cidx);
            float den = interp_density(s, cw, cidx);
            float shift = s.act_shift;
            if (KIND == K4_KIND_DMPIGO) {
                // act_shift grid [1,1,1,1,D]: 1-D lerp along world z (lib/dmpigo.py:316)
                const int z0 = cell.z0, z1 = cell.z0 + 1;
                float a = 0.f;
                if (z0 >= 0 && z0 < s.mpi_depth) a = __fmul_rn(__ldg(s.act_grid + z0), cell.wz0);
                if (z1 >= 0 && z1 < s.mpi_depth) a = __fmaf_rn(__ldg(s.act_grid + z1), cell.wz1, a);
                den = __fadd_rn(den, a);
                shift = 0.f;
            }
            // Raw2Alpha (render_utils_kernel.cu:439-441)
            const float e = expf(__fadd_rn(den, shift));
            const float alpha = __fsub_rn(1.f, powf(__fadd_rn(1.f, e), -rp.interval));
            if (!(s.thres > 0.f) || alpha > s.thres) {
                // Alphas2Weights (render_utils_kernel.cu:593-600)
                const float w = __fmul_rn(st.T, alpha);
                st.T = (float)((double)st.T * (1.0 - (double)alpha));
                if ((double)st.T < 1e-3) st.done = true;
                if (!(s.thres > 0.f) || w > s.thres) {
                    shade = true;
                    w_sample = w;
                    ++st.cnt_c;
                    if (rp.render_depth) {
                        // DVGO/MPI: s = (step + 0.5) / N_samples; DCVGO: s = 1 - 1/(1+t)  (lib/dcvgo.py:353)
                        const float sd = (KIND == K4_KIND_DCVGO)
                            ? __fsub_rn(1.f, __fdiv_rn(1.f, __fadd_rn(1.f, t_i)))
                            : __fmul_rn(__fadd_rn((float)i, 0.5f), rp.inv_nsamples);
                        st.acc_depth = __fadd_rn(st.acc_depth, __fmul_rn(w, sd));
                    }
                }
            }
        }
    }
    return shade;
}

// ---------------------------------------------------------------------------------------------
// results
// ---------------------------------------------------------------------------------------------
// One finished ray; (cr, cg, cb) is its accumulated colour without the background.
template <int KIND>
__device__ __forceinline__ void finish_ray(const K4RenderParams& rp, long long ray_i, const Ray& r, const MarchState<KIND>& st,
                                           float cr, float cg, float cb) {
    // rgb_marched = rgb_feature + alphainv_last * bg   (lib/dvgo.py:425-427)
    const float bgt = __fmul_rn(st.T, rp.bg);
    k4_store_ray(rp, ray_i, __fadd_rn(cr, bgt), __fadd_rn(cg, bgt), __fadd_rn(cb, bgt), st.T, st.acc_depth);
    if (rp.ray_stats) reinterpret_cast<int4*>(rp.ray_stats)[ray_i] = make_int4(r.n_steps, st.cnt_m, st.cnt_d, st.cnt_c);
    if (rp.t_minmax) { rp.t_minmax[2 * ray_i] = r.t_min; rp.t_minmax[2 * ray_i + 1] = r.t_max; }
}

// A warp's S_m / S_d / S_c totals into rp.counters[0..2] (which the caller has checked to be there).  counters[3], the
// number of MLP batches, stays with each kernel: who counts them differs.
__device__ __forceinline__ void flush_counters(const K4RenderParams& rp, unsigned long long tot_m, unsigned long long tot_d,
                                               unsigned long long tot_c, int lane) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
        tot_m += __shfl_xor_sync(FULL, tot_m, o);
        tot_d += __shfl_xor_sync(FULL, tot_d, o);
        tot_c += __shfl_xor_sync(FULL, tot_c, o);
    }
    if (lane == 0) {
        atomicAdd(rp.counters + 0, tot_m);
        atomicAdd(rp.counters + 1, tot_d);
        atomicAdd(rp.counters + 2, tot_c);
    }
}

}  // namespace
