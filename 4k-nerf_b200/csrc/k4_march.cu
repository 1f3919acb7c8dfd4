// k4_march.cu -- the fused ray marcher of libk4nerf.so (sm_90a).
//
// ONE launch replaces the reference's per-chunk chain of ~60-80 kernels and ~14 host syncs
// (SURVEY.md section 3.2):
//   sample_pts_on_rays / sample_ndc_pts_on_rays   lib/cuda/render_utils_kernel.cu:12-79,167-194,245-270
//   maskcache_lookup                               lib/cuda/render_utils_kernel.cu:373-392
//   DenseGrid.forward (F.grid_sample trilinear)    lib/grid.py:117-128  (ATen grid_sampler_3d)
//   raw2alpha                                      lib/cuda/render_utils_kernel.cu:431-443
//   alpha2weight (+ T < 1e-3 early-out)            lib/cuda/render_utils_kernel.cu:577-605
//   the three threshold compactions                lib/dvgo.py:353-369
//   view/pos embedding, rgbnet, sigmoid            lib/dvgo.py:387-412, lib/dmpigo.py:338-379
//   segment_coo sums, background, depth            lib/dvgo.py:415-446
// Nothing is materialised per sample: one thread walks one ray (lanes of a warp = neighbouring
// pixels, so a warp's gathers hit a handful of voxels and stay in L1), samples that survive the
// thresholds are shaded immediately (fp32 mode) or queued per warp and shaded 32 at a time on the
// tensor cores (f16 modes, k4_march_mma.cuh).
//
// Floating-point shape: every `a*b+c` that nvcc contracts in the reference kernels is written as
// an explicit __fmaf_rn here, and everything else uses the _rn intrinsics, so that the geometric
// results (t_min/t_max, step counts, in-box and occupancy masks) are bit-identical to the
// reference's device code regardless of this file's own compiler flags.
#include "k4_internal.cuh"
#include "k4_march_common.cuh"
#include "k4_march_mma.cuh"

namespace {

// ---------------------------------------------------------------------------------------------
// per-ray geometry
// ---------------------------------------------------------------------------------------------
struct Ray {
    float sx, sy, sz;      // DVGO: start point; MPI: origin
    float dx, dy, dz;      // DVGO: unit direction; MPI: rays_d (un-normalised NDC direction)
    int n_steps;
    float t_min, t_max;
};

// infer_t_minmax / infer_n_samples / infer_ray_start_dir (render_utils_kernel.cu:12-79).
__device__ __forceinline__ Ray setup_ray_dvgo(const K4Dev& s, const K4RenderParams& rp, Vec3 o, Vec3 d) {
    Ray r;
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
    return r;
}

__device__ __forceinline__ long long tile_ray(const K4RenderParams& rp, long long tile, int lane) {
    if (rp.image_w > 0) {
        const int tiles_x = (rp.image_w + 7) >> 3;
        const int ty = (int)(tile / tiles_x), tx = (int)(tile - (long long)ty * tiles_x);
        const int px = tx * 8 + (lane & 7), py = ty * 4 + (lane >> 3);
        if (px >= rp.image_w || py >= rp.image_h) return -1;
        return (long long)py * rp.image_w + px;
    }
    const long long r = tile * 32 + lane;
    return (r < rp.n_rays) ? r : -1;
}

// ---------------------------------------------------------------------------------------------
// The fused kernel.  KIND: K4_KIND_DVGO / K4_KIND_DMPIGO.  MODE: K4_MLP_FP32 or a tensor-core mode.  ACT: the rgbnet's
// hidden activation (K4_ACT_*); only DirectMPIGO is instantiated with the non-relu ones.
// ---------------------------------------------------------------------------------------------
template <int KIND, int MODE, int ACT>
__global__ void __launch_bounds__(K4_MARCH_THREADS)
k4_march_kernel(const __grid_constant__ K4Dev s, const __grid_constant__ K4RenderParams rp) {
    extern __shared__ __align__(16) unsigned char smem_raw[];
    const int lane = threadIdx.x & 31;
    const int warp = threadIdx.x >> 5;

    MmaWarpCtx<MODE, ACT> mma;
    if (MODE != K4_MLP_FP32) mma.init(s, smem_raw, warp, lane);

    unsigned long long tot_m = 0, tot_d = 0, tot_c = 0;

    for (;;) {
        long long tile = 0;
        if (lane == 0) tile = (long long)atomicAdd(rp.tile_counter, 1u);
        tile = __shfl_sync(FULL, tile, 0);
        if (tile >= rp.n_tiles) break;

        const long long ray_i = tile_ray(rp, tile, lane);
        const bool have_ray = ray_i >= 0;

        Ray r;
        float vemb[3 + 6 * 10];
        int n_vemb = 0;
        r.n_steps = 0; r.t_min = 0.f; r.t_max = 0.f;
        r.sx = r.sy = r.sz = r.dx = r.dy = r.dz = 0.f;
        if (have_ray) {
            const Vec3 o = ld3(rp.rays_o, ray_i), d = ld3(rp.rays_d, ray_i);
            if (KIND == K4_KIND_DVGO) {
                r = setup_ray_dvgo(s, rp, o, d);
            } else if (KIND == K4_KIND_DCVGO) {
                // sample_ray, lib/dcvgo.py:237-238: o' = (o - center) / radius ; d' = d / ||d||  (torch ops)
                r.sx = __fdiv_rn(__fsub_rn(o.x, s.scene_center[0]), s.scene_radius[0]);
                r.sy = __fdiv_rn(__fsub_rn(o.y, s.scene_center[1]), s.scene_radius[1]);
                r.sz = __fdiv_rn(__fsub_rn(o.z, s.scene_center[2]), s.scene_radius[2]);
                const float dn = l2norm3_aten(d.x, d.y, d.z);
                r.dx = __fdiv_rn(d.x, dn); r.dy = __fdiv_rn(d.y, dn); r.dz = __fdiv_rn(d.z, dn);
                r.n_steps = rp.n_samples;
            } else {
                r.sx = o.x; r.sy = o.y; r.sz = o.z; r.dx = d.x; r.dy = d.y; r.dz = d.z;
                r.n_steps = rp.n_samples;
            }
            if (s.depth > 0) {
                const Vec3 v = ld3(rp.viewdirs, ray_i);
                const float vv[3] = {v.x, v.y, v.z};
                n_vemb = embed3(vv, s.viewpe, vemb);
            }
        }
        if (MODE != K4_MLP_FP32) mma.begin_tile(s, vemb, n_vemb, lane);

        float T = 1.f;
        float acc_r = 0.f, acc_g = 0.f, acc_b = 0.f, acc_depth = 0.f;
        int cnt_m = 0, cnt_d = 0, cnt_c = 0;
        bool done = !have_ray;
        const float mpi_den = (float)(rp.n_samples - 1);
        float cum_dist = 0.f, qx = 0.f, qy = 0.f, qz = 0.f;      // DCVGO: cumdist_thres state, previous contracted point

        for (int i = 0; ; ++i) {
            const bool active = !done && (i < r.n_steps);
            if (!__any_sync(FULL, active)) break;
            bool shade = false;
            float w_sample = 0.f;
            Cell cell;
            float cw[8];
            int cidx[8];
            if (active) {
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
                if (KIND == K4_KIND_DCVGO) {
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
                        cum_dist = __fadd_rn(cum_dist, l2norm3_aten(__fsub_rn(px, qx), __fsub_rn(py, qy), __fsub_rn(pz, qz)));
                        over = cum_dist > rp.dist_thres;
                        if (over) cum_dist = 0.f;
                    }
                    qx = px; qy = py; qz = pz;
                    outb = !(inner | over);
                } else {
                    outb = (s.xyz_min[0] > px) | (s.xyz_min[1] > py) | (s.xyz_min[2] > pz) |
                           (s.xyz_max[0] < px) | (s.xyz_max[1] < py) | (s.xyz_max[2] < pz);
                }
                if (!outb) {
                    ++cnt_m;
                    // MaskGrid.forward -> maskcache_lookup (render_utils_kernel.cu:385-390)
                    const int mi = (int)roundf(__fmaf_rn(px, s.m_scale[0], s.m_shift[0]));
                    const int mj = (int)roundf(__fmaf_rn(py, s.m_scale[1], s.m_shift[1]));
                    const int mk = (int)roundf(__fmaf_rn(pz, s.m_scale[2], s.m_shift[2]));
                    bool occ = false;
                    const bool in_mask = (0 <= mi) & (mi < s.mX) & (0 <= mj) & (mj < s.mY) & (0 <= mk) & (mk < s.mZ);
                    if (in_mask) occ = __ldg(s.mask + ((size_t)mi * s.mY + mj) * s.mZ + mk) != 0;
                    if (KIND != K4_KIND_DCVGO && !occ && in_mask && s.skip) {
                        // empty-space skipping (k4_march_common.cuh): the next n samples are in-box and unoccupied
                        const float h = (KIND == K4_KIND_DVGO) ? rp.stepdist : __fdiv_rn(1.f, mpi_den);
                        const int n = skip_steps(s, mi, mj, mk, r.sx, r.sy, r.sz, r.dx * h, r.dy * h, r.dz * h, i, r.n_steps);
                        cnt_m += n;
                        i += n;
                    }
                    if (occ) {
                        ++cnt_d;
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
                            const float w = __fmul_rn(T, alpha);
                            T = (float)((double)T * (1.0 - (double)alpha));
                            if ((double)T < 1e-3) done = true;
                            if (!(s.thres > 0.f) || w > s.thres) {
                                shade = true;
                                w_sample = w;
                                ++cnt_c;
                                if (rp.render_depth) {
                                    // DVGO/MPI: s = (step + 0.5) / N_samples; DCVGO: s = 1 - 1/(1+t)  (lib/dcvgo.py:353)
                                    const float sd = (KIND == K4_KIND_DCVGO)
                                        ? __fsub_rn(1.f, __fdiv_rn(1.f, __fadd_rn(1.f, t_i)))
                                        : __fmul_rn(__fadd_rn((float)i, 0.5f), rp.inv_nsamples);
                                    acc_depth = __fadd_rn(acc_depth, __fmul_rn(w, sd));
                                }
                            }
                        }
                    }
                }
            }
            if (MODE == K4_MLP_FP32) {
                if (shade) {
                    float k0v[32];
                    interp_k0<8>(s, cw, cidx, k0v);
                    float rgb[3];
                    if (s.depth == 0) {
                        rgb[0] = sigmoid_ref(k0v[0]); rgb[1] = sigmoid_ref(k0v[1]); rgb[2] = sigmoid_ref(k0v[2]);
                    } else {
                        float x[K4_MAX_DIM0];
                        int n = 0;
                        for (int c = s.k0_view_off; c < s.C; ++c) x[n++] = k0v[c];
                        if (KIND == K4_KIND_DMPIGO) {
                            const float pe[3] = {cell.cz, cell.cy, cell.cx};   // .flip(-1), lib/dmpigo.py:338
                            n += embed3(pe, s.spape, x + n);
                        }
                        for (int c = 0; c < n_vemb; ++c) x[n++] = vemb[c];
                        mlp_fp32<ACT>(s, x, rgb);
                        if (KIND == K4_KIND_DVGO && !s.direct) {
                            rgb[0] = __fadd_rn(rgb[0], k0v[0]); rgb[1] = __fadd_rn(rgb[1], k0v[1]);
                            rgb[2] = __fadd_rn(rgb[2], k0v[2]);
                        }
                        rgb[0] = sigmoid_ref(rgb[0]); rgb[1] = sigmoid_ref(rgb[1]); rgb[2] = sigmoid_ref(rgb[2]);
                    }
                    acc_r = __fadd_rn(acc_r, __fmul_rn(w_sample, rgb[0]));
                    acc_g = __fadd_rn(acc_g, __fmul_rn(w_sample, rgb[1]));
                    acc_b = __fadd_rn(acc_b, __fmul_rn(w_sample, rgb[2]));
                }
            } else {
                mma.template push<KIND>(s, shade, w_sample, cell, cw, cidx, vemb, n_vemb, lane);
            }
        }
        if (MODE != K4_MLP_FP32) mma.end_tile(s, lane, acc_r, acc_g, acc_b);

        if (have_ray) {
            // rgb_marched = rgb_feature + alphainv_last * bg   (lib/dvgo.py:425-427)
            const float bgt = __fmul_rn(T, rp.bg);
            k4_store_ray(rp, ray_i, __fadd_rn(acc_r, bgt), __fadd_rn(acc_g, bgt), __fadd_rn(acc_b, bgt), T, acc_depth);
            if (rp.ray_stats) {
                int4 st = make_int4(r.n_steps, cnt_m, cnt_d, cnt_c);
                reinterpret_cast<int4*>(rp.ray_stats)[ray_i] = st;
            }
            if (rp.t_minmax) { rp.t_minmax[2 * ray_i] = r.t_min; rp.t_minmax[2 * ray_i + 1] = r.t_max; }
        }
        tot_m += cnt_m; tot_d += cnt_d; tot_c += cnt_c;
    }

    if (rp.counters) {
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
            if (MODE != K4_MLP_FP32) atomicAdd(rp.counters + 3, (unsigned long long)mma.n_batches);
        }
    }
}

template <int KIND, int MODE, int ACT = K4_ACT_RELU>
int launch_variant(const k4_scene* sc, const K4RenderParams& rp, cudaStream_t st) {
    auto kern = k4_march_kernel<KIND, MODE, ACT>;
    size_t smem = MmaWarpCtx<MODE>::smem_bytes(sc->dev);
    if (smem > 48 * 1024) K4_CUDA_TRY(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    int dev = 0, sms = 0, per_sm = 0;
    K4_CUDA_TRY(cudaGetDevice(&dev));
    K4_CUDA_TRY(cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev));
    K4_CUDA_TRY(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, kern, K4_MARCH_THREADS, smem));
    if (per_sm < 1) per_sm = 1;
    const long long warps_per_block = K4_MARCH_THREADS / 32;
    long long blocks = (rp.n_tiles + warps_per_block - 1) / warps_per_block;
    const long long cap = (long long)sms * per_sm;     // persistent: a multiple of the SM count
    if (blocks > cap) blocks = cap;
    if (blocks < 1) blocks = 1;
    kern<<<(unsigned)blocks, K4_MARCH_THREADS, smem, st>>>(sc->dev, rp);
    K4_CUDA_TRY(cudaGetLastError());
    return K4_OK;
}

// DirectMPIGO with a gauss / lkrelu rgbnet (act_type, lib/dmpigo.py:89-95)
template <int ACT>
int launch_mpi_act(const k4_scene* sc, const K4RenderParams& rp, int mlp_mode, cudaStream_t st) {
    if (mlp_mode == K4_MLP_FP32 || sc->dev.depth == 0) return launch_variant<K4_KIND_DMPIGO, K4_MLP_FP32, ACT>(sc, rp, st);
    if (mlp_mode == K4_MLP_F16 && MmaWarpCtx<K4_MLP_F16>::supported(sc->dev)) return launch_variant<K4_KIND_DMPIGO, K4_MLP_F16, ACT>(sc, rp, st);
    if (mlp_mode == K4_MLP_F16X3 && MmaWarpCtx<K4_MLP_F16X3>::supported(sc->dev))
        return launch_variant<K4_KIND_DMPIGO, K4_MLP_F16X3, ACT>(sc, rp, st);
    return K4_ERR_UNSUPPORTED;
}

}  // namespace

int k4_launch_march(const k4_scene* sc, const K4RenderParams& rp, int mlp_mode, cudaStream_t st) {
    if (sc->act != K4_ACT_RELU) {           // k4_scene_create admits them for DirectMPIGO only
        if (sc->dev.kind != K4_KIND_DMPIGO) return K4_ERR_UNSUPPORTED;
        return sc->act == K4_ACT_GAUSS ? launch_mpi_act<K4_ACT_GAUSS>(sc, rp, mlp_mode, st)
                                       : launch_mpi_act<K4_ACT_LKRELU>(sc, rp, mlp_mode, st);
    }
    if (sc->dev.kind == K4_KIND_DCVGO) {
        if (mlp_mode == K4_MLP_FP32 || sc->dev.depth == 0) return launch_variant<K4_KIND_DCVGO, K4_MLP_FP32>(sc, rp, st);
        if (mlp_mode == K4_MLP_F16 && MmaWarpCtx<K4_MLP_F16>::supported(sc->dev)) return launch_variant<K4_KIND_DCVGO, K4_MLP_F16>(sc, rp, st);
        if (mlp_mode == K4_MLP_F16X3 && MmaWarpCtx<K4_MLP_F16X3>::supported(sc->dev))
            return launch_variant<K4_KIND_DCVGO, K4_MLP_F16X3>(sc, rp, st);
        return K4_ERR_UNSUPPORTED;
    }
    const bool mpi = sc->dev.kind == K4_KIND_DMPIGO;
    if (mlp_mode == K4_MLP_FP32 || sc->dev.depth == 0) {
        return mpi ? launch_variant<K4_KIND_DMPIGO, K4_MLP_FP32>(sc, rp, st)
                   : launch_variant<K4_KIND_DVGO, K4_MLP_FP32>(sc, rp, st);
    }
    if (mlp_mode == K4_MLP_F16 && MmaWarpCtx<K4_MLP_F16>::supported(sc->dev)) {
        return mpi ? launch_variant<K4_KIND_DMPIGO, K4_MLP_F16>(sc, rp, st)
                   : launch_variant<K4_KIND_DVGO, K4_MLP_F16>(sc, rp, st);
    }
    if (mlp_mode == K4_MLP_F16X3 && MmaWarpCtx<K4_MLP_F16X3>::supported(sc->dev)) {
        return mpi ? launch_variant<K4_KIND_DMPIGO, K4_MLP_F16X3>(sc, rp, st)
                   : launch_variant<K4_KIND_DVGO, K4_MLP_F16X3>(sc, rp, st);
    }
    return K4_ERR_UNSUPPORTED;
}
