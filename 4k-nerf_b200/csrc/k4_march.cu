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
// The per-ray geometry, the marching step up to the shade decision and the ray's results are in
// k4_march_ray.cuh, the one copy this kernel shares with k4_march_ws.cu (its header gives the
// floating-point shape that keeps the geometry bit-identical to the reference).
#include "k4_internal.cuh"
#include "k4_march_common.cuh"
#include "k4_march_ray.cuh"
#include "k4_march_mma.cuh"

namespace {

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

        Ray r = no_ray();
        float vemb[3 + 6 * 10];
        int n_vemb = 0;
        if (have_ray) {
            r = setup_ray<KIND>(s, rp, ld3(rp.rays_o, ray_i), ld3(rp.rays_d, ray_i));
            if (s.depth > 0) {
                const Vec3 v = ld3(rp.viewdirs, ray_i);
                const float vv[3] = {v.x, v.y, v.z};
                n_vemb = embed3(vv, s.viewpe, vemb);
            }
        }
        if (MODE != K4_MLP_FP32) mma.begin_tile(s, vemb, n_vemb, lane);

        MarchState<KIND> st(have_ray);
        float acc_r = 0.f, acc_g = 0.f, acc_b = 0.f;
        const float mpi_den = (float)(rp.n_samples - 1);

        for (int i = 0; ; ++i) {
            const bool active = !st.done && (i < r.n_steps);
            if (!__any_sync(FULL, active)) break;
            bool shade = false;
            float w_sample = 0.f;
            Cell cell;
            float cw[8];
            int cidx[8];
            if (active) shade = march_step<KIND, true>(s, rp, r, mpi_den, st, i, w_sample, cell, cw, cidx);
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

        if (have_ray) finish_ray(rp, ray_i, r, st, acc_r, acc_g, acc_b);
        tot_m += st.cnt_m; tot_d += st.cnt_d; tot_c += st.cnt_c;
    }

    if (rp.counters) {
        flush_counters(rp, tot_m, tot_d, tot_c, lane);
        if (MODE != K4_MLP_FP32 && lane == 0) atomicAdd(rp.counters + 3, (unsigned long long)mma.n_batches);
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
