// k4_march_tc.cu -- the fused marcher with the rgbnet on the Hopper tensor cores: gather on the CUDA cores,
// MLP as warpgroup MMAs with register-resident activations.  Same reference chain as k4_march.cu
// (lib/dvgo.py:327-448 / lib/dmpigo.py:292-427 in one launch), different execution shape:
//
//  * one persistent CTA per SM, 256 threads = two WARPGROUPS of 128; a warpgroup owns 128 rays (a
//    16x8 pixel block: lanes of a warp are an 8x4 pixel tile, so a warp's gathers fall into a few
//    voxels and hit L1), one thread marches one ray;
//  * samples that survive the alpha / weight thresholds are appended as fp16 feature rows to the
//    warpgroup's 256-row ring in shared memory, already in the canonical K-major wgmma layout
//    (8 rows x 16 B core matrices: a quarter-warp's 16-byte stores are one contiguous 128 B line);
//  * whenever 128 rows are pending the warpgroup runs the whole MLP for them on the tensor cores
//    (mlp_batch_wgmma, k4_march_mlp.cuh); the two warpgroups are independent pipelines that share
//    only the tensor core, so one gathers while the other's MMAs run;
//  * weights + bias tiles (62 KB) are staged once per CTA with a single TMA bulk copy.
//
// Geometry and thresholds are the one copy every marcher compiles (k4_march_ray.cuh), the config, the sample features and
// the PTX helpers the ones of k4_march_ws.cu (k4_march_ring.cuh); only the MLP runs in fp16 operands / fp32 accumulate, like
// K4_MLP_F16.  This marcher does not skip empty space and has no DCVGO config.
#include "k4_internal.cuh"
#include "k4_march_common.cuh"
#include "k4_march_ray.cuh"
#include "k4_march_mlp.cuh"
#include "k4_march_ring.cuh"

namespace {

constexpr int TC_THREADS = 256;

// ACT: the rgbnet's hidden activation (K4_ACT_*); CfgB, the DirectMPIGO shape, is also built with gauss and lkrelu.
template <class Cfg, int ACT>
__global__ void __launch_bounds__(TC_THREADS, 1)
k4_march_tc_kernel(const __grid_constant__ K4Dev s, const __grid_constant__ K4RenderParams rp) {
    extern __shared__ __align__(1024) unsigned char smem[];
    constexpr int W = Cfg::W, KPAD = Cfg::KPAD, KCH = Cfg::KCH, TC_RING = Cfg::RING;
    const int tid = threadIdx.x, wg = tid >> 7, wt = tid & 127, lane = tid & 31, warp_in_wg = wt >> 5;

    unsigned char* blob = smem;
    unsigned char* wgb = smem + Cfg::BLOB_PAD + wg * Cfg::WG_BYTES;      // the ring's tiles come first
    float* qw = reinterpret_cast<float*>(wgb + Cfg::WG_QW);
    float* racc = reinterpret_cast<float*>(wgb + Cfg::WG_RACC);
    unsigned char* qowner = wgb + Cfg::WG_OWNER;
    volatile unsigned int* tailp = reinterpret_cast<volatile unsigned int*>(wgb + Cfg::WG_MISC);
    volatile long long* tile_slot = reinterpret_cast<volatile long long*>(wgb + Cfg::WG_MISC + 8);   // [2]
    uint64_t* wbar = reinterpret_cast<uint64_t*>(smem + Cfg::CTA_MISC);

    const TcBlobLayout BL = tc_blob_layout(KPAD, W);

    // ---------------- one-time CTA setup ----------------
    if (tid == 0) {
        mbar_init(wbar, 1);
        mbar_init_fence();
    }
    {   // zero this warpgroup's block (A rings incl. their K padding, accumulators, counters)
        uint32_t* z = reinterpret_cast<uint32_t*>(wgb);
        for (int i = wt; i < (Cfg::WG_MISC + 32) / 4; i += TC_WG) z[i] = 0u;
    }
    __syncthreads();
    bias_ones_ring<Cfg>(wgb, TC_RING, wt);
    if (tid == 0) stage_blob(blob, s.tc_blob, BL.total, wbar);
    mbar_wait(wbar, 0);
    const uint32_t a_ring_s = smem_u32(wgb);

    unsigned head = 0;
    unsigned long long tot_m = 0, tot_d = 0, tot_c = 0, n_batches = 0;
    const float mpi_den = (float)(rp.n_samples - 1);

    // One MLP batch over ring rows [head, head+128); `valid` of them are real samples.
    auto flush = [&](int valid) {
        const uint32_t a_tile = a_ring_s + ((head >> 7) & 1u) * Cfg::TILE_BYTES;
        fence_proxy_async();
        named_bar(wg + 1);
        if (wt == 0) ++n_batches;
        mlp_batch_wgmma<W, KPAD, true, ACT, Cfg::BIASC>(a_tile, blob, BL, valid, head & (TC_RING - 1), qw, qowner, nullptr, racc, wt, s.act_c,
                                            [] {}, true);
    };

    for (unsigned iter = 0;; ++iter) {
        // ---------------- next 128-ray tile of this warpgroup ----------------
        if (wt == 0) tile_slot[iter & 1] = (long long)atomicAdd(rp.tile_counter, 1u);
        named_bar(wg + 1);
        const long long tile = tile_slot[iter & 1];
        if (tile >= rp.n_tiles) break;

        long long ray_i;
        if (rp.image_w > 0) {
            const int tiles_x = (rp.image_w + 15) >> 4;
            const int ty = (int)(tile / tiles_x), tx = (int)(tile - (long long)ty * tiles_x);
            const int px = tx * 16 + (warp_in_wg & 1) * 8 + (lane & 7);
            const int py = ty * 8 + (warp_in_wg >> 1) * 4 + (lane >> 3);
            ray_i = (px < rp.image_w && py < rp.image_h) ? (long long)py * rp.image_w + px : -1;
        } else {
            ray_i = tile * TC_WG + wt;
            if (ray_i >= rp.n_rays) ray_i = -1;
        }
        const bool have_ray = ray_i >= 0;

        Ray r = no_ray();
        uint32_t vw[Cfg::NVW];
#pragma unroll
        for (int j = 0; j < Cfg::NVW; ++j) vw[j] = 0u;
        if (have_ray) {
            r = setup_ray<Cfg::KIND>(s, rp, ld3(rp.rays_o, ray_i), ld3(rp.rays_d, ray_i));
            pack_view_embedding<Cfg>(ld3(rp.viewdirs, ray_i), vw);
        }

        MarchState<Cfg::KIND> st(have_ray);
        int i = 0;

        for (;;) {
            // ---------------- a round of marching ----------------
#pragma unroll 1
            for (int rr = 0; rr < TC_ROUND; ++rr) {
                // a batch is pending -> go flush it.  Read once per warp and broadcast: the decision must
                // be warp-uniform (lanes may still be diverged from the previous step's branches, and the
                // other warps keep appending, so per-lane reads could disagree and split the warp).
                unsigned pend = 0;
                if (lane == 0) pend = *tailp - head;
                pend = __shfl_sync(FULL, pend, 0);
                if (pend >= 128u) break;
                const bool active = !st.done && (i < r.n_steps);
                if (!__any_sync(FULL, active)) break;
                bool shade = false;
                float w_sample = 0.f;
                Cell cell;
                float cw[8];
                int cidx[8];
                // no empty-space skipping in this marcher (SKIP = false)
                if (active) shade = march_step<Cfg::KIND, false>(s, rp, r, mpi_den, st, i, w_sample, cell, cw, cidx);
                ++i;
                // ---------------- append surviving samples to the warpgroup's ring ----------------
                const unsigned bal = __ballot_sync(FULL, shade);
                if (bal != 0u) {
                    unsigned base = 0;
                    if (lane == 0) base = atomicAdd(const_cast<unsigned int*>(tailp), (unsigned)__popc(bal));
                    base = __shfl_sync(FULL, base, 0);
                    if (shade) {
                        const unsigned slot = (base + __popc(bal & ((1u << lane) - 1u))) & (TC_RING - 1);
                        float f[Cfg::NF];
                        sample_features<Cfg>(s, cell, cw, cidx, f);
                        uint32_t row[KPAD / 2];
#pragma unroll
                        for (int j = 0; j < KPAD / 2; ++j) {
                            if (j < Cfg::NS / 2) row[j] = h2_sat(f[2 * j], f[2 * j + 1]);
                            else if (j < Cfg::NS / 2 + Cfg::NVW) row[j] = vw[j - Cfg::NS / 2];
                            else row[j] = row_pad_word<Cfg>(j);
                        }
                        unsigned char* rowp = wgb + (slot >> 7) * Cfg::TILE_BYTES + tc_canon_off((int)(slot & 127), 0, KCH);
#pragma unroll
                        for (int kc = 0; kc < KCH; ++kc)
                            if (kc * 4 < Cfg::NS / 2 + Cfg::NVW)        // chunks that are all padding stay zero
                                *reinterpret_cast<uint4*>(rowp + kc * 128) = make_uint4(row[4 * kc], row[4 * kc + 1], row[4 * kc + 2], row[4 * kc + 3]);
                        qw[slot] = w_sample;
                        qowner[slot] = (unsigned char)wt;
                    }
                }
            }
            // ---------------- warpgroup rendezvous ----------------
            const bool live = named_bar_or(wg + 1, !st.done && (i < r.n_steps));
            const unsigned tail = *tailp;                          // stable: nobody appends before the next barrier
            if (tail - head >= 128u) {
                flush(128);
                head += 128u;
            } else if (!live) {
                if (tail != head) {
                    flush((int)(tail - head));
                    head += 128u;
                    named_bar(wg + 1);                                     // everyone has read `tail` and the ring
                    if (wt == 0) *tailp = head;
                }
                break;
            } else {
                named_bar(wg + 1);
            }
        }
        named_bar(wg + 1);                                                 // all atomics into racc have landed
        if (have_ray) finish_ray(rp, ray_i, r, st, racc[wt * 3 + 0], racc[wt * 3 + 1], racc[wt * 3 + 2]);
        racc[wt * 3 + 0] = 0.f; racc[wt * 3 + 1] = 0.f; racc[wt * 3 + 2] = 0.f;
        tot_m += st.cnt_m; tot_d += st.cnt_d; tot_c += st.cnt_c;
    }

    if (rp.counters) {
        flush_counters(rp, tot_m, tot_d, tot_c, lane);
        if (wt == 0) atomicAdd(rp.counters + 3, n_batches);
    }
}

template <class Cfg, int ACT = K4_ACT_RELU>
int launch_tc(const k4_scene* sc, K4RenderParams rp, cudaStream_t st) {
    auto kern = k4_march_tc_kernel<Cfg, ACT>;
    K4_CUDA_TRY(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, Cfg::SMEM));
    int dev = 0, sms = 0;
    K4_CUDA_TRY(cudaGetDevice(&dev));
    K4_CUDA_TRY(cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev));
    const long long blocks = wg_launch_geometry(rp, sms);
    kern<<<(unsigned)blocks, TC_THREADS, Cfg::SMEM, st>>>(sc->dev, rp);
    K4_CUDA_TRY(cudaGetLastError());
    return K4_OK;
}

using CfgA = TcCfg<-1, K4_KIND_DVGO, 12, 4, 0, 128, 1, 2, false>;    // configs/default.py:107-119 fine stage
using CfgB = TcCfg<-1, K4_KIND_DMPIGO, 9, 0, 0, 64, 1, 2, false>;    // configs/llff/llff_default_lg.py + fern_lg_joint_l1.py

template <class Cfg>
bool matches(const K4Dev& v) {
    return v.kind == Cfg::KIND && v.C == Cfg::C && v.viewpe == Cfg::VIEWPE && v.width == Cfg::W && v.depth == 3 &&
           v.dim0 == Cfg::DIM0 && (Cfg::KIND == K4_KIND_DMPIGO ? v.spape == Cfg::SPAPE : v.direct != 0) &&
           v.tc_blob != nullptr && v.tc_kpad == Cfg::KPAD && v.tc_exact != 0 && v.Cpad == Cfg::CPAD;
}

}  // namespace

bool k4_tc_supported(const K4Dev& v) { return matches<CfgA>(v) || matches<CfgB>(v); }

int k4_launch_march_tc(const k4_scene* sc, K4RenderParams rp, cudaStream_t st) {
    if (sc->act != K4_ACT_RELU) {           // DirectMPIGO only (k4_scene_create)
        if (!matches<CfgB>(sc->dev)) return K4_ERR_UNSUPPORTED;
        return sc->act == K4_ACT_GAUSS ? launch_tc<CfgB, K4_ACT_GAUSS>(sc, rp, st) : launch_tc<CfgB, K4_ACT_LKRELU>(sc, rp, st);
    }
    if (matches<CfgA>(sc->dev)) return launch_tc<CfgA>(sc, rp, st);
    if (matches<CfgB>(sc->dev)) return launch_tc<CfgB>(sc, rp, st);
    return K4_ERR_UNSUPPORTED;
}
