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
// Geometry and thresholds are evaluated exactly as in k4_march.cu (bit-identical masks); only the
// MLP runs in fp16 operands / fp32 accumulate, like K4_MLP_F16.
#include "k4_internal.cuh"
#include "k4_march_common.cuh"
#include "k4_march_mlp.cuh"

namespace {

constexpr int TC_THREADS = 256;
constexpr int TC_WG = 128;
constexpr int TC_RING = 256;
constexpr int TC_ROUND = 8;          // marching steps between warpgroup rendezvous when nothing is pending

template <int KIND_, int C_, int VIEWPE_, int SPAPE_, int W_>
struct TcCfg {
    static constexpr int KIND = KIND_, C = C_, VIEWPE = VIEWPE_, SPAPE = SPAPE_, W = W_;
    static constexpr int CPAD = (C + 3) & ~3;
    static constexpr int NVEMB = 3 + 6 * VIEWPE;
    static constexpr int NPOS = (KIND == K4_KIND_DMPIGO) ? 3 + 6 * SPAPE : 0;
    static constexpr int NS = C + NPOS;                 // per-sample features (must be even)
    static constexpr int DIM0 = NS + NVEMB;
    static constexpr int KPAD = (DIM0 + 15) & ~15;
    static constexpr int KCH = KPAD / 8;                // 16-byte chunks per A row
    static constexpr int NVW = (NVEMB + 1) / 2;         // packed per-ray words
    static constexpr int TILE_BYTES = 128 * KPAD * 2;
    static_assert(NS % 2 == 0, "per-sample feature count must be even for the packed row layout");
    static_assert(W == 128 || W == 64, "hidden width");
    // shared memory map
    static constexpr int BLOB = W * KPAD * 2 + W * W * 2 + 16 * W * 2 + 2 * W * 16 * 2 + 16 * 16 * 2 + 128 * 16 * 2;
    static constexpr int BLOB_PAD = (BLOB + 1023) & ~1023;
    static constexpr int WG_A = 2 * TILE_BYTES;
    static constexpr int WG_QW = WG_A;                       // float[256]
    static constexpr int WG_RACC = WG_QW + TC_RING * 4;      // float[128*3]
    static constexpr int WG_OWNER = WG_RACC + 128 * 3 * 4;   // u8[256]
    static constexpr int WG_MISC = WG_OWNER + TC_RING;       // tail, tile slots
    static constexpr int WG_BYTES = (WG_MISC + 64 + 1023) & ~1023;
    static constexpr int CTA_MISC = BLOB_PAD + 2 * WG_BYTES; // weight mbarrier
    static constexpr int SMEM = CTA_MISC + 64;
};

__device__ __forceinline__ uint32_t s_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }

__device__ __forceinline__ void tc_mbar_init(uint64_t* bar, int count) {
    asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;\n" :: "r"(s_u32(bar)), "r"(count));
}
__device__ __forceinline__ void tc_mbar_wait(uint64_t* bar, uint32_t parity) {
    uint32_t ok = 0;
    while (!ok) {
        asm volatile("{\n.reg .pred p;\nmbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\nselp.u32 %0, 1, 0, p;\n}\n"
                     : "=r"(ok) : "r"(s_u32(bar)), "r"(parity) : "memory");
    }
}
__device__ __forceinline__ uint32_t pack2(float lo, float hi) {
    uint32_t d;      // saturating: a feature beyond the fp16 range becomes +-65504, never inf
    asm("cvt.rn.satfinite.f16x2.f32 %0, %1, %2;\n" : "=r"(d) : "f"(hi), "f"(lo));
    return d;
}
__device__ __forceinline__ void wg_bar(int wg) { asm volatile("bar.sync %0, 128;\n" :: "r"(wg + 1) : "memory"); }
__device__ __forceinline__ bool wg_bar_or(int wg, bool pred) {
    uint32_t r;
    asm volatile("{\n.reg .pred p, q;\nsetp.ne.u32 p, %2, 0;\nbarrier.cta.red.or.pred q, %1, 128, p;\nselp.u32 %0, 1, 0, q;\n}\n"
                 : "=r"(r) : "r"(wg + 1), "r"((uint32_t)pred) : "memory");
    return r != 0;
}

struct TcRay {
    float sx, sy, sz, dx, dy, dz;
    int n_steps;
    float t_min, t_max;
};

// ACT: the rgbnet's hidden activation (K4_ACT_*); CfgB, the DirectMPIGO shape, is also built with gauss and lkrelu.
template <class Cfg, int ACT>
__global__ void __launch_bounds__(TC_THREADS, 1)
k4_march_tc_kernel(const __grid_constant__ K4Dev s, const __grid_constant__ K4RenderParams rp) {
    extern __shared__ __align__(1024) unsigned char smem[];
    constexpr int W = Cfg::W, KPAD = Cfg::KPAD, KCH = Cfg::KCH;
    const int tid = threadIdx.x, wg = tid >> 7, wt = tid & 127, lane = tid & 31, warp_in_wg = wt >> 5;

    unsigned char* blob = smem;
    unsigned char* wgb = smem + Cfg::BLOB_PAD + wg * Cfg::WG_BYTES;
    unsigned char* aring = wgb;
    float* qw = reinterpret_cast<float*>(wgb + Cfg::WG_QW);
    float* racc = reinterpret_cast<float*>(wgb + Cfg::WG_RACC);
    unsigned char* qowner = wgb + Cfg::WG_OWNER;
    volatile unsigned int* tailp = reinterpret_cast<volatile unsigned int*>(wgb + Cfg::WG_MISC);
    volatile long long* tile_slot = reinterpret_cast<volatile long long*>(wgb + Cfg::WG_MISC + 8);   // [2]
    uint64_t* wbar = reinterpret_cast<uint64_t*>(smem + Cfg::CTA_MISC);

    const TcBlobLayout BL = tc_blob_layout(KPAD, W);

    // ---------------- one-time CTA setup ----------------
    if (tid == 0) {
        tc_mbar_init(wbar, 1);
        asm volatile("fence.mbarrier_init.release.cluster;\n" ::: "memory");
    }
    {   // zero this warpgroup's block (A rings incl. their K padding, accumulators, counters)
        uint32_t* z = reinterpret_cast<uint32_t*>(wgb);
        for (int i = wt; i < (Cfg::WG_MISC + 32) / 4; i += TC_WG) z[i] = 0u;
    }
    __syncthreads();
    if (tid == 0) {
        asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;\n" :: "r"(s_u32(wbar)), "r"((uint32_t)BL.total) : "memory");
        asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];\n"
                     :: "r"(s_u32(blob)), "l"(s.tc_blob), "r"((uint32_t)BL.total), "r"(s_u32(wbar)) : "memory");
    }
    tc_mbar_wait(wbar, 0);
    const uint32_t a_ring_s = s_u32(aring);

    unsigned head = 0;
    unsigned long long tot_m = 0, tot_d = 0, tot_c = 0, n_batches = 0;
    const float mpi_den = (float)(rp.n_samples - 1);

    // One MLP batch over ring rows [head, head+128); `valid` of them are real samples.
    auto flush = [&](int valid) {
        const uint32_t a_tile = a_ring_s + ((head >> 7) & 1u) * Cfg::TILE_BYTES;
        asm volatile("fence.proxy.async.shared::cta;\n" ::: "memory");      // generic smem writes -> async proxy
        wg_bar(wg);
        if (wt == 0) ++n_batches;
        mlp_batch_wgmma<W, KPAD, true, ACT>(a_tile, blob, BL, valid, head & (TC_RING - 1), qw, qowner, nullptr, racc, wt, s.act_c,
                                            [] {}, true);
    };

    for (unsigned iter = 0;; ++iter) {
        // ---------------- next 128-ray tile of this warpgroup ----------------
        if (wt == 0) tile_slot[iter & 1] = (long long)atomicAdd(rp.tile_counter, 1u);
        wg_bar(wg);
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

        TcRay r;
        r.n_steps = 0; r.t_min = r.t_max = 0.f; r.sx = r.sy = r.sz = r.dx = r.dy = r.dz = 0.f;
        uint32_t vw[Cfg::NVW];
#pragma unroll
        for (int j = 0; j < Cfg::NVW; ++j) vw[j] = 0u;
        if (have_ray) {
            const Vec3 o = ld3(rp.rays_o, ray_i), d = ld3(rp.rays_d, ray_i);
            if (Cfg::KIND == K4_KIND_DVGO) {
                // infer_t_minmax / infer_n_samples / infer_ray_start_dir (render_utils_kernel.cu:12-79)
                const float vx = (d.x == 0.f) ? 1e-6f : d.x, vy = (d.y == 0.f) ? 1e-6f : d.y, vz = (d.z == 0.f) ? 1e-6f : d.z;
                const float ax = __fdiv_rn(__fsub_rn(s.xyz_max[0], o.x), vx), bx = __fdiv_rn(__fsub_rn(s.xyz_min[0], o.x), vx);
                const float ay = __fdiv_rn(__fsub_rn(s.xyz_max[1], o.y), vy), by = __fdiv_rn(__fsub_rn(s.xyz_min[1], o.y), vy);
                const float az = __fdiv_rn(__fsub_rn(s.xyz_max[2], o.z), vz), bz = __fdiv_rn(__fsub_rn(s.xyz_min[2], o.z), vz);
                r.t_min = fmaxf(fminf(fmaxf(fmaxf(fminf(ax, bx), fminf(ay, by)), fminf(az, bz)), rp.far_), rp.near_);
                r.t_max = fmaxf(fminf(fminf(fminf(fmaxf(ax, bx), fmaxf(ay, by)), fmaxf(az, bz)), rp.far_), rp.near_);
                float nn = __fmul_rn(d.y, d.y);
                nn = __fmaf_rn(d.x, d.x, nn);
                nn = __fmaf_rn(d.z, d.z, nn);
                const float rnorm = __fsqrt_rn(nn);
                const float ns = ceilf(__fdiv_rn(__fmul_rn(__fsub_rn(r.t_max, r.t_min), rnorm), rp.stepdist));
                r.n_steps = (ns > 1.f) ? ((ns >= 2147483520.f) ? 2147483647 : (int)ns) : 1;
                r.sx = __fmaf_rn(d.x, r.t_min, o.x); r.sy = __fmaf_rn(d.y, r.t_min, o.y); r.sz = __fmaf_rn(d.z, r.t_min, o.z);
                r.dx = __fdiv_rn(d.x, rnorm); r.dy = __fdiv_rn(d.y, rnorm); r.dz = __fdiv_rn(d.z, rnorm);
            } else {
                r.sx = o.x; r.sy = o.y; r.sz = o.z; r.dx = d.x; r.dy = d.y; r.dz = d.z;
                r.n_steps = rp.n_samples;
            }
            // view-direction embedding, packed once per ray (lib/dvgo.py:387-388)
            const Vec3 v = ld3(rp.viewdirs, ray_i);
            float ve[Cfg::NVEMB + 1];
            const float vv[3] = {v.x, v.y, v.z};
            ve[0] = vv[0]; ve[1] = vv[1]; ve[2] = vv[2];
#pragma unroll
            for (int c = 0; c < 3; ++c)
#pragma unroll
                for (int f = 0; f < Cfg::VIEWPE; ++f) {
                    const float a = __fmul_rn(vv[c], (float)(1 << f));
                    ve[3 + c * Cfg::VIEWPE + f] = sinf(a);
                    ve[3 + 3 * Cfg::VIEWPE + c * Cfg::VIEWPE + f] = cosf(a);
                }
            ve[Cfg::NVEMB] = 0.f;
#pragma unroll
            for (int j = 0; j < Cfg::NVW; ++j) vw[j] = pack2(ve[2 * j], ve[2 * j + 1]);
        }

        float T = 1.f, acc_depth = 0.f;
        int cnt_m = 0, cnt_d = 0, cnt_c = 0;
        bool done = !have_ray;
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
                const bool active = !done && (i < r.n_steps);
                if (!__any_sync(FULL, active)) break;
                bool shade = false;
                float w_sample = 0.f;
                Cell cell;
                float cw[8];
                int cidx[8];
                if (active) {
                    float px, py, pz;
                    if (Cfg::KIND == K4_KIND_DVGO) {
                        const float dist = __fmul_rn(rp.stepdist, (float)i);
                        px = __fmaf_rn(r.dx, dist, r.sx); py = __fmaf_rn(r.dy, dist, r.sy); pz = __fmaf_rn(r.dz, dist, r.sz);
                    } else {
                        const float dist = __fdiv_rn((float)i, mpi_den);
                        px = __fmaf_rn(r.dx, dist, r.sx); py = __fmaf_rn(r.dy, dist, r.sy); pz = __fmaf_rn(r.dz, dist, r.sz);
                    }
                    const bool outb = (s.xyz_min[0] > px) | (s.xyz_min[1] > py) | (s.xyz_min[2] > pz) |
                                      (s.xyz_max[0] < px) | (s.xyz_max[1] < py) | (s.xyz_max[2] < pz);
                    if (!outb) {
                        ++cnt_m;
                        const int mi = (int)roundf(__fmaf_rn(px, s.m_scale[0], s.m_shift[0]));
                        const int mj = (int)roundf(__fmaf_rn(py, s.m_scale[1], s.m_shift[1]));
                        const int mk = (int)roundf(__fmaf_rn(pz, s.m_scale[2], s.m_shift[2]));
                        bool occ = false;
                        if ((0 <= mi) & (mi < s.mX) & (0 <= mj) & (mj < s.mY) & (0 <= mk) & (mk < s.mZ))
                            occ = __ldg(s.mask + ((size_t)mi * s.mY + mj) * s.mZ + mk) != 0;
                        if (occ) {
                            ++cnt_d;
                            cell = make_cell(s, px, py, pz);
                            corner_setup(s, cell, cw, cidx);
                            float den = interp_density(s, cw, cidx);
                            float shift = s.act_shift;
                            if (Cfg::KIND == K4_KIND_DMPIGO) {
                                const int z0 = cell.z0, z1 = cell.z0 + 1;
                                float a = 0.f;
                                if (z0 >= 0 && z0 < s.mpi_depth) a = __fmul_rn(__ldg(s.act_grid + z0), cell.wz0);
                                if (z1 >= 0 && z1 < s.mpi_depth) a = __fmaf_rn(__ldg(s.act_grid + z1), cell.wz1, a);
                                den = __fadd_rn(den, a);
                                shift = 0.f;
                            }
                            const float e = expf(__fadd_rn(den, shift));
                            const float alpha = __fsub_rn(1.f, powf(__fadd_rn(1.f, e), -rp.interval));
                            if (!(s.thres > 0.f) || alpha > s.thres) {
                                const float w = __fmul_rn(T, alpha);
                                T = (float)((double)T * (1.0 - (double)alpha));
                                if ((double)T < 1e-3) done = true;
                                if (!(s.thres > 0.f) || w > s.thres) {
                                    shade = true;
                                    w_sample = w;
                                    ++cnt_c;
                                    if (rp.render_depth)
                                        acc_depth = __fadd_rn(acc_depth, __fmul_rn(w, __fmul_rn(__fadd_rn((float)i, 0.5f), rp.inv_nsamples)));
                                }
                            }
                        }
                    }
                }
                ++i;
                // ---------------- append surviving samples to the warpgroup's ring ----------------
                const unsigned bal = __ballot_sync(FULL, shade);
                if (bal != 0u) {
                    unsigned base = 0;
                    if (lane == 0) base = atomicAdd(const_cast<unsigned int*>(tailp), (unsigned)__popc(bal));
                    base = __shfl_sync(FULL, base, 0);
                    if (shade) {
                        const unsigned slot = (base + __popc(bal & ((1u << lane) - 1u))) & (TC_RING - 1);
                        float f[Cfg::NS];
                        interp_k0_cfg<Cfg::CPAD / 4>(s, cw, cidx, f);       // f[0..C) (CPAD >= C; extra lanes unused)
                        if (Cfg::KIND == K4_KIND_DMPIGO) {
                            const float pe[3] = {cell.cz, cell.cy, cell.cx};
                            f[Cfg::C + 0] = pe[0]; f[Cfg::C + 1] = pe[1]; f[Cfg::C + 2] = pe[2];
#pragma unroll
                            for (int c = 0; c < 3; ++c)
#pragma unroll
                                for (int q = 0; q < Cfg::SPAPE; ++q) {
                                    const float a = __fmul_rn(pe[c], (float)(1 << q));
                                    f[Cfg::C + 3 + c * Cfg::SPAPE + q] = sinf(a);
                                    f[Cfg::C + 3 + 3 * Cfg::SPAPE + c * Cfg::SPAPE + q] = cosf(a);
                                }
                        }
                        uint32_t row[KPAD / 2];
#pragma unroll
                        for (int j = 0; j < KPAD / 2; ++j) {
                            if (j < Cfg::NS / 2) row[j] = pack2(f[2 * j], f[2 * j + 1]);
                            else if (j < Cfg::NS / 2 + Cfg::NVW) row[j] = vw[j - Cfg::NS / 2];
                            else row[j] = 0u;
                        }
                        unsigned char* rowp = aring + (slot >> 7) * Cfg::TILE_BYTES + tc_canon_off((int)(slot & 127), 0, KCH);
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
            const bool live = wg_bar_or(wg, !done && (i < r.n_steps));
            const unsigned tail = *tailp;                          // stable: nobody appends before the next barrier
            if (tail - head >= 128u) {
                flush(128);
                head += 128u;
            } else if (!live) {
                if (tail != head) {
                    flush((int)(tail - head));
                    head += 128u;
                    wg_bar(wg);                                     // everyone has read `tail` and the ring
                    if (wt == 0) *tailp = head;
                }
                break;
            } else {
                wg_bar(wg);
            }
        }
        wg_bar(wg);                                                 // all atomics into racc have landed
        if (have_ray) {
            const float bgt = __fmul_rn(T, rp.bg);
            k4_store_ray(rp, ray_i, __fadd_rn(racc[wt * 3 + 0], bgt), __fadd_rn(racc[wt * 3 + 1], bgt),
                         __fadd_rn(racc[wt * 3 + 2], bgt), T, acc_depth);
            if (rp.ray_stats) reinterpret_cast<int4*>(rp.ray_stats)[ray_i] = make_int4(r.n_steps, cnt_m, cnt_d, cnt_c);
            if (rp.t_minmax) { rp.t_minmax[2 * ray_i] = r.t_min; rp.t_minmax[2 * ray_i + 1] = r.t_max; }
        }
        racc[wt * 3 + 0] = 0.f; racc[wt * 3 + 1] = 0.f; racc[wt * 3 + 2] = 0.f;
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
        }
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
    if (rp.image_w > 0) rp.n_tiles = (long long)((rp.image_w + 15) / 16) * ((rp.image_h + 7) / 8);
    else rp.n_tiles = (rp.n_rays + TC_WG - 1) / TC_WG;
    long long blocks = (rp.n_tiles + 1) / 2;
    if (blocks > sms) blocks = sms;                     // persistent: one CTA per SM
    if (blocks < 1) blocks = 1;
    kern<<<(unsigned)blocks, TC_THREADS, Cfg::SMEM, st>>>(sc->dev, rp);
    K4_CUDA_TRY(cudaGetLastError());
    return K4_OK;
}

using CfgA = TcCfg<K4_KIND_DVGO, 12, 4, 0, 128>;    // configs/default.py:107-119 fine stage
using CfgB = TcCfg<K4_KIND_DMPIGO, 9, 0, 0, 64>;    // configs/llff/llff_default_lg.py + fern_lg_joint_l1.py

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
