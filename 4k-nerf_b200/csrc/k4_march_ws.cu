// k4_march_ws.cu -- warp-specialised Hopper marcher: the pipeline of k4_march_tc.cu with the MLP moved to
// its own warpgroup, so that marching never waits for the tensor core.
//
// CTA = 512 threads = 4 warpgroups (one persistent CTA per SM), 128 registers per thread in every group (the MLP
// groups hold a 64 x 128 fp32 accumulator next to the fp16 activations):
//   WG0, WG1  MARCHERS.  128 rays each (16x8 pixels), one thread per ray.  Surviving samples are
//             appended as fp16 feature rows to the warpgroup's 384-row ring (3 tiles of 128 rows in
//             the canonical K-major wgmma layout).  When 128 rows are pending the group fences,
//             barriers and arrives on its FULL mbarrier -- and keeps marching into the next tile.
//             Back-pressure: batch B may only be submitted once batch B-1 has been consumed (DONE
//             mbarrier), so one batch per marcher group is in flight while the next one fills.
//   WG2, WG3  MLP, one group per marcher slot: wait FULL -> the three layers as warpgroup MMAs with
//             register-resident activations (mlp_batch_wgmma, k4_march_mlp.cuh) -> arrive DONE once the
//             batch's rows and queue slots are read -> colours accumulated into the owning rays while the
//             marchers refill the ring.  A ray tile's last batch arrives on DONE only after its colours
//             (WgCtl::last), since the marchers read them next.  The two MLP groups and the two marcher
//             groups all run concurrently, so gathers, epilogues and MMAs of different batches overlap.
// Arithmetic is identical to k4_march_tc.cu (same rows, same MMAs, same epilogues).
#include "k4_internal.cuh"
#include "k4_march_common.cuh"
#include "k4_ws_cfgs.h"
#include "k4_march_mlp.cuh"

namespace {

constexpr int TC_THREADS = 512;
constexpr int TC_WG = 128;
constexpr int TC_TILES = 3;
constexpr int TC_RING = TC_TILES * 128;
constexpr int TC_ROUND = 8;          // marching steps between warpgroup rendezvous when nothing is pending

// One entry of K4_WS_CFG_LIST (k4_ws_cfgs.h).  Row layout of the A operand (fp16): [per-sample features: k0 channels
// K0OFF..C-1, MPI position + its sin/cos, zero-padded to an even count NS][view embedding: v, sin, cos (NVEMB)][zeros to KPAD].
template <int ID_, int KIND_, int C_, int VIEWPE_, int SPAPE_, int W_, int DIRECT_>
struct TcCfg {
    static constexpr int ID = ID_, KIND = KIND_, C = C_, VIEWPE = VIEWPE_, SPAPE = SPAPE_, W = W_, DIRECT = DIRECT_;
    static constexpr int CPAD = (C + 3) & ~3;
    static constexpr int NVEMB = 3 + 6 * VIEWPE;
    static constexpr int NPOS = (KIND == K4_KIND_DMPIGO) ? 3 + 6 * SPAPE : 0;
    static constexpr int K0OFF = DIRECT ? 0 : 3;        // rgbnet_direct=False: k0[0:3] is the diffuse logit (lib/dvgo.py:385-386,412)
    static constexpr int NS0 = C - K0OFF + NPOS;        // per-sample features
    static constexpr int NS = (NS0 + 1) & ~1;           // ... padded to an even count (rows are packed as fp16 pairs)
    static constexpr int NF = ((CPAD > C + NPOS) ? CPAD : C + NPOS) + 1;   // feature scratch (k0 quads, position code, pad)
    static constexpr int DIM0 = NS + NVEMB;
    static constexpr int KPAD = (DIM0 + 15) & ~15;
    static constexpr int KCH = KPAD / 8;                // 16-byte chunks per A row
    static constexpr int NVW = (NVEMB + 1) / 2;         // packed per-ray words
    static constexpr int TILE_BYTES = 128 * KPAD * 2;
    static_assert(W == 128 || W == 64, "hidden width");
    static_assert(DIRECT || KIND == K4_KIND_DVGO, "the diffuse term exists in DirectVoxGO only");
    // shared memory map
    static constexpr int BLOB = W * KPAD * 2 + W * W * 2 + 16 * W * 2 + 2 * W * 16 * 2 + 16 * 16 * 2 + 128 * 16 * 2;
    static constexpr int BLOB_PAD = (BLOB + 1023) & ~1023;
    static constexpr int WG_A = TC_TILES * TILE_BYTES;
    static constexpr int WG_QW = WG_A;                       // float[384]
    static constexpr int WG_RACC = WG_QW + TC_RING * 4;      // float[128*3]
    static constexpr int WG_OWNER = WG_RACC + 128 * 3 * 4;   // u8[384]
    static constexpr int WG_QDIFF = WG_OWNER + TC_RING;      // float[384*3]: diffuse logits of the queued samples (!DIRECT only)
    static constexpr int WG_VW = WG_QDIFF + (DIRECT ? 0 : TC_RING * 3 * 4);     // u32[NVW][128]: packed view embedding per ray
    static constexpr int WG_MISC = WG_VW + NVW * 128 * 4;    // tail, tile slots, valid counts, exit flag, mbarriers
    static constexpr int WG_BYTES = (WG_MISC + 128 + 1023) & ~1023;
    static constexpr int CTA_MISC = BLOB_PAD + 2 * WG_BYTES; // weight mbarrier
    static constexpr int SMEM = CTA_MISC + 64;
    static constexpr int PROF_SMEM = SMEM + 4 * PhaseClock::WORDS * 8;   // + the phase counters of the profiled kernel
    static_assert(PROF_SMEM <= 227 * 1024, "shared memory of one block");
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

__device__ __forceinline__ void mbar_arrive(uint64_t* bar) {
    asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];\n" :: "r"(s_u32(bar)) : "memory");
}
__device__ __forceinline__ bool mbar_test(uint64_t* bar, uint32_t parity) {
    uint32_t ok;
    asm volatile("{\n.reg .pred p;\nmbarrier.test_wait.parity.shared::cta.b64 p, [%1], %2;\nselp.u32 %0, 1, 0, p;\n}\n"
                 : "=r"(ok) : "r"(s_u32(bar)), "r"(parity) : "memory");
    return ok != 0;
}
__device__ __forceinline__ void named_bar(int id) { asm volatile("bar.sync %0, 128;\n" :: "r"(id) : "memory"); }

// per-marcher-group control block inside shared memory (at WG_MISC)
struct WgCtl {
    unsigned int tail;             // rows appended so far (monotonic)
    unsigned int exit_flag;        // set when the group has no more tiles
    long long tile_slot[2];
    int valid[TC_TILES];           // real rows of the batch in each ring tile
    int last[TC_TILES];            // the batch is its ray tile's last: DONE only once its colours are accumulated
    uint64_t full_bar;             // marcher -> MLP: a batch is complete            (count 1)
    uint64_t done_bar;             // MLP -> marcher: a batch's rows and queue slots are free, and for a tile's last
                                   // batch its colours are accumulated                (count 128)
};

// PROF: the profiled instantiation (k4_testing_march_phases).  It adds the phase marks of PhaseClock and nothing else, and
// writes each warpgroup's counters to phases[(blockIdx.x * 4 + wg) * K4_PHASE_SLOTS ..].  ACT: the rgbnet's hidden
// activation (K4_ACT_*); the DirectMPIGO configs are also built with gauss and lkrelu, the profiled kernel with relu only.
template <class Cfg, int ACT, bool PROF>
__global__ void __launch_bounds__(TC_THREADS, 1)
k4_march_ws_kernel(const __grid_constant__ K4Dev s, const __grid_constant__ K4RenderParams rp, unsigned long long* phases) {
    extern __shared__ __align__(1024) unsigned char smem[];
    constexpr int W = Cfg::W, KPAD = Cfg::KPAD, KCH = Cfg::KCH;
    const int tid = threadIdx.x, wg = tid >> 7, wt = tid & 127, lane = tid & 31, warp_in_wg = wt >> 5;

    unsigned char* blob = smem;
    uint64_t* wbar = reinterpret_cast<uint64_t*>(smem + Cfg::CTA_MISC);
    auto wg_base = [&](int g) { return smem + Cfg::BLOB_PAD + g * Cfg::WG_BYTES; };
    auto wg_ctl = [&](int g) { return reinterpret_cast<WgCtl*>(wg_base(g) + Cfg::WG_MISC); };

    const TcBlobLayout BL = tc_blob_layout(KPAD, W);

    // ---------------- one-time CTA setup ----------------
    if (tid < 256) {   // the two marcher groups zero their own blocks
        uint32_t* z = reinterpret_cast<uint32_t*>(wg_base(wg));
        for (int i = wt; i < (Cfg::WG_MISC + (int)sizeof(WgCtl)) / 4; i += TC_WG) z[i] = 0u;
    }
    __syncthreads();
    if (tid == 0) {
        tc_mbar_init(wbar, 1);
        for (int g = 0; g < 2; ++g) {
            tc_mbar_init(&wg_ctl(g)->full_bar, 1);
            tc_mbar_init(&wg_ctl(g)->done_bar, 128);
        }
        asm volatile("fence.mbarrier_init.release.cluster;\n" ::: "memory");
    }
    __syncthreads();
    if (tid == 0) {
        asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;\n" :: "r"(s_u32(wbar)), "r"((uint32_t)BL.total) : "memory");
        asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];\n"
                     :: "r"(s_u32(blob)), "l"(s.tc_blob), "r"((uint32_t)BL.total), "r"(s_u32(wbar)) : "memory");
    }
    tc_mbar_wait(wbar, 0);
    const PhaseClock clk{reinterpret_cast<unsigned long long*>(smem + Cfg::SMEM) + wg * PhaseClock::WORDS, PROF && wt == 0};
    auto mark = [&](int p) { if (PROF) clk(p); };
    if (PROF) clk.begin();

    if (wg >= 2) {
        // =====================================================================================
        // MLP warpgroup of marcher slot g = wg - 2
        // =====================================================================================
        const int g = wg - 2;
        WgCtl* c = wg_ctl(g);
        const uint32_t ring_s = s_u32(wg_base(g));
        const float* qw = reinterpret_cast<const float*>(wg_base(g) + Cfg::WG_QW);
        const unsigned char* qowner = wg_base(g) + Cfg::WG_OWNER;
        const float* qdiff = reinterpret_cast<const float*>(wg_base(g) + Cfg::WG_QDIFF);
        float* racc = reinterpret_cast<float*>(wg_base(g) + Cfg::WG_RACC);
        uint32_t full_ph = 0;
        unsigned nb = 0;
        unsigned long long n_batches = 0;
        auto consumed = [&] { mbar_arrive(&c->done_bar); };      // 128 arrivals = DONE
        for (;;) {
            tc_mbar_wait(&c->full_bar, full_ph); full_ph ^= 1;
            mark(K4_PH_L_WAIT_FULL);
            if (*reinterpret_cast<volatile unsigned int*>(&c->exit_flag)) break;
            const unsigned tile = nb % TC_TILES;
            if (wt == 0) ++n_batches;
            const int valid = *reinterpret_cast<volatile int*>(&c->valid[tile]);
            const bool last = *reinterpret_cast<volatile int*>(&c->last[tile]) != 0;
            if (PROF)
                mlp_batch_wgmma<W, KPAD, Cfg::DIRECT != 0, ACT>(ring_s + tile * Cfg::TILE_BYTES, blob, BL, valid, tile * 128u, qw,
                                                                qowner, qdiff, racc, wt, s.act_c, consumed, last, clk);
            else
                mlp_batch_wgmma<W, KPAD, Cfg::DIRECT != 0, ACT>(ring_s + tile * Cfg::TILE_BYTES, blob, BL, valid, tile * 128u, qw,
                                                                qowner, qdiff, racc, wt, s.act_c, consumed, last);
            ++nb;
        }
        if (rp.counters && wt == 0) atomicAdd(rp.counters + 3, n_batches);
        if (PROF) clk.end(n_batches, phases + ((size_t)blockIdx.x * 4 + wg) * K4_PHASE_SLOTS);
    } else {
        // =====================================================================================
        // marcher warpgroups
        // =====================================================================================
        unsigned char* wgb = wg_base(wg);
        unsigned char* aring = wgb;
        float* qw = reinterpret_cast<float*>(wgb + Cfg::WG_QW);
        float* racc = reinterpret_cast<float*>(wgb + Cfg::WG_RACC);
        unsigned char* qowner = wgb + Cfg::WG_OWNER;
        float* qdiff = reinterpret_cast<float*>(wgb + Cfg::WG_QDIFF);
        uint32_t* vws = reinterpret_cast<uint32_t*>(wgb + Cfg::WG_VW) + wt;     // this ray's words at a stride of 128
        WgCtl* ctl = wg_ctl(wg);
        volatile unsigned int* tailp = &ctl->tail;
        volatile long long* tile_slot = ctl->tile_slot;

        unsigned head = 0;                 // rows submitted so far (multiple of 128)
        unsigned n_sub = 0, n_done = 0;    // batches submitted / waited-for
        uint32_t done_ph = 0;
        unsigned long long tot_m = 0, tot_d = 0, tot_c = 0;
        const float mpi_den = (float)(rp.n_samples - 1);

        // hand the batch in ring tile (n_sub % 3) to the MLP group; `valid` real rows.
        // At most ONE batch per group is outstanding: the FULL mbarrier has a single pending phase,
        // so the arrive for batch B may only happen once batch B-1 has been consumed (DONE).  The
        // group keeps marching into the next tile(s) while its outstanding batch is in the MLP group;
        // with 3 ring tiles the rows of batches B+1 (filling) and B+2 (overflow of a step) never
        // alias the tile of the outstanding batch B.
        // `last`: no more rows of this ray tile follow, so the MLP group arrives on DONE only after the batch's
        // colours are in racc (other batches arrive as soon as their rows are read, before their epilogue).
        bool tile_open = false;            // a batch of this ray tile was submitted without `last`
        auto submit = [&](int valid, bool last) {
            asm volatile("fence.proxy.async.shared::cta;\n" ::: "memory");      // generic smem writes -> async proxy
            named_bar(wg + 1);
            mark(K4_PH_M_RENDEZVOUS);
            while (n_done < n_sub) { tc_mbar_wait(&ctl->done_bar, done_ph); done_ph ^= 1; ++n_done; }
            mark(K4_PH_M_WAIT_DONE);
            if (wt == 0) {
                *reinterpret_cast<volatile int*>(&ctl->valid[n_sub % TC_TILES]) = valid;
                *reinterpret_cast<volatile int*>(&ctl->last[n_sub % TC_TILES]) = last ? 1 : 0;
                __threadfence_block();
                mbar_arrive(&ctl->full_bar);
            }
            ++n_sub;
            head += 128u;
            tile_open = !last;
        };

        for (unsigned iter = 0;; ++iter) {
            if (wt == 0) tile_slot[iter & 1] = (long long)atomicAdd(rp.tile_counter, 1u);
            named_bar(wg + 1);
            const long long tile = tile_slot[iter & 1];
            if (tile >= rp.n_tiles) break;

            long long ray_i;
            if (rp.image_w > 0) {
                // Tiles are handed out centre first, image border last (rows centre-out, columns centre-out inside a row):
                // the rays through the middle of the volume are the long ones, so the expensive tiles start early and
                // the cheap ones fill the tail -- with only 2-3 tiles per warpgroup (a 1008x756 frame on 8 GPUs) the
                // order of the dynamic queue decides how long the last warpgroup runs.
                const int tiles_x = (rp.image_w + 15) >> 4, tiles_y = (rp.image_h + 7) >> 3;
                const int ty_s = (int)(tile / tiles_x), tx_s = (int)(tile - (long long)ty_s * tiles_x);
                const int ty = (ty_s & 1) ? (tiles_y >> 1) - ((ty_s + 1) >> 1) : (tiles_y >> 1) + (ty_s >> 1);
                const int tx = (tx_s & 1) ? (tiles_x >> 1) - ((tx_s + 1) >> 1) : (tiles_x >> 1) + (tx_s >> 1);
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
                } else if (Cfg::KIND == K4_KIND_DCVGO) {
                    // sample_ray, lib/dcvgo.py:237-238 (see k4_march.cu for the derivation)
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
            // kept in shared memory while marching, where it would hold NVW registers of the capped 128 for the whole tile
#pragma unroll
            for (int j = 0; j < Cfg::NVW; ++j) vws[j * 128] = vw[j];

            mark(K4_PH_M_SETUP);
            float T = 1.f, acc_depth = 0.f;
            int cnt_m = 0, cnt_d = 0, cnt_c = 0;
            bool done = !have_ray;
            int i = 0;
            float cum_dist = 0.f, qx = 0.f, qy = 0.f, qz = 0.f;      // DCVGO: cumdist_thres state, previous point

            for (;;) {
#pragma unroll 1
                for (int rr = 0; rr < TC_ROUND; ++rr) {
                    unsigned pend = 0;
                    if (lane == 0) pend = *tailp - head;
                    pend = __shfl_sync(FULL, pend, 0);
                    if (pend >= 128u) break;                           // a batch is complete: go submit it
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
                        } else if (Cfg::KIND == K4_KIND_DMPIGO) {
                            const float dist = __fdiv_rn((float)i, mpi_den);
                            px = __fmaf_rn(r.dx, dist, r.sx); py = __fmaf_rn(r.dy, dist, r.sy); pz = __fmaf_rn(r.dz, dist, r.sz);
                        }
                        bool outb;
                        float t_i = 0.f;
                        if (Cfg::KIND == K4_KIND_DCVGO) {
                            // lib/dcvgo.py:249-262,282-285: contracted sample + cumdist_thres (as k4_march.cu)
                            t_i = __ldg(rp.t_list + i);
                            px = __fadd_rn(r.sx, __fmul_rn(r.dx, t_i));
                            py = __fadd_rn(r.sy, __fmul_rn(r.dy, t_i));
                            pz = __fadd_rn(r.sz, __fmul_rn(r.dz, t_i));
                            const float nrm = fmaxf(fabsf(px), fmaxf(fabsf(py), fabsf(pz)));
                            const bool inner = nrm <= 1.f;
                            if (!inner) {
                                const float f = __fsub_rn(s.one_plus_bg, __fmul_rn(__fdiv_rn(1.f, nrm), s.bg_len));
                                px = __fmul_rn(__fdiv_rn(px, nrm), f);
                                py = __fmul_rn(__fdiv_rn(py, nrm), f);
                                pz = __fmul_rn(__fdiv_rn(pz, nrm), f);
                            }
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
                            const int mi = (int)roundf(__fmaf_rn(px, s.m_scale[0], s.m_shift[0]));
                            const int mj = (int)roundf(__fmaf_rn(py, s.m_scale[1], s.m_shift[1]));
                            const int mk = (int)roundf(__fmaf_rn(pz, s.m_scale[2], s.m_shift[2]));
                            bool occ = false;
                            const bool in_mask = (0 <= mi) & (mi < s.mX) & (0 <= mj) & (mj < s.mY) & (0 <= mk) & (mk < s.mZ);
                            if (in_mask) occ = __ldg(s.mask + ((size_t)mi * s.mY + mj) * s.mZ + mk) != 0;
                            if (Cfg::KIND != K4_KIND_DCVGO && !occ && in_mask && s.skip) {
                                // empty-space skipping: the following n steps are provably in-box and unoccupied
                                const float h = (Cfg::KIND == K4_KIND_DVGO) ? rp.stepdist : __fdiv_rn(1.f, mpi_den);
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
                                        if (rp.render_depth) {
                                            const float sd = (Cfg::KIND == K4_KIND_DCVGO)
                                                ? __fsub_rn(1.f, __fdiv_rn(1.f, __fadd_rn(1.f, t_i)))
                                                : __fmul_rn(__fadd_rn((float)i, 0.5f), rp.inv_nsamples);
                                            acc_depth = __fadd_rn(acc_depth, __fmul_rn(w, sd));
                                        }
                                    }
                                }
                            }
                        }
                    }
                    ++i;
                    const unsigned bal = __ballot_sync(FULL, shade);
                    if (bal != 0u) {
                        unsigned base = 0;
                        if (lane == 0) base = atomicAdd(const_cast<unsigned int*>(tailp), (unsigned)__popc(bal));
                        base = __shfl_sync(FULL, base, 0);
                        if (shade) {
                            const unsigned slot = (base + __popc(bal & ((1u << lane) - 1u))) % (unsigned)TC_RING;
                            float f[Cfg::NF];
                            interp_k0_cfg<Cfg::CPAD / 4>(s, cw, cidx, f);
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
                            if (Cfg::NS0 & 1) f[Cfg::K0OFF + Cfg::NS0] = 0.f;          // pad column of an odd feature count
                            unsigned char* rowp = aring + (slot >> 7) * Cfg::TILE_BYTES + tc_canon_off((int)(slot & 127), 0, KCH);
#pragma unroll
                            for (int kc = 0; kc < KCH; ++kc) {
                                if (kc * 4 >= Cfg::NS / 2 + Cfg::NVW) break;           // chunks that are all padding stay zero
                                uint32_t q[4];
#pragma unroll
                                for (int e = 0; e < 4; ++e) {
                                    const int j = 4 * kc + e;
                                    if (j < Cfg::NS / 2) q[e] = pack2(f[Cfg::K0OFF + 2 * j], f[Cfg::K0OFF + 2 * j + 1]);
                                    else if (j < Cfg::NS / 2 + Cfg::NVW) q[e] = vws[(j - Cfg::NS / 2) * 128];
                                    else q[e] = 0u;
                                }
                                *reinterpret_cast<uint4*>(rowp + kc * 128) = make_uint4(q[0], q[1], q[2], q[3]);
                            }
                            qw[slot] = w_sample;
                            qowner[slot] = (unsigned char)wt;
                            if (!Cfg::DIRECT) { qdiff[slot * 3 + 0] = f[0]; qdiff[slot * 3 + 1] = f[1]; qdiff[slot * 3 + 2] = f[2]; }
                        }
                    }
                }
                // ---------------- warpgroup rendezvous ----------------
                mark(K4_PH_M_MARCH);
                const bool live = wg_bar_or(wg, !done && (i < r.n_steps));
                mark(K4_PH_M_RENDEZVOUS);
                const unsigned tail = *tailp;                          // stable until the next barrier
                if (tail - head >= 128u) {
                    submit(128, !live && tail - head == 128u);
                } else if (!live) {
                    if (tail != head || tile_open) {                   // without rows the tile's last batch only carries `last`
                        submit((int)(tail - head), true);
                        named_bar(wg + 1);                             // everyone has read `tail`
                        if (wt == 0) *tailp = head;
                        mark(K4_PH_M_RENDEZVOUS);
                    }
                    break;
                } else {
                    named_bar(wg + 1);
                    mark(K4_PH_M_RENDEZVOUS);
                }
            }
            // all of this tile's batches must be consumed before the accumulators are read
            while (n_done < n_sub) { tc_mbar_wait(&ctl->done_bar, done_ph); done_ph ^= 1; ++n_done; }
            named_bar(wg + 1);
            mark(K4_PH_M_DRAIN);
            if (have_ray) {
                const float bgt = __fmul_rn(T, rp.bg);
                k4_store_ray(rp, ray_i, __fadd_rn(racc[wt * 3 + 0], bgt), __fadd_rn(racc[wt * 3 + 1], bgt),
                             __fadd_rn(racc[wt * 3 + 2], bgt), T, acc_depth);
                if (rp.ray_stats) reinterpret_cast<int4*>(rp.ray_stats)[ray_i] = make_int4(r.n_steps, cnt_m, cnt_d, cnt_c);
                if (rp.t_minmax) { rp.t_minmax[2 * ray_i] = r.t_min; rp.t_minmax[2 * ray_i + 1] = r.t_max; }
            }
            racc[wt * 3 + 0] = 0.f; racc[wt * 3 + 1] = 0.f; racc[wt * 3 + 2] = 0.f;
            tot_m += cnt_m; tot_d += cnt_d; tot_c += cnt_c;
            mark(K4_PH_M_STORE);
        }
        if (wt == 0) {   // all batches are consumed: release this slot's MLP group
            *reinterpret_cast<volatile unsigned int*>(&ctl->exit_flag) = 1u;
            __threadfence_block();
            mbar_arrive(&ctl->full_bar);
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
        }
        mark(K4_PH_M_SETUP);
        if (PROF) clk.end(n_sub, phases + ((size_t)blockIdx.x * 4 + wg) * K4_PHASE_SLOTS);
    }
}

// phases: NULL for the production kernel, else the profiled one writes there (room for max_ctas CTAs); *n_ctas: CTAs launched
template <class Cfg, int ACT>
int launch_ws(const k4_scene* sc, K4RenderParams rp, cudaStream_t st, unsigned long long* phases, int max_ctas, int* n_ctas) {
    if (sc->dev.Cpad != Cfg::CPAD) return K4_ERR_UNSUPPORTED;     // the k0 gather's stride is the config's
    auto kern = k4_march_ws_kernel<Cfg, ACT, false>;
    int smem = Cfg::SMEM;
    if constexpr (ACT == K4_ACT_RELU) {
        if (phases) { kern = k4_march_ws_kernel<Cfg, ACT, true>; smem = Cfg::PROF_SMEM; }
    } else if (phases) {
        return K4_ERR_UNSUPPORTED;                              // the profiled kernel is built with relu only
    }
    int dev = 0, sms = 0;
    K4_CUDA_TRY(cudaGetDevice(&dev));
    K4_CUDA_TRY(cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev));
    if (rp.image_w > 0) rp.n_tiles = (long long)((rp.image_w + 15) / 16) * ((rp.image_h + 7) / 8);
    else rp.n_tiles = (rp.n_rays + TC_WG - 1) / TC_WG;
    long long blocks = (rp.n_tiles + 1) / 2;
    if (blocks > sms) blocks = sms;                     // persistent: one CTA per SM
    if (blocks < 1) blocks = 1;
    if (phases && blocks > max_ctas) return K4_ERR_INVALID_ARG;
    if (n_ctas) *n_ctas = (int)blocks;
    K4_CUDA_TRY(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, smem));
    kern<<<(unsigned)blocks, TC_THREADS, smem, st>>>(sc->dev, rp, phases);
    K4_CUDA_TRY(cudaGetLastError());
    return K4_OK;
}

// k4_testing_rgbnet, wgmma modes: one CTA = one warpgroup = one batch of up to 128 caller rows.  The operand blob is staged
// as the marchers stage it; row r goes to ring-tile row r through the scene's column map (pack2, other columns zero), its
// weight / owner / diffuse logits to the queue, and mlp_batch_wgmma accumulates the colours into racc.
template <class Cfg, int ACT>
__global__ void __launch_bounds__(TC_WG, 1)
k4_test_rgbnet_ws_kernel(const __grid_constant__ K4Dev s, const float* __restrict__ xs, const float* __restrict__ diffs,
                         const float* __restrict__ ws, const int* __restrict__ owners, long long n, float* __restrict__ racc_out) {
    extern __shared__ __align__(1024) unsigned char smem[];
    constexpr int W = Cfg::W, KPAD = Cfg::KPAD, KCH = Cfg::KCH;
    unsigned char* blob = smem;
    unsigned char* tile = smem + Cfg::BLOB_PAD;
    float* qw = reinterpret_cast<float*>(tile + Cfg::TILE_BYTES);
    float* qdiff = qw + TC_WG;
    float* racc = qdiff + TC_WG * 3;
    unsigned char* qowner = reinterpret_cast<unsigned char*>(racc + TC_WG * 3);
    uint64_t* bar = reinterpret_cast<uint64_t*>(qowner + TC_WG);
    const int wt = threadIdx.x;
    const TcBlobLayout BL = tc_blob_layout(KPAD, W);

    if (wt == 0) {
        tc_mbar_init(bar, 1);
        asm volatile("fence.mbarrier_init.release.cluster;\n" ::: "memory");
    }
    __syncthreads();
    if (wt == 0) {
        asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;\n" :: "r"(s_u32(bar)), "r"((uint32_t)BL.total) : "memory");
        asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];\n"
                     :: "r"(s_u32(blob)), "l"(s.tc_blob), "r"((uint32_t)BL.total), "r"(s_u32(bar)) : "memory");
    }
    const long long r0 = (long long)blockIdx.x * TC_WG;
    const int valid = (int)(n - r0 < TC_WG ? n - r0 : TC_WG);
    const long long r = r0 + wt;
    float f[KPAD];
#pragma unroll
    for (int k = 0; k < KPAD; ++k) f[k] = 0.f;
    if (wt < valid)
        for (int k = 0; k < s.dim0; ++k) f[__ldg(s.tc_colmap + k)] = xs[r * s.dim0 + k];
    unsigned char* rowp = tile + tc_canon_off(wt, 0, KCH);
#pragma unroll
    for (int kc = 0; kc < KCH; ++kc)
        *reinterpret_cast<uint4*>(rowp + kc * 128) = make_uint4(pack2(f[8 * kc + 0], f[8 * kc + 1]), pack2(f[8 * kc + 2], f[8 * kc + 3]),
                                                                pack2(f[8 * kc + 4], f[8 * kc + 5]), pack2(f[8 * kc + 6], f[8 * kc + 7]));
    qw[wt] = wt < valid ? ws[r] : 0.f;
    qowner[wt] = (unsigned char)(wt < valid ? (owners[r] & (TC_WG - 1)) : 0);
#pragma unroll
    for (int c = 0; c < 3; ++c) {
        qdiff[3 * wt + c] = (diffs && wt < valid) ? diffs[3 * r + c] : 0.f;
        racc[3 * wt + c] = 0.f;
    }
    asm volatile("fence.proxy.async.shared::cta;\n" ::: "memory");      // generic smem writes -> async proxy
    tc_mbar_wait(bar, 0);
    __syncthreads();
    mlp_batch_wgmma<W, KPAD, Cfg::DIRECT != 0, ACT>(s_u32(tile), blob, BL, valid, 0u, qw, qowner, qdiff, racc, wt, s.act_c, [] {}, true);
    __syncthreads();
#pragma unroll
    for (int c = 0; c < 3; ++c) racc_out[3 * (r0 + wt) + c] = racc[3 * wt + c];
}

template <class Cfg, int ACT>
int launch_test_rgbnet_ws(const k4_scene* sc, const k4_rgbnet_test_args* a, cudaStream_t st) {
    auto kern = k4_test_rgbnet_ws_kernel<Cfg, ACT>;
    constexpr int smem = Cfg::BLOB_PAD + Cfg::TILE_BYTES + TC_WG * (4 + 12 + 12 + 1) + 16;
    K4_CUDA_TRY(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, smem));
    const long long blocks = (a->n + TC_WG - 1) / TC_WG;
    kern<<<(unsigned)blocks, TC_WG, smem, st>>>(sc->dev, a->d_x, a->d_diffuse, a->d_w, a->d_owner, a->n, a->d_racc);
    K4_CUDA_TRY(cudaGetLastError());
    return K4_OK;
}

// The instantiation of a config for the scene's activation: relu for every config, gauss and lkrelu for the DirectMPIGO
// ones (the only kind whose reference builds them).
template <class Cfg>
int launch_ws_act(const k4_scene* sc, K4RenderParams rp, cudaStream_t st, unsigned long long* phases, int max_ctas, int* n_ctas) {
    if constexpr (Cfg::KIND == K4_KIND_DMPIGO) {
        if (sc->act == K4_ACT_GAUSS) return launch_ws<Cfg, K4_ACT_GAUSS>(sc, rp, st, phases, max_ctas, n_ctas);
        if (sc->act == K4_ACT_LKRELU) return launch_ws<Cfg, K4_ACT_LKRELU>(sc, rp, st, phases, max_ctas, n_ctas);
    }
    if (sc->act != K4_ACT_RELU) return K4_ERR_UNSUPPORTED;
    return launch_ws<Cfg, K4_ACT_RELU>(sc, rp, st, phases, max_ctas, n_ctas);
}
template <class Cfg>
int launch_test_rgbnet_ws_act(const k4_scene* sc, const k4_rgbnet_test_args* a, cudaStream_t st) {
    if constexpr (Cfg::KIND == K4_KIND_DMPIGO) {
        if (sc->act == K4_ACT_GAUSS) return launch_test_rgbnet_ws<Cfg, K4_ACT_GAUSS>(sc, a, st);
        if (sc->act == K4_ACT_LKRELU) return launch_test_rgbnet_ws<Cfg, K4_ACT_LKRELU>(sc, a, st);
    }
    if (sc->act != K4_ACT_RELU) return K4_ERR_UNSUPPORTED;
    return launch_test_rgbnet_ws<Cfg, K4_ACT_RELU>(sc, a, st);
}

}  // namespace

int k4_testing_rgbnet_ws(const k4_scene* sc, const k4_rgbnet_test_args* a, cudaStream_t st) {
    if (!sc->dev.tc_blob || !sc->dev.tc_colmap) return K4_ERR_UNSUPPORTED;
    switch (sc->dev.tc_cfg) {
#define K4_X(id, kind, C, vpe, spe, W, direct) case id: return launch_test_rgbnet_ws_act<TcCfg<id, kind, C, vpe, spe, W, direct>>(sc, a, st);
        K4_WS_CFG_LIST(K4_X)
#undef K4_X
        default: return K4_ERR_UNSUPPORTED;
    }
}

int k4_launch_march_ws(const k4_scene* sc, K4RenderParams rp, cudaStream_t st, unsigned long long* phases, int max_ctas, int* n_ctas) {
    if (!sc->dev.tc_blob) return K4_ERR_UNSUPPORTED;
    switch (sc->dev.tc_cfg) {
#define K4_X(id, kind, C, vpe, spe, W, direct) \
        case id: return launch_ws_act<TcCfg<id, kind, C, vpe, spe, W, direct>>(sc, rp, st, phases, max_ctas, n_ctas);
        K4_WS_CFG_LIST(K4_X)
#undef K4_X
        default: return K4_ERR_UNSUPPORTED;
    }
}

bool k4_ws_supported(const K4Dev& v) { return v.tc_blob != nullptr && v.tc_cfg >= 0; }
