// k4_march_ws.cu -- warp-specialised Hopper marcher: gather on the CUDA cores, the rgbnet as warpgroup MMAs in
// warpgroups of its own, so that marching never waits for the tensor core.
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
// Weights + bias tiles are staged once per CTA with a single TMA bulk copy.  The per-ray geometry and marching step are
// the one copy every marcher compiles (k4_march_ray.cuh); only the MLP runs in fp16 operands / fp32 accumulate.
#include "k4_internal.cuh"
#include "k4_march_common.cuh"
#include "k4_march_ray.cuh"
#include "k4_ws_cfgs.h"
#include "k4_march_mlp.cuh"
#include "k4_ptx.cuh"

namespace {

constexpr int TC_WG = 128;           // threads of a warpgroup = rays of a tile = rows of an MLP batch
constexpr int TC_ROUND = 8;          // marching steps between warpgroup rendezvous when nothing is pending
constexpr int TC_THREADS = 512;
constexpr int TC_TILES = 3;          // ring tiles per marcher group: one in the MLP group, one filling, one for a step's overflow

// The operand blob (weights + bias tiles) from global to shared memory as one TMA bulk copy that completes on `bar`.
// One thread calls it, once bar's mbarrier.init is visible; everybody then waits for phase 0 of bar.
__device__ __forceinline__ void stage_blob(unsigned char* blob, const void* src, int bytes, uint64_t* bar) {
    mbar_arrive_expect_tx(bar, (uint32_t)bytes);
    bulk_g2s(blob, src, (uint32_t)bytes, bar);
}

// ---------------------------------------------------------------------------------------------
// A model shape the kernel is built for: an entry of K4_WS_CFG_LIST (k4_ws_cfgs.h).  Row layout of the A operand (fp16):
// [per-sample features: k0 channels K0OFF..C-1, MPI position + its sin/cos, zero-padded to an even count NS][view
// embedding: v, sin, cos (NVEMB)][zeros to KPAD, but for layer 1's bias ones in columns BIASC, BIASC + 1].
// ---------------------------------------------------------------------------------------------
template <int ID_, int KIND_, int C_, int VIEWPE_, int SPAPE_, int W_, int DIRECT_>
struct TcCfg {
    static constexpr int ID = ID_, KIND = KIND_, C = C_, VIEWPE = VIEWPE_, SPAPE = SPAPE_, W = W_, DIRECT = DIRECT_;
    static constexpr int TILES = TC_TILES, RING = TILES * 128;
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
    // Layer 1's bias inside K: the first even column at or past DIM0, if it and the next one lie below KPAD, else -1
    // (k4_ws_bias_col).  Row word BIASW = NS/2 + NVW, the first padding word, holds fp16 1.0 in both halves, W1 the
    // bias hi / lo (mlp_batch_wgmma).  BIAS_STORED: the row store writes BIASW's chunk anyway and puts the word there;
    // otherwise the chunk is never written and the word is set once, when the ring is zeroed (bias_ones_ring).
    static constexpr int BIASC = (((DIM0 + 1) & ~1) + 1 < KPAD) ? ((DIM0 + 1) & ~1) : -1;
    static constexpr int BIASW = BIASC >= 0 ? BIASC / 2 : -1;
    static constexpr bool BIAS_STORED = BIASC >= 0 && (BIASW % 4) != 0;
    static_assert(BIASC < 0 || BIASW == NS / 2 + NVW, "the bias word is the row's first padding word");
    static_assert(W == 128 || W == 64, "hidden width");
    static_assert(DIRECT || KIND == K4_KIND_DVGO, "the diffuse term exists in DirectVoxGO only");
    // shared memory map: [blob][marcher group 0][marcher group 1][weight mbarrier]; offsets WG_* inside a group's block
    static constexpr int BLOB = W * KPAD * 2 + W * W * 2 + 16 * W * 2 + 2 * W * 16 * 2 + 16 * 16 * 2 + 128 * 16 * 2;
    static constexpr int BLOB_PAD = (BLOB + 1023) & ~1023;
    static constexpr int WG_A = TILES * TILE_BYTES;
    static constexpr int WG_QW = WG_A;                       // float[RING]
    static constexpr int WG_RACC = WG_QW + RING * 4;         // float[128*3]
    static constexpr int WG_OWNER = WG_RACC + 128 * 3 * 4;   // u8[RING]
    static constexpr int WG_QDIFF = WG_OWNER + RING;         // float[RING*3]: diffuse logits of the queued samples (!DIRECT only)
    static constexpr int WG_VW = WG_QDIFF + (DIRECT ? 0 : RING * 3 * 4);     // u32[NVW][128]: packed view embedding per ray
    static constexpr int WG_MISC = WG_VW + NVW * 128 * 4;                    // the control block (WgCtl)
    static constexpr int WG_BYTES = (WG_MISC + 128 + 1023) & ~1023;
    static constexpr int CTA_MISC = BLOB_PAD + 2 * WG_BYTES; // weight mbarrier
    static constexpr int SMEM = CTA_MISC + 64;
    static constexpr int PROF_SMEM = SMEM + 4 * PhaseClock::WORDS * 8;   // + the phase counters of a profiled kernel
    static_assert(PROF_SMEM <= 227 * 1024, "shared memory of one block");
};

constexpr uint32_t H2_ONES = 0x3C003C00u;   // fp16x2 (1.0, 1.0)

// Word j of a ring row outside the sample's features and view embedding: the bias ones or zero padding.
template <class Cfg>
__device__ __forceinline__ uint32_t row_pad_word(int j) { return j == Cfg::BIASW ? H2_ONES : 0u; }

// The bias ones of every row of a freshly zeroed ring of `rows` rows at `ring`, where the row store never writes them
// (!Cfg::BIAS_STORED).  Called by the 128 threads of one warpgroup after the zeroing is visible to them.
template <class Cfg>
__device__ __forceinline__ void bias_ones_ring(unsigned char* ring, int rows, int wt) {
    if constexpr (Cfg::BIASC >= 0 && !Cfg::BIAS_STORED)
        for (int r = wt; r < rows; r += TC_WG)
            *reinterpret_cast<uint32_t*>(ring + (r >> 7) * Cfg::TILE_BYTES + tc_canon_off(r & 127, Cfg::BIASC >> 3, Cfg::KCH) +
                                         (Cfg::BIASC & 7) * 2) = H2_ONES;
}

// ---------------------------------------------------------------------------------------------
// per ray
// ---------------------------------------------------------------------------------------------
// view-direction embedding, packed once per ray into NVW fp16 pairs (lib/dvgo.py:387-388)
template <class Cfg>
__device__ __forceinline__ void pack_view_embedding(Vec3 v, uint32_t vw[Cfg::NVW]) {
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
    for (int j = 0; j < Cfg::NVW; ++j) vw[j] = h2_sat(ve[2 * j], ve[2 * j + 1]);
}

// ---------------------------------------------------------------------------------------------
// per surviving sample
// ---------------------------------------------------------------------------------------------
// f[0..C): the k0 features; behind them DirectMPIGO's position code (lib/dmpigo.py:338,347-351); a zero where the row's
// feature count is odd.  The row takes f[K0OFF ..].
template <class Cfg>
__device__ __forceinline__ void sample_features(const K4Dev& s, const Cell& cell, const float cw[8], const int cidx[8], float f[Cfg::NF]) {
    interp_k0_cfg<Cfg::CPAD / 4>(s, cw, cidx, f);       // f[0..C) (CPAD >= C; extra lanes unused)
    if (Cfg::KIND == K4_KIND_DMPIGO) {
        const float pe[3] = {cell.cz, cell.cy, cell.cx};   // .flip(-1)
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
}

// ---------------------------------------------------------------------------------------------
// launch geometry of the persistent marcher: 128-ray tiles (16x8 pixels of an image, or 128 consecutive rays), two
// marcher groups per CTA, at most one CTA per SM.  Sets rp.n_tiles, returns the number of CTAs.
// ---------------------------------------------------------------------------------------------
inline long long wg_launch_geometry(K4RenderParams& rp, int sms) {
    if (rp.image_w > 0) rp.n_tiles = (long long)((rp.image_w + 15) / 16) * ((rp.image_h + 7) / 8);
    else rp.n_tiles = (rp.n_rays + TC_WG - 1) / TC_WG;
    long long blocks = (rp.n_tiles + 1) / 2;
    if (blocks > sms) blocks = sms;                     // persistent: one CTA per SM
    if (blocks < 1) blocks = 1;
    return blocks;
}

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
    constexpr int W = Cfg::W, KPAD = Cfg::KPAD;
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
    if (tid < 256) bias_ones_ring<Cfg>(wg_base(wg), Cfg::RING, wt);
    if (tid == 0) {
        mbar_init(wbar, 1);
        for (int g = 0; g < 2; ++g) {
            mbar_init(&wg_ctl(g)->full_bar, 1);
            mbar_init(&wg_ctl(g)->done_bar, 128);
        }
        mbar_init_fence();
    }
    __syncthreads();
    if (tid == 0) stage_blob(blob, s.tc_blob, BL.total, wbar);
    mbar_wait(wbar, 0);
    const PhaseClock clk{reinterpret_cast<unsigned long long*>(smem + Cfg::SMEM) + wg * PhaseClock::WORDS, PROF && wt == 0};
    auto mark = [&](int p) { if (PROF) clk(p); };
    if (PROF) clk.begin();

    if (wg >= 2) {
        // =====================================================================================
        // MLP warpgroup of marcher slot g = wg - 2
        // =====================================================================================
        const int g = wg - 2;
        WgCtl* c = wg_ctl(g);
        const uint32_t ring_s = smem_u32(wg_base(g));
        const float* qw = reinterpret_cast<const float*>(wg_base(g) + Cfg::WG_QW);
        const unsigned char* qowner = wg_base(g) + Cfg::WG_OWNER;
        const float* qdiff = reinterpret_cast<const float*>(wg_base(g) + Cfg::WG_QDIFF);
        float* racc = reinterpret_cast<float*>(wg_base(g) + Cfg::WG_RACC);
        uint32_t full_ph = 0;
        unsigned nb = 0;
        unsigned long long n_batches = 0;
        auto consumed = [&] { mbar_arrive(&c->done_bar); };      // 128 arrivals = DONE
        for (;;) {
            mbar_wait(&c->full_bar, full_ph); full_ph ^= 1;
            mark(K4_PH_L_WAIT_FULL);
            if (*reinterpret_cast<volatile unsigned int*>(&c->exit_flag)) break;
            const unsigned tile = nb % TC_TILES;
            if (wt == 0) ++n_batches;
            const int valid = *reinterpret_cast<volatile int*>(&c->valid[tile]);
            const bool last = *reinterpret_cast<volatile int*>(&c->last[tile]) != 0;
            if (PROF)
                mlp_batch_wgmma<W, KPAD, Cfg::DIRECT != 0, ACT, Cfg::BIASC>(ring_s + tile * Cfg::TILE_BYTES, blob, BL, valid, tile * 128u, qw,
                                                                qowner, qdiff, racc, wt, s.act_c, consumed, last, clk);
            else
                mlp_batch_wgmma<W, KPAD, Cfg::DIRECT != 0, ACT, Cfg::BIASC>(ring_s + tile * Cfg::TILE_BYTES, blob, BL, valid, tile * 128u, qw,
                                                                qowner, qdiff, racc, wt, s.act_c, consumed, last);
            ++nb;
        }
        if (rp.counters && wt == 0) atomicAdd(rp.counters + 3, n_batches);
        if (PROF) clk.end(n_batches, phases + ((size_t)blockIdx.x * 4 + wg) * K4_PHASE_SLOTS);
    } else {
        // =====================================================================================
        // marcher warpgroups
        // =====================================================================================
        unsigned char* wgb = wg_base(wg);      // the ring's tiles come first
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
            fence_proxy_async();
            named_bar(wg + 1);
            mark(K4_PH_M_RENDEZVOUS);
            while (n_done < n_sub) { mbar_wait(&ctl->done_bar, done_ph); done_ph ^= 1; ++n_done; }
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

            Ray r = no_ray();
            uint32_t vw[Cfg::NVW];
#pragma unroll
            for (int j = 0; j < Cfg::NVW; ++j) vw[j] = 0u;
            if (have_ray) {
                r = setup_ray<Cfg::KIND>(s, rp, ld3(rp.rays_o, ray_i), ld3(rp.rays_d, ray_i));
                pack_view_embedding<Cfg>(ld3(rp.viewdirs, ray_i), vw);
            }
            // kept in shared memory while marching, where it would hold NVW registers of the capped 128 for the whole tile
#pragma unroll
            for (int j = 0; j < Cfg::NVW; ++j) vws[j * 128] = vw[j];

            mark(K4_PH_M_SETUP);
            MarchState<Cfg::KIND> st(have_ray);
            int i = 0;

            for (;;) {
#pragma unroll 1
                for (int rr = 0; rr < TC_ROUND; ++rr) {
                    unsigned pend = 0;
                    if (lane == 0) pend = *tailp - head;
                    pend = __shfl_sync(FULL, pend, 0);
                    if (pend >= 128u) break;                           // a batch is complete: go submit it
                    const bool active = !st.done && (i < r.n_steps);
                    if (!__any_sync(FULL, active)) break;
                    bool shade = false;
                    float w_sample = 0.f;
                    Cell cell;
                    float cw[8];
                    int cidx[8];
                    if (active) shade = march_step<Cfg::KIND, true>(s, rp, r, mpi_den, st, i, w_sample, cell, cw, cidx);
                    ++i;
                    const unsigned bal = __ballot_sync(FULL, shade);
                    if (bal != 0u) {
                        unsigned base = 0;
                        if (lane == 0) base = atomicAdd(const_cast<unsigned int*>(tailp), (unsigned)__popc(bal));
                        base = __shfl_sync(FULL, base, 0);
                        if (shade) {
                            const unsigned slot = (base + __popc(bal & ((1u << lane) - 1u))) % (unsigned)Cfg::RING;
                            float f[Cfg::NF];
                            sample_features<Cfg>(s, cell, cw, cidx, f);
                            unsigned char* rowp = wgb + (slot >> 7) * Cfg::TILE_BYTES + tc_canon_off((int)(slot & 127), 0, Cfg::KCH);
#pragma unroll
                            for (int kc = 0; kc < Cfg::KCH; ++kc) {
                                if (kc * 4 >= Cfg::NS / 2 + Cfg::NVW) break;           // chunks that are all padding stay zero
                                uint32_t q[4];
#pragma unroll
                                for (int e = 0; e < 4; ++e) {
                                    const int j = 4 * kc + e;
                                    if (j < Cfg::NS / 2) q[e] = h2_sat(f[Cfg::K0OFF + 2 * j], f[Cfg::K0OFF + 2 * j + 1]);
                                    else if (j < Cfg::NS / 2 + Cfg::NVW) q[e] = vws[(j - Cfg::NS / 2) * 128];
                                    else q[e] = row_pad_word<Cfg>(j);
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
                const bool live = named_bar_or(wg + 1, !st.done && (i < r.n_steps));
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
            while (n_done < n_sub) { mbar_wait(&ctl->done_bar, done_ph); done_ph ^= 1; ++n_done; }
            named_bar(wg + 1);
            mark(K4_PH_M_DRAIN);
            if (have_ray) finish_ray(rp, ray_i, r, st, racc[wt * 3 + 0], racc[wt * 3 + 1], racc[wt * 3 + 2]);
            racc[wt * 3 + 0] = 0.f; racc[wt * 3 + 1] = 0.f; racc[wt * 3 + 2] = 0.f;
            tot_m += st.cnt_m; tot_d += st.cnt_d; tot_c += st.cnt_c;
            mark(K4_PH_M_STORE);
        }
        if (wt == 0) {   // all batches are consumed: release this slot's MLP group
            *reinterpret_cast<volatile unsigned int*>(&ctl->exit_flag) = 1u;
            __threadfence_block();
            mbar_arrive(&ctl->full_bar);
        }
        if (rp.counters) flush_counters(rp, tot_m, tot_d, tot_c, lane);
        mark(K4_PH_M_SETUP);
        if (PROF) clk.end(n_sub, phases + ((size_t)blockIdx.x * 4 + wg) * K4_PHASE_SLOTS);
    }
}

// the blob's W1 carries layer 1's bias where the config's kernels expect it (k4_scene_create packs by k4_ws_bias_col)
#define K4_X(id, kind, C, vpe, spe, W, direct)                                                                    \
    static_assert(TcCfg<id, kind, C, vpe, spe, W, direct>::BIASC ==                                \
                  k4_ws_bias_col(K4WsCfg{id, kind, C, vpe, spe, W, direct}), "layer-1 bias column of config " #id); \
    static_assert(TcCfg<id, kind, C, vpe, spe, W, direct>::KPAD == k4_ws_kpad(K4WsCfg{id, kind, C, vpe, spe, W, direct}));
K4_WS_CFG_LIST(K4_X)
#undef K4_X

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
    const long long blocks = wg_launch_geometry(rp, sms);
    if (phases && blocks > max_ctas) return K4_ERR_INVALID_ARG;
    if (n_ctas) *n_ctas = (int)blocks;
    K4_CUDA_TRY(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, smem));
    kern<<<(unsigned)blocks, TC_THREADS, smem, st>>>(sc->dev, rp, phases);
    K4_CUDA_TRY(cudaGetLastError());
    return K4_OK;
}

// k4_testing_rgbnet, wgmma modes: one CTA = one warpgroup = one batch of up to 128 caller rows.  The operand blob is staged
// as the marchers stage it; row r goes to ring-tile row r through the scene's column map (h2_sat, other columns zero), its
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
        mbar_init(bar, 1);
        mbar_init_fence();
    }
    __syncthreads();
    if (wt == 0) stage_blob(blob, s.tc_blob, BL.total, bar);
    const long long r0 = (long long)blockIdx.x * TC_WG;
    const int valid = (int)(n - r0 < TC_WG ? n - r0 : TC_WG);
    const long long r = r0 + wt;
    float f[KPAD];
#pragma unroll
    for (int k = 0; k < KPAD; ++k) f[k] = 0.f;
    if (wt < valid)
        for (int k = 0; k < s.dim0; ++k) f[__ldg(s.tc_colmap + k)] = xs[r * s.dim0 + k];
    if (Cfg::BIASC >= 0) f[Cfg::BIASC] = f[Cfg::BIASC + 1] = 1.f;
    unsigned char* rowp = tile + tc_canon_off(wt, 0, KCH);
#pragma unroll
    for (int kc = 0; kc < KCH; ++kc)
        *reinterpret_cast<uint4*>(rowp + kc * 128) = make_uint4(h2_sat(f[8 * kc + 0], f[8 * kc + 1]), h2_sat(f[8 * kc + 2], f[8 * kc + 3]),
                                                                h2_sat(f[8 * kc + 4], f[8 * kc + 5]), h2_sat(f[8 * kc + 6], f[8 * kc + 7]));
    qw[wt] = wt < valid ? ws[r] : 0.f;
    qowner[wt] = (unsigned char)(wt < valid ? (owners[r] & (TC_WG - 1)) : 0);
#pragma unroll
    for (int c = 0; c < 3; ++c) {
        qdiff[3 * wt + c] = (diffs && wt < valid) ? diffs[3 * r + c] : 0.f;
        racc[3 * wt + c] = 0.f;
    }
    fence_proxy_async();
    mbar_wait(bar, 0);
    __syncthreads();
    mlp_batch_wgmma<W, KPAD, Cfg::DIRECT != 0, ACT, Cfg::BIASC>(smem_u32(tile), blob, BL, valid, 0u, qw, qowner, qdiff, racc, wt, s.act_c, [] {}, true);
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

int k4_ws_row_layout(int id, int32_t out[4]) {
    switch (id) {
#define K4_X(id, kind, C, vpe, spe, W, direct)                                                  \
        case id: {                                                                              \
            using Cfg = TcCfg<id, kind, C, vpe, spe, W, direct>;                \
            out[0] = Cfg::DIM0; out[1] = Cfg::KPAD; out[2] = Cfg::BIASC; out[3] = Cfg::BIAS_STORED; \
            return K4_OK;                                                                       \
        }
        K4_WS_CFG_LIST(K4_X)
#undef K4_X
        default: return K4_ERR_INVALID_ARG;
    }
}
