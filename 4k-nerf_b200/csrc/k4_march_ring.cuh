// k4_march_ring.cuh -- what the two wgmma marchers (k4_march_tc.cu, k4_march_ws.cu) share beyond k4_march_ray.cuh:
// the config (derived constants and shared-memory map), the TMA staging of the operand blob, the packed view embedding
// of a ray and the features of a surviving sample.  Each kernel reserves ring rows and stores them itself:
// k4_march_ws.cu packs a row chunk by chunk with the view words read from shared memory to stay under its 128 registers,
// k4_march_tc.cu builds the row in registers.  Marcher group wg synchronises its warpgroup on named barrier wg + 1.
#pragma once
#include "k4_internal.cuh"
#include "k4_march_common.cuh"
#include "k4_march_mlp.cuh"
#include "k4_ptx.cuh"

namespace {

constexpr int TC_WG = 128;           // threads of a warpgroup = rays of a tile = rows of an MLP batch
constexpr int TC_ROUND = 8;          // marching steps between warpgroup rendezvous when nothing is pending

// The operand blob (weights + bias tiles) from global to shared memory as one TMA bulk copy that completes on `bar`.
// One thread calls it, once bar's mbarrier.init is visible; everybody then waits for phase 0 of bar.
__device__ __forceinline__ void stage_blob(unsigned char* blob, const void* src, int bytes, uint64_t* bar) {
    mbar_arrive_expect_tx(bar, (uint32_t)bytes);
    bulk_g2s(blob, src, (uint32_t)bytes, bar);
}

// ---------------------------------------------------------------------------------------------
// A model shape one of the kernels is built for: an entry of K4_WS_CFG_LIST (k4_ws_cfgs.h) for k4_march_ws.cu, CfgA /
// CfgB (ID -1) for k4_march_tc.cu.  Row layout of the A operand (fp16): [per-sample features: k0 channels K0OFF..C-1, MPI
// position + its sin/cos, zero-padded to an even count NS][view embedding: v, sin, cos (NVEMB)][zeros to KPAD, but for
// layer 1's bias ones in columns BIASC, BIASC + 1].
// TILES: 128-row tiles of a marcher group's ring.  VWS: the marcher keeps its ray's packed view embedding in shared
// memory (WG_VW) rather than in registers.
// ---------------------------------------------------------------------------------------------
template <int ID_, int KIND_, int C_, int VIEWPE_, int SPAPE_, int W_, int DIRECT_, int TILES_, bool VWS_>
struct TcCfg {
    static constexpr int ID = ID_, KIND = KIND_, C = C_, VIEWPE = VIEWPE_, SPAPE = SPAPE_, W = W_, DIRECT = DIRECT_;
    static constexpr int TILES = TILES_, RING = TILES * 128;
    static constexpr bool VWS = VWS_;
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
    static constexpr int WG_VW = WG_QDIFF + (DIRECT ? 0 : RING * 3 * 4);     // u32[NVW][128]: packed view embedding per ray (VWS only)
    static constexpr int WG_MISC = WG_VW + (VWS ? NVW * 128 * 4 : 0);        // the kernel's control block: tail first, then its own
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
// launch geometry of the persistent wgmma marchers: 128-ray tiles (16x8 pixels of an image, or 128 consecutive rays), two
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

}  // namespace
