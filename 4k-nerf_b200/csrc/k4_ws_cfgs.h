// k4_ws_cfgs.h -- the shapes the warp-specialised wgmma marcher (k4_march_ws.cu) is instantiated for, shared by the
// kernel TU (instantiation + dispatch) and by k4_scene_create (which packs the rgbnet into the operand blob of the
// config a model runs on).
//
// A model does not need a config of exactly its own shape: a config COVERS every model of the same kind / direct-ness
// with at most as many k0 channels, view / position frequencies and hidden units.  The config's extra inputs meet zero
// weight columns.  A hidden unit the model does not have has zero incoming weights and bias, so its pre-activation is 0,
// but its activated value need not be (gauss(0) = 1): what makes it contribute nothing is that its OUTGOING weights --
// its column of W2 or W3 -- are exact zeros in the packed blob (k4_scene_create zeroes the blob and writes only the
// model's own rows and columns).  The fp32 and mma.sync packs never hold such units: their widths are the model's own,
// and the fp32 pack's padded columns (ldw > n_out) are computed but never read as inputs.  The first covering config in list order is used,
// so the list goes from cheap to expensive within a kind.  Shapes of the shipped reference configs come first:
//   configs/default.py:107-119            DVGO   k0 12, viewbase_pe 4 (ctor default lib/dvgo.py:33), width 128, direct
//   configs/syn/1x_chair_joint_l1+gan.py  DVGO   k0 12, viewbase_pe 0, width 128, direct
//   configs/llff/*.py                     MPI    k0  9, viewbase_pe 0, spatial_pe 0, width 64
//   lib/dcvgo.py with the fine-stage MLP  DCVGO  k0 12, viewbase_pe 4, width 128
// plus rgbnet_direct=False (lib/dvgo.py:100-104,412: first 3 k0 channels are a diffuse logit added before the sigmoid),
// 64-wide variants and one large MPI shape with view and position frequencies (lib/dmpigo.py:96-100).
#pragma once
#include "../../include/k4nerf.h"

//        id kind            C   vpe spe W    direct
#define K4_WS_CFG_LIST(X)                       \
    X(2,  K4_KIND_DVGO,   12, 0,  0,  64,  1)   \
    X(0,  K4_KIND_DVGO,   12, 0,  0,  128, 1)   \
    X(3,  K4_KIND_DVGO,   12, 4,  0,  64,  1)   \
    X(1,  K4_KIND_DVGO,   12, 4,  0,  128, 1)   \
    X(4,  K4_KIND_DVGO,   15, 4,  0,  128, 0)   \
    X(5,  K4_KIND_DVGO,   16, 6,  0,  128, 1)   \
    X(6,  K4_KIND_DMPIGO, 9,  0,  0,  64,  1)   \
    X(7,  K4_KIND_DMPIGO, 12, 4,  0,  128, 1)   \
    X(8,  K4_KIND_DMPIGO, 12, 4,  5,  128, 1)   \
    X(9,  K4_KIND_DCVGO,  12, 0,  0,  128, 1)   \
    X(10, K4_KIND_DCVGO,  12, 4,  0,  128, 1)   \
    X(11, K4_KIND_DCVGO,  16, 6,  0,  128, 1)

struct K4WsCfg { int id, kind, C, vpe, spe, W, direct; };

// per-sample features, padded to an even count (rows are packed as fp16 pairs; the per-ray view embedding follows)
constexpr int k4_ws_ns(const K4WsCfg& c) { return (c.direct ? c.C : c.C - 3) + (c.kind == K4_KIND_DMPIGO ? 3 + 6 * c.spe : 0); }
constexpr int k4_ws_nsp(const K4WsCfg& c) { return (k4_ws_ns(c) + 1) & ~1; }
constexpr int k4_ws_dim0(const K4WsCfg& c) { return k4_ws_nsp(c) + 3 + 6 * c.vpe; }
constexpr int k4_ws_kpad(const K4WsCfg& c) { return (k4_ws_dim0(c) + 15) & ~15; }
// Layer 1's bias rides inside K where the row has two spare columns: the first even column at or past the config's
// input count, if it and the next one lie below kpad; the rows hold fp16 1.0 there and W1 the bias hi / lo.  -1: no room,
// layer 1 adds its bias with one more MMA against the ONES tile.  Of the list above, every config with view frequencies
// folds (1, 3, 4, 10: column 40; 5, 11: 56; 7: 44; 8: 74); 0, 2, 6 and 9 (kpad 16 = 15 inputs + 1) do not.
constexpr int k4_ws_bias_col(const K4WsCfg& c) {
    return (((k4_ws_dim0(c) + 1) & ~1) + 1 < k4_ws_kpad(c)) ? ((k4_ws_dim0(c) + 1) & ~1) : -1;
}

inline const K4WsCfg* k4_ws_cfg_table(int* n) {
    static const K4WsCfg tab[] = {
#define K4_X(id, kind, C, vpe, spe, W, direct) {id, kind, C, vpe, spe, W, direct},
        K4_WS_CFG_LIST(K4_X)
#undef K4_X
    };
    *n = (int)(sizeof(tab) / sizeof(tab[0]));
    return tab;
}

// first config that covers the model (see the comment at the top), or nullptr.  want >= 0: the config of that id if it
// covers the model, else nullptr (K4_WS_CONFIG, k4_scene_create).
inline const K4WsCfg* k4_ws_pick(int kind, int C, int vpe, int spe, int width, int direct, int depth, int want = -1) {
    if (depth != 3) return nullptr;
    int n = 0;
    const K4WsCfg* tab = k4_ws_cfg_table(&n);
    if (kind != K4_KIND_DVGO) direct = 1;
    for (int i = 0; i < n; ++i) {
        const K4WsCfg& c = tab[i];
        if (want >= 0 && c.id != want) continue;
        if (c.kind != kind || c.direct != direct) continue;
        if (C > c.C || (!direct && C < 4) || vpe > c.vpe || spe > c.spe || width > c.W) continue;
        return &c;
    }
    return nullptr;
}
