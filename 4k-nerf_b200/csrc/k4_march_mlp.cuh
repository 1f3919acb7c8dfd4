// k4_march_mlp.cuh -- the rgbnet of the warp-specialised marcher (k4_march_ws.cu) on Hopper warpgroup MMAs.
//
// One warpgroup runs a batch of 128 queued sample rows through the three layers, 64 rows (one wgmma M) at a time:
//   L1  acc[64 x W] = A(ring tile, smem) * W1(smem) + bias             wgmma SS, fp32 accumulate in registers
//   E1  activation + cvt to fp16x2 of the accumulator = the A fragments of L2   (no trip through shared memory;
//       relu is the fused cvt.rn.relu.f16x2, gauss / lkrelu are evaluated in fp32 first: mlp_act_h2)
//   L2  acc[64 x W] = H1(registers) * W2(smem) + bias                  wgmma RS
//   E2  same repack -> H2
//   L3  acc[64 x 8] = H2(registers) * W3(smem) + bias -> sigmoid -> weight -> shared-memory atomicAdd into the ray
// A bias is one more K=16 MMA against the constant ONES tile of the operand blob (bias = fp16 hi + fp16 lo columns), as
// in the blob's layout (tc_blob_layout) -- except layer 1's where the config has room for it inside K (TcCfg::BIASC):
// there the ring rows carry fp16 1.0 in two padding columns and W1 the bias hi / lo in the same columns, so the bias
// products ride in L1's last k16 step.
#pragma once
#include "k4_march_common.cuh"
#include "k4_ptx.cuh"
#include "k4_wgmma.cuh"

// act(lo), act(hi) as one fp16x2 word: relu stays the fused cvt.rn.relu; the other activations are evaluated in fp32
// on the accumulator (RgbAct::tc, c = K4Dev::act_c) and rounded once.
template <int ACT>
__device__ __forceinline__ uint32_t mlp_act_h2(float lo, float hi, float c) {
    if constexpr (ACT == K4_ACT_RELU) {
        return h2_relu_sat(lo, hi);
    } else {
        const float h = RgbAct<ACT>::tc(hi, c), l = RgbAct<ACT>::tc(lo, c);
        return h2_sat(l, h);
    }
}

// 64 accumulator columns (block nc of a hidden layer) -> activated fp16 A fragments of k16 steps 4*nc .. 4*nc+3
template <int ACT>
__device__ __forceinline__ void mlp_repack(const float (&acc)[32], uint32_t (*h)[4], float c) {
#pragma unroll
    for (int q = 0; q < 4; ++q) {
        h[q][0] = mlp_act_h2<ACT>(acc[8 * q + 0], acc[8 * q + 1], c);     // row g,     k 2t, 2t+1
        h[q][1] = mlp_act_h2<ACT>(acc[8 * q + 2], acc[8 * q + 3], c);     // row g + 8
        h[q][2] = mlp_act_h2<ACT>(acc[8 * q + 4], acc[8 * q + 5], c);     // row g,     k 2t+8, 2t+9
        h[q][3] = mlp_act_h2<ACT>(acc[8 * q + 6], acc[8 * q + 7], c);     // row g + 8
    }
}

// Phase accounting of the profiled ws marcher (k4_testing_march_phases): mark(p) charges the SM cycles since the previous
// mark to counter p (K4_PH_*) of the warpgroup.  Thread 0 of the group keeps the clock and the counters in shared memory.
// NoPhases, the marker of every production kernel, compiles to nothing.
struct NoPhases {
    __device__ __forceinline__ void operator()(int) const {}
};
struct PhaseClock {
    static constexpr int START = K4_PHASE_SLOTS, LAST = K4_PHASE_SLOTS + 1, WORDS = K4_PHASE_SLOTS + 2;
    unsigned long long* ctr;     // [WORDS]: the counters, the group's start, the previous mark
    bool on;                     // thread 0 of the warpgroup
    __device__ __forceinline__ void begin() const {
        if (!on) return;
        for (int i = 0; i < K4_PHASE_SLOTS; ++i) ctr[i] = 0ull;
        ctr[START] = ctr[LAST] = clock64_now();
    }
    __device__ __forceinline__ void operator()(int p) const {
        if (!on) return;
        const unsigned long long t = clock64_now();
        ctr[p] += t - ctr[LAST];
        ctr[LAST] = t;
    }
    // the elapsed cycles and the batch count into slots K4_PH_ELAPSED / 7, all slots to out[0 .. K4_PHASE_SLOTS)
    __device__ __forceinline__ void end(unsigned long long batches, unsigned long long* out) const {
        if (!on) return;
        ctr[K4_PH_ELAPSED] = ctr[LAST] - ctr[START];
        ctr[K4_PHASE_SLOTS - 1] = batches;
        for (int i = 0; i < K4_PHASE_SLOTS; ++i) out[i] = ctr[i];
    }
};

// What the epilogue needs of a lane's two rows of a 64-row half (rows g and g + 8 of its warp's 16): channel t's logit
// (o[0] / o[2] of the m64n8 accumulator, diffuse term added), the sample weight and the owning ray; owner -1 for a row
// beyond `valid` and for lane t == 3, which has no channel.
struct MlpEpiRows {
    float logit[2], w[2];
    int owner[2];
};

// The rows' weights, owners and diffuse logits (into logit[], 0 for DIRECT): shared-memory reads that do not depend on L3,
// issued while its MMAs run.
template <bool DIRECT>
__device__ __forceinline__ MlpEpiRows mlp_epi_inputs(int row0, int valid, unsigned slot0, const float* qw, const unsigned char* qowner,
                                                     const float* qdiff, int t) {
    MlpEpiRows e;
#pragma unroll
    for (int rr = 0; rr < 2; ++rr) {
        const int row = row0 + 8 * rr;
        e.logit[rr] = 0.f;
        e.w[rr] = 0.f;
        e.owner[rr] = -1;
        if (t < 3 && row < valid) {
            const unsigned slot = slot0 + (unsigned)row;
            if (!DIRECT) e.logit[rr] = qdiff[slot * 3 + t];
            e.w[rr] = qw[slot];
            e.owner[rr] = qowner[slot];
        }
    }
    return e;
}

// ... and the retired L3 accumulator: logit = rgb_logit (+ k0_diffuse)
template <bool DIRECT>
__device__ __forceinline__ void mlp_epi_logits(MlpEpiRows& e, const float (&o)[4]) {
#pragma unroll
    for (int rr = 0; rr < 2; ++rr) e.logit[rr] = DIRECT ? o[2 * rr] : __fadd_rn(o[2 * rr], e.logit[rr]);
}

// w * sigmoid(logit) of the rows, added to racc[3 * owner + t].  A shared-memory float atomicAdd is a compare-and-swap
// loop on sm_90; per-warp accumulator slices with plain adds and a same-owner check instead measured 1 % slower per
// frame, so the atomics stay.
__device__ __forceinline__ void mlp_epilogue(const MlpEpiRows& e, float* racc, int t) {
#pragma unroll
    for (int rr = 0; rr < 2; ++rr)
        if (e.owner[rr] >= 0) atomicAdd(racc + e.owner[rr] * 3 + t, e.w[rr] * sigmoid_ref(e.logit[rr]));
}

// Rows [0, valid) of the ring tile at shared address a_tile (canonical K-major, KPAD/8 chunks per row).  Row r is
// queue slot slot0 + r: its colour, weighted by qw[slot], is added to racc[3 * qowner[slot] + c].  Called by all 128
// threads of one warpgroup (wt = thread index in the group); `valid` must be the same for all of them.
//
// consumed() is called once by every thread when the batch's ring rows and queue slots may be reused: after the last
// L3 has retired and the last half's epilogue inputs are in registers.  That epilogue runs after it, while the marchers
// already fill the ring, unless colour_first is set; then consumed() also means "colours accumulated".  Running the
// first half's epilogue under the second half's L1 MMAs instead keeps the accumulator, the epilogue and its inputs
// live at once: the 128-wide configurations then need 150 registers of the 128 and ptxas serialises the wgmmas (C7518).
// `mark` receives the phase boundaries (PhaseClock).  ACT: the hidden activation of E1 / E2 (K4_ACT_*), act_c its
// constant (K4Dev::act_c; unused by relu).  BIASC: the first of the two columns of the A tile that hold fp16 1.0 and of W1
// that hold layer 1's bias hi / lo (TcCfg::BIASC), -1 where layer 1 adds its bias against the ONES tile.
template <int W, int KPAD, bool DIRECT, int ACT, int BIASC, class Consumed, class Mark = NoPhases>
__device__ __forceinline__ void mlp_batch_wgmma(uint32_t a_tile, const unsigned char* blob, const TcBlobLayout& BL, int valid,
                                                unsigned slot0, const float* qw, const unsigned char* qowner, const float* qdiff,
                                                float* racc, int wt, float act_c, const Consumed& consumed, bool colour_first,
                                                const Mark& mark = Mark()) {
    constexpr int KCH = KPAD / 8, KCHW = W / 8, NC = W / 64;      // NC: 64-column blocks of a hidden layer
    static_assert(W % 64 == 0, "hidden width");
    static_assert(BIASC < 0 || (BIASC % 2 == 0 && BIASC + 1 < KPAD), "layer-1 bias columns");
    const int warp = wt >> 5, g = (wt & 31) >> 2, t = wt & 3;
    const uint32_t blob_s = smem_u32(blob);
    const uint32_t w1 = blob_s + BL.off_w1, w2 = blob_s + BL.off_w2, w3 = blob_s + BL.off_w3;
    const uint32_t b1 = blob_s + BL.off_b1, b2 = blob_s + BL.off_b2, b3 = blob_s + BL.off_b3, ones = blob_s + BL.off_ones;
    const uint64_t d_ones = wg_desc(ones, 128, 256);
    const int halves = valid > 64 ? 2 : (valid > 0 ? 1 : 0);
    MlpEpiRows pend;                                    // the last half's epilogue inputs
#pragma unroll 1
    for (int mh = 0; mh < halves; ++mh) {
        const uint32_t a_half = a_tile + mh * 8 * KCH * 128;
        uint32_t h1[W / 16][4], h2[W / 16][4];
        // L1 and L2 each run as ONE chain over all W output columns.  Splitting them into 64-column chains that differ
        // only in their B descriptor is not safe: ptxas of CUDA 12.9 merges such chains and feeds the first chunk's
        // result to every chunk.
        {
            float acc[W / 2];
            wg_fence();
#pragma unroll
            for (int k = 0; k < KPAD / 16; ++k)
                wgmma_ss(acc, wg_desc(a_half + k * 256, 128, KCH * 128), wg_desc(w1 + k * 256, 128, KCH * 128), k > 0);
            if constexpr (BIASC < 0) wgmma_ss(acc, d_ones, wg_desc(b1, 128, 256), 1);
            wg_commit();
            wg_wait<0>();
            wg_fence_acc(acc);
            mark(K4_PH_L_L1);
#pragma unroll
            for (int nc = 0; nc < NC; ++nc) mlp_repack<ACT>(*reinterpret_cast<const float (*)[32]>(acc + 32 * nc), h1 + 4 * nc, act_c);
            mark(K4_PH_L_REPACK);
        }
        {
            float acc[W / 2];
            wg_fence();
#pragma unroll
            for (int k = 0; k < W / 16; ++k) wgmma_rs(acc, h1[k], wg_desc(w2 + k * 256, 128, KCHW * 128), k > 0);
            wgmma_ss(acc, d_ones, wg_desc(b2, 128, 256), 1);
            wg_commit();
            wg_wait<0>();
            wg_fence_acc(acc);
            mark(K4_PH_L_L2);
#pragma unroll
            for (int nc = 0; nc < NC; ++nc) mlp_repack<ACT>(*reinterpret_cast<const float (*)[32]>(acc + 32 * nc), h2 + 4 * nc, act_c);
            mark(K4_PH_L_REPACK);
        }
        // W3 / B3 hold output channel c in column 2c (k4_scene_create), so channel c of rows g / g+8 is o[0] / o[2] of lane
        // t = c: three lanes of each quad share the epilogue.  Columns 0..7 of the 16-row tiles are all there is, so L3
        // runs at N = 8.
        float o[4];
        wg_fence();
#pragma unroll
        for (int k = 0; k < W / 16; ++k) wgmma_rs(o, h2[k], wg_desc(w3 + k * 256, 128, KCHW * 128), k > 0);
        wgmma_ss(o, d_ones, wg_desc(b3, 128, 256), 1);
        wg_commit();
        pend = mlp_epi_inputs<DIRECT>(mh * 64 + warp * 16 + g, valid, slot0, qw, qowner, qdiff, t);
        wg_wait<0>();
        wg_fence_acc(o);
        mlp_epi_logits<DIRECT>(pend, o);
        mark(K4_PH_L_L3);
        if (mh + 1 < halves) {
            mlp_epilogue(pend, racc, t);
            mark(K4_PH_L_EPILOGUE);
        }
    }
    if (!colour_first) consumed();
    if (halves > 0) {
        mlp_epilogue(pend, racc, t);
        mark(K4_PH_L_EPILOGUE);
    }
    if (colour_first) consumed();
}
