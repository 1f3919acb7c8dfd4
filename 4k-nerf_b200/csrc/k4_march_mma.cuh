// k4_march_mma.cuh -- warp-level tensor-core evaluation of rgbnet inside the fused marcher.
//
// Replaces the reference's three cuBLAS GEMMs + ReLU/sigmoid kernels + segment_coo for the colour
// head (lib/dvgo.py:116-124,407-419): activations never leave the SM.
//
// Each warp owns a 64-row ring of fp16 feature rows in shared memory.  Lanes whose sample survived
// the alpha / weight thresholds append one row (ballot + popc slot assignment); whenever 32 rows
// are pending the warp runs the whole MLP for them with mma.sync.m16n8k16 (fp16 operands, fp32
// accumulate):  layer-1 accumulators are activated and re-packed IN REGISTERS as the A fragments of
// layer 2 (the C-fragment layout of two n8 tiles is exactly one k16 A fragment), layer-2 output is
// consumed 16 columns at a time by layer 3, so no activation ever touches shared memory.  Weights
// ([n][k] fp16, k contiguous, +16 B row padding => conflict-free ldmatrix) are staged once per CTA
// with a TMA bulk copy (cp.async.bulk + mbarrier).  Results are weighted and accumulated into the
// owning ray's RGB accumulator with shared-memory float atomics.
//
// K4_MLP_F16   : one pass, operands rounded to fp16 (10-bit mantissa, same as TF32).
// K4_MLP_F16X3 : error-compensated split x = hi + lo for activations AND weights, three MMAs per
//                product (hi*hi + lo*hi + hi*lo), ~2^-21 relative error, i.e. fp32-class results.
#pragma once
#include "k4_internal.cuh"
#include "k4_march_common.cuh"
#include "k4_ptx.cuh"

#ifndef K4_MARCH_THREADS
#define K4_MARCH_THREADS 256
#endif
#define K4_MARCH_WARPS (K4_MARCH_THREADS / 32)

namespace {

// Host+device description of the shared-memory weight pack (built by k4_scene.cu, one contiguous
// blob per precision part so that a single bulk copy stages it).
struct MlpPackLayout {
    int kstride[3];    // halves per row (kpad + 8)
    int npad[3];
    int off_w[3];      // byte offsets of each layer's [npad][kstride] fp16 block inside a part
    int part_bytes;    // bytes of one part (hi or lo), multiple of 16
    int off_bias[3];   // float offsets inside the bias block
    int bias_floats;
};

__host__ __device__ inline MlpPackLayout mlp_pack_layout(const K4Dev& s) {
    MlpPackLayout L;
    int off = 0;
    for (int l = 0; l < 3; ++l) {
        L.kstride[l] = s.kpad[l] + 8;
        L.npad[l] = s.npad[l];
        L.off_w[l] = off;
        off += L.npad[l] * L.kstride[l] * 2;
    }
    L.part_bytes = (off + 15) & ~15;
    int bo = 0;
    for (int l = 0; l < 3; ++l) { L.off_bias[l] = bo; bo += L.npad[l]; }
    L.bias_floats = bo;
    return L;
}

// ACT: the hidden activation (K4_ACT_*, RgbAct in k4_march_common.cuh), applied to the fp32 accumulators before they
// are rounded (F16) or split (F16X3) into the next layer's fp16 A fragments.
template <int MODE, int ACT = K4_ACT_RELU>
struct MmaWarpCtx {
    static constexpr bool kX3 = (MODE == K4_MLP_F16X3);
    static constexpr int kParts = kX3 ? 2 : 1;
    static constexpr int kRing = 64;

    // shared-memory carve-up (byte offsets)
    int astride;            // halves per A-tile row
    unsigned char* w_part[2];
    const float* bias;
    unsigned char* a_part[2];     // this warp's ring, hi / lo
    float* qw;                    // [64]
    unsigned char* qowner;        // [64]
    float* qdiff;                 // [64][3] (DVGO, !direct)
    float* racc;                  // [32][3]
    MlpPackLayout L;
    int head, count;
    int n_batches;
    int ks1;                      // k16 steps of layer 1

    // The shape is built and this mode's shared memory fits a block (sm_90: 227 KB).  F16X3 holds two weight parts and
    // two rings, which do not fit for width 128 with 49..64 inputs (kpad 64).
    __host__ __device__ static bool supported(const K4Dev& s) {
        return s.depth == 3 && (s.width == 128 || s.width == 64) && s.dim0 <= 64 && s.dim0 > 0 && smem_bytes(s) <= 227 * 1024;
    }

    __host__ __device__ static int a_stride(const K4Dev& s) { return s.kpad[0] + 8; }

    __host__ __device__ static size_t warp_bytes(const K4Dev& s) {
        size_t b = (size_t)kParts * kRing * a_stride(s) * 2;   // A ring(s)
        b += kRing * 4;                                        // qw
        b += kRing;                                            // qowner
        b += kRing * 3 * 4;                                    // qdiff
        b += 32 * 3 * 4;                                       // racc
        return (b + 15) & ~(size_t)15;
    }

    __host__ __device__ static size_t smem_bytes(const K4Dev& s) {
        if (MODE == K4_MLP_FP32) return 0;
        MlpPackLayout L = mlp_pack_layout(s);
        size_t b = 16;                                         // mbarrier
        b += (size_t)kParts * L.part_bytes;
        b += ((size_t)L.bias_floats * 4 + 15) & ~(size_t)15;
        b += (size_t)K4_MARCH_WARPS * warp_bytes(s);
        return b;
    }

    __device__ void init(const K4Dev& s, unsigned char* smem, int warp, int lane) {
        if (MODE == K4_MLP_FP32) return;
        L = mlp_pack_layout(s);
        astride = a_stride(s);
        ks1 = s.kpad[0] >> 4;
        uint64_t* bar = reinterpret_cast<uint64_t*>(smem);
        unsigned char* p = smem + 16;
        for (int q = 0; q < kParts; ++q) { w_part[q] = p; p += L.part_bytes; }
        float* bias_s = reinterpret_cast<float*>(p);
        bias = bias_s;
        p += ((size_t)L.bias_floats * 4 + 15) & ~(size_t)15;
        unsigned char* wb = p + (size_t)warp * warp_bytes(s);
        for (int q = 0; q < kParts; ++q) { a_part[q] = wb; wb += (size_t)kRing * astride * 2; }
        qw = reinterpret_cast<float*>(wb); wb += kRing * 4;
        qdiff = reinterpret_cast<float*>(wb); wb += kRing * 3 * 4;
        racc = reinterpret_cast<float*>(wb); wb += 32 * 3 * 4;
        qowner = wb;
        head = 0; count = 0; n_batches = 0;

        // stage weights with one TMA bulk copy per part; biases with plain loads
        if (threadIdx.x == 0) {
            mbar_init(bar, 1);
            mbar_init_fence();
        }
        __syncthreads();
        if (threadIdx.x == 0) {
            mbar_arrive_expect_tx(bar, (uint32_t)(kParts * L.part_bytes));
            bulk_g2s(w_part[0], s.wh[0], (uint32_t)L.part_bytes, bar);
            if (kX3) bulk_g2s(w_part[1], s.wl[0], (uint32_t)L.part_bytes, bar);
        }
        for (int i = threadIdx.x; i < L.bias_floats; i += blockDim.x) {
            int l = (i >= L.off_bias[2]) ? 2 : (i >= L.off_bias[1]) ? 1 : 0;
            int j = i - L.off_bias[l];
            bias_s[i] = (j < s.n_out[l]) ? __ldg(s.bias[l] + j) : 0.f;
        }
        // zero this warp's rings and accumulators
        {
            uint32_t* z = reinterpret_cast<uint32_t*>(a_part[0]);
            const int nwords = (int)(warp_bytes(s) / 4);
            for (int i = lane; i < nwords; i += 32) z[i] = 0u;
        }
        mbar_wait(bar, 0);
        __syncthreads();
    }

    __device__ void begin_tile(const K4Dev&, const float*, int, int) {}

    // Append this lane's sample (if any) to the warp's ring; run the MLP when 32 rows are pending.
    template <int KIND, typename CellT>
    __device__ void push(const K4Dev& s, bool shade, float w, const CellT& cell, const float cw[8],
                         const int cidx[8], const float* vemb, int n_vemb, int lane) {
        float k0v[32];
        float x[64];
        if (shade) {
            interp_k0<8>(s, cw, cidx, k0v);
            int n = 0;
            for (int c = s.k0_view_off; c < s.C; ++c) x[n++] = k0v[c];
            if (KIND == K4_KIND_DMPIGO) {
                const float pe[3] = {cell.cz, cell.cy, cell.cx};
                n += embed3(pe, s.spape, x + n);
            }
            for (int c = 0; c < n_vemb; ++c) x[n++] = vemb[c];
            const int kp = s.kpad[0];
            for (; n < kp; ++n) x[n] = 0.f;
        }
        push_row(s, shade, w, x, (KIND == K4_KIND_DVGO && !s.direct) ? k0v : nullptr, lane, lane);
    }

    // Append a row x[0 .. kpad[0]) (model-layout inputs, zero padded) owned by `owner` to the ring, with its diffuse
    // logits diff[0..2] (nullptr: none); run the MLP when 32 rows are pending.  Called by all 32 lanes.
    __device__ __forceinline__ void push_row(const K4Dev& s, bool shade, float w, const float* x, const float* diff,
                                             int owner, int lane) {
        const unsigned bal = __ballot_sync(0xffffffffu, shade);
        if (bal == 0) return;
        if (shade) {
            const int slot = (head + count + __popc(bal & ((1u << lane) - 1))) & (kRing - 1);
            const int kp = s.kpad[0];
            uint32_t* rh = reinterpret_cast<uint32_t*>(a_part[0] + (size_t)slot * astride * 2);
            uint32_t* rl = kX3 ? reinterpret_cast<uint32_t*>(a_part[1] + (size_t)slot * astride * 2) : nullptr;
            for (int j = 0; j < kp; j += 2) {
                if constexpr (kX3) {
                    uint32_t hi, lo;
                    split_h2(x[j], x[j + 1], hi, lo);
                    rh[j >> 1] = hi; rl[j >> 1] = lo;
                } else {
                    rh[j >> 1] = h2_rn(x[j], x[j + 1]);
                }
            }
            qw[slot] = w;
            qowner[slot] = (unsigned char)owner;
            if (diff) {
                qdiff[slot * 3 + 0] = diff[0]; qdiff[slot * 3 + 1] = diff[1]; qdiff[slot * 3 + 2] = diff[2];
            }
        }
        count += __popc(bal);
        __syncwarp();
        if (count >= 32) {
            flush(s, lane, 32);
            head = (head + 32) & (kRing - 1);
            count -= 32;
        }
    }

    __device__ void end_tile(const K4Dev& s, int lane, float& r, float& g, float& b) {
        if (count > 0) {
            flush(s, lane, count);
            head = (head + 32) & (kRing - 1);   // keep the head 32-aligned
            count = 0;
        }
        __syncwarp();
        r = racc[lane * 3 + 0]; g = racc[lane * 3 + 1]; b = racc[lane * 3 + 2];
        racc[lane * 3 + 0] = 0.f; racc[lane * 3 + 1] = 0.f; racc[lane * 3 + 2] = 0.f;
        __syncwarp();
    }

    // One MLP batch: rows [head, head+32) of the ring, the first `valid` of which are real.
    __device__ __noinline__ void flush(const K4Dev& s, int lane, int valid) {
        ++n_batches;
        const int g = lane >> 2, t = lane & 3;
        const int W = s.width;                   // 128 or 64
        const int np_cnt = W >> 4;               // n-pairs (16 columns) per hidden layer
        const float* b1 = bias + L.off_bias[0];
        const float* b2 = bias + L.off_bias[1];
        const float* b3 = bias + L.off_bias[2];
        constexpr int MT = kX3 ? 1 : 2;          // m16 tiles processed per pass

        // ldmatrix lane addressing
        const int a_row = ((lane >> 3) & 1) * 8 + (lane & 7);      // row inside the m16 tile
        const int a_kof = (lane >> 4) * 8;                         // k offset (halves)
        const int b_row = (lane >> 4) * 8 + (lane & 7);            // n inside the 16-column pair
        const int b_kof = ((lane >> 3) & 1) * 8;

        for (int mt0 = 0; mt0 < 2; mt0 += MT) {
            if (mt0 * 16 >= valid) break;
            // ---------------- layer 1 ----------------
            uint32_t h1h[MT][8][4];
            uint32_t h1l[kX3 ? MT : 1][kX3 ? 8 : 1][4];
            {
                uint32_t a1h[MT][4][4];
                uint32_t a1l[kX3 ? MT : 1][kX3 ? 4 : 1][4];
#pragma unroll
                for (int m = 0; m < MT; ++m)
#pragma unroll
                    for (int ks = 0; ks < 4; ++ks) {
                        if (ks < ks1) {
                            const int row = (head + (mt0 + m) * 16 + a_row) & (kRing - 1);
                            const uint32_t off = (uint32_t)((row * astride + ks * 16 + a_kof) * 2);
                            ldsm_x4(smem_u32(a_part[0]) + off, a1h[m][ks][0], a1h[m][ks][1], a1h[m][ks][2], a1h[m][ks][3]);
                            if constexpr (kX3) ldsm_x4(smem_u32(a_part[1]) + off, a1l[m][ks][0], a1l[m][ks][1], a1l[m][ks][2], a1l[m][ks][3]);
                        }
                    }
#pragma unroll
                for (int np = 0; np < 8; ++np) {
                    if (np < np_cnt) {
                        float acc[MT][2][4];
#pragma unroll
                        for (int m = 0; m < MT; ++m)
#pragma unroll
                            for (int nt = 0; nt < 2; ++nt) {
                                const float bb0 = b1[np * 16 + nt * 8 + 2 * t], bb1 = b1[np * 16 + nt * 8 + 2 * t + 1];
                                acc[m][nt][0] = bb0; acc[m][nt][1] = bb1; acc[m][nt][2] = bb0; acc[m][nt][3] = bb1;
                            }
#pragma unroll
                        for (int ks = 0; ks < 4; ++ks) {
                            if (ks < ks1) {
                                const uint32_t off = (uint32_t)(L.off_w[0] + ((np * 16 + b_row) * L.kstride[0] + ks * 16 + b_kof) * 2);
                                uint32_t bh[4];
                                ldsm_x4(smem_u32(w_part[0]) + off, bh[0], bh[1], bh[2], bh[3]);
#pragma unroll
                                for (int m = 0; m < MT; ++m) {
                                    mma_16816(acc[m][0], a1h[m][ks], bh[0], bh[1]);
                                    mma_16816(acc[m][1], a1h[m][ks], bh[2], bh[3]);
                                }
                                if constexpr (kX3) {
                                    uint32_t bl[4];
                                    ldsm_x4(smem_u32(w_part[1]) + off, bl[0], bl[1], bl[2], bl[3]);
#pragma unroll
                                    for (int m = 0; m < MT; ++m) {
                                        mma_16816(acc[m][0], a1l[m][ks], bh[0], bh[1]);
                                        mma_16816(acc[m][1], a1l[m][ks], bh[2], bh[3]);
                                        mma_16816(acc[m][0], a1h[m][ks], bl[0], bl[1]);
                                        mma_16816(acc[m][1], a1h[m][ks], bl[2], bl[3]);
                                    }
                                }
                            }
                        }
#pragma unroll
                        for (int m = 0; m < MT; ++m) {
                            float v[8];
#pragma unroll
                            for (int q = 0; q < 4; ++q) { v[q] = RgbAct<ACT>::tc(acc[m][0][q], s.act_c); v[4 + q] = RgbAct<ACT>::tc(acc[m][1][q], s.act_c); }
                            if constexpr (kX3) {
                                split_h2(v[0], v[1], h1h[m][np][0], h1l[m][np][0]);
                                split_h2(v[2], v[3], h1h[m][np][1], h1l[m][np][1]);
                                split_h2(v[4], v[5], h1h[m][np][2], h1l[m][np][2]);
                                split_h2(v[6], v[7], h1h[m][np][3], h1l[m][np][3]);
                            } else {
                                h1h[m][np][0] = h2_rn(v[0], v[1]);
                                h1h[m][np][1] = h2_rn(v[2], v[3]);
                                h1h[m][np][2] = h2_rn(v[4], v[5]);
                                h1h[m][np][3] = h2_rn(v[6], v[7]);
                            }
                        }
                    }
                }
            }
            // ---------------- layers 2 + 3 ----------------
            float acc3[MT][4];
#pragma unroll
            for (int m = 0; m < MT; ++m) {
                const float bb0 = b3[2 * t], bb1 = b3[2 * t + 1];
                acc3[m][0] = bb0; acc3[m][1] = bb1; acc3[m][2] = bb0; acc3[m][3] = bb1;
            }
#pragma unroll
            for (int np = 0; np < 8; ++np) {
                if (np < np_cnt) {
                    float acc[MT][2][4];
#pragma unroll
                    for (int m = 0; m < MT; ++m)
#pragma unroll
                        for (int nt = 0; nt < 2; ++nt) {
                            const float bb0 = b2[np * 16 + nt * 8 + 2 * t], bb1 = b2[np * 16 + nt * 8 + 2 * t + 1];
                            acc[m][nt][0] = bb0; acc[m][nt][1] = bb1; acc[m][nt][2] = bb0; acc[m][nt][3] = bb1;
                        }
#pragma unroll
                    for (int ks = 0; ks < 8; ++ks) {
                        if (ks < np_cnt) {
                            const uint32_t off = (uint32_t)(L.off_w[1] + ((np * 16 + b_row) * L.kstride[1] + ks * 16 + b_kof) * 2);
                            uint32_t bh[4];
                            ldsm_x4(smem_u32(w_part[0]) + off, bh[0], bh[1], bh[2], bh[3]);
#pragma unroll
                            for (int m = 0; m < MT; ++m) {
                                mma_16816(acc[m][0], h1h[m][ks], bh[0], bh[1]);
                                mma_16816(acc[m][1], h1h[m][ks], bh[2], bh[3]);
                            }
                            if constexpr (kX3) {
                                uint32_t bl[4];
                                ldsm_x4(smem_u32(w_part[1]) + off, bl[0], bl[1], bl[2], bl[3]);
#pragma unroll
                                for (int m = 0; m < MT; ++m) {
                                    mma_16816(acc[m][0], h1l[m][ks], bh[0], bh[1]);
                                    mma_16816(acc[m][1], h1l[m][ks], bh[2], bh[3]);
                                    mma_16816(acc[m][0], h1h[m][ks], bl[0], bl[1]);
                                    mma_16816(acc[m][1], h1h[m][ks], bl[2], bl[3]);
                                }
                            }
                        }
                    }
                    // activation, repack as the k16 A fragment `np` of layer 3, and consume it at once
                    const uint32_t off3 = (uint32_t)(L.off_w[2] + (((lane & 7)) * L.kstride[2] + np * 16 + ((lane >> 3) & 1) * 8) * 2);
                    uint32_t b3h[2], b3l[2];
                    ldsm_x2(smem_u32(w_part[0]) + off3, b3h[0], b3h[1]);
                    if constexpr (kX3) ldsm_x2(smem_u32(w_part[1]) + off3, b3l[0], b3l[1]);
#pragma unroll
                    for (int m = 0; m < MT; ++m) {
                        float v[8];
#pragma unroll
                        for (int q = 0; q < 4; ++q) { v[q] = RgbAct<ACT>::tc(acc[m][0][q], s.act_c); v[4 + q] = RgbAct<ACT>::tc(acc[m][1][q], s.act_c); }
                        uint32_t ah[4], al[4];
                        if constexpr (kX3) {
                            split_h2(v[0], v[1], ah[0], al[0]); split_h2(v[2], v[3], ah[1], al[1]);
                            split_h2(v[4], v[5], ah[2], al[2]); split_h2(v[6], v[7], ah[3], al[3]);
                        } else {
                            ah[0] = h2_rn(v[0], v[1]); ah[1] = h2_rn(v[2], v[3]);
                            ah[2] = h2_rn(v[4], v[5]); ah[3] = h2_rn(v[6], v[7]);
                        }
                        mma_16816(acc3[m], ah, b3h[0], b3h[1]);
                        if constexpr (kX3) {
                            mma_16816(acc3[m], al, b3h[0], b3h[1]);
                            mma_16816(acc3[m], ah, b3l[0], b3l[1]);
                        }
                    }
                }
            }
            // ---------------- epilogue: sigmoid, weight, accumulate into the owning ray ----------------
#pragma unroll
            for (int m = 0; m < MT; ++m) {
#pragma unroll
                for (int hh = 0; hh < 2; ++hh) {
                    const int rrow = (mt0 + m) * 16 + hh * 8 + g;        // row inside the batch
                    if (rrow < valid && t < 2) {
                        const int slot = (head + rrow) & (kRing - 1);
                        const float wq = qw[slot];
                        const int owner = qowner[slot];
                        float l0 = acc3[m][hh * 2 + 0], l1 = acc3[m][hh * 2 + 1];
                        if (s.kind == K4_KIND_DVGO && !s.direct) {
                            l0 += qdiff[slot * 3 + 2 * t];
                            if (t == 0) l1 += qdiff[slot * 3 + 1];
                        }
                        const float r0 = __fdiv_rn(1.f, 1.f + expf(-l0));
                        atomicAdd(racc + owner * 3 + 2 * t, wq * r0);
                        if (t == 0) {
                            const float r1 = __fdiv_rn(1.f, 1.f + expf(-l1));
                            atomicAdd(racc + owner * 3 + 1, wq * r1);
                        }
                    }
                }
            }
        }
        __syncwarp();
    }
};

// fp32 mode: the context is an empty shell.
template <int ACT>
struct MmaWarpCtx<K4_MLP_FP32, ACT> {
    int n_batches;
    __host__ __device__ static bool supported(const K4Dev&) { return true; }
    __host__ __device__ static size_t smem_bytes(const K4Dev&) { return 0; }
    __device__ void init(const K4Dev&, unsigned char*, int, int) { n_batches = 0; }
    __device__ void begin_tile(const K4Dev&, const float*, int, int) {}
    template <int KIND, typename CellT>
    __device__ void push(const K4Dev&, bool, float, const CellT&, const float*, const int*, const float*, int, int) {}
    __device__ void end_tile(const K4Dev&, int, float&, float&, float&) {}
};

}  // namespace
