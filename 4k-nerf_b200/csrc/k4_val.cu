// k4_val.cu -- the two pieces of run_sr.py's joint-stage validation (run_sr.py:1131-1138) that had no device form:
//
//   k4_op_resize_quarter  cv2.resize(img, None, fx=1/4, fy=1/4) of an fp32 [H, W, 3] frame (INTER_LINEAR), the
//                         frames LPIPS scores when load_sr == 1.  Output h x w = cvRound(H / 4) x cvRound(W / 4).
//                         Per axis of n source pixels, output k reads the pair (4k+1, 4k+2) with t = 0.5; when
//                         4k + 3 > n the pair is (n-2, n-1) with t = 1.  One value is lerp(a, b, t) = a + (b - a) t,
//                         each operation rounded once; columns first, then rows.  When H or W is 3 (a one-pixel output
//                         axis) cv2 takes another path: rows first, and a clamped pair reads pixel n-1 alone.
//   k4_op_mse_f32         np.mean(np.square(a - b)) of two float32 [H, W, 3] frames, bit for bit: the difference and
//                         the square in fp32, the sum in numpy's pairwise order (pairwise_sum, loops_utils.h) over the
//                         elements in the order numpy visits them, and numpy's float32(float64(sum) / n).
//
// numpy's pairwise sum of n values: a block of at most 128 values uses 8 running accumulators combined as
// ((r0+r1)+(r2+r3))+((r4+r5)+(r6+r7)), then adds the remainder in sequence (fewer than 8 values: in sequence from
// -0.0); a longer range splits at n2 = n/2 rounded down to a multiple of 8.  The tree depends on n only.  Let U be the
// first depth holding a leaf: every node above it is split, so the nodes at depth U are 2^U "units" in a perfect
// binary tree, and each unit's own subtree is at most two levels deep (checked on the host).
//   mse_unit_kernel   one thread per unit: its range by descending U levels, its subtree's sum, then the CTA's units
//                     combined as the perfect tree's lower levels in shared memory.
//   mse_tree_kernel   one CTA per 256 consecutive partial sums: the next 8 levels of the perfect tree; the last CTA
//                     of the last pass adds the sum to numpy's initial 0 and divides.
// No atomics, no host synchronisation: the result is bitwise reproducible.
#include "k4_internal.cuh"

namespace {

// ---- resize ----------------------------------------------------------------------------------------------------
constexpr int RZ_NT = 256;

__device__ __forceinline__ float rz_lerp(float a, float b, float t) { return __fadd_rn(a, __fmul_rn(__fsub_rn(b, a), t)); }

// source pair and weight of output k along an axis of n pixels; clamp_last: cv2's own path (pixel n-1 alone)
__device__ __forceinline__ void rz_axis(long long k, long long n, bool clamp_last, long long& i0, long long& i1, float& t) {
    if (4 * k + 3 <= n) { i0 = 4 * k + 1; i1 = i0 + 1; t = 0.5f; }
    else if (clamp_last) { i0 = i1 = n - 1; t = 0.0f; }
    else { i0 = n - 2; i1 = n - 1; t = 1.0f; }
}

__global__ void __launch_bounds__(RZ_NT) resize_quarter_kernel(const float* __restrict__ src, long long H, long long W,
                                                               long long sy, long long sx, long long sc, long long h,
                                                               long long w, float* __restrict__ dst) {
    const long long i = (long long)blockIdx.x * RZ_NT + threadIdx.x;
    if (i >= h * w * 3) return;
    const int c = (int)(i % 3);
    const long long p = i / 3, oy = p / w, ox = p - oy * w;
    const bool rows_first = H == 3 || W == 3;
    long long y0, y1, x0, x1;
    float ty, tx;
    rz_axis(oy, H, rows_first, y0, y1, ty);
    rz_axis(ox, W, rows_first, x0, x1, tx);
    const float* s = src + c * sc;
    const float a00 = __ldg(s + y0 * sy + x0 * sx), a01 = __ldg(s + y0 * sy + x1 * sx);
    const float a10 = __ldg(s + y1 * sy + x0 * sx), a11 = __ldg(s + y1 * sy + x1 * sx);
    float v;
    if (rows_first) {
        const float c0 = ty == 0.0f ? a00 : rz_lerp(a00, a10, ty), c1 = ty == 0.0f ? a01 : rz_lerp(a01, a11, ty);
        v = tx == 0.0f ? c0 : rz_lerp(c0, c1, tx);
    } else {
        v = rz_lerp(rz_lerp(a00, a01, tx), rz_lerp(a10, a11, tx), ty);
    }
    dst[i] = v;
}

long long rz_out(long long n) {          // cvRound(n * 0.25): round half to even
    const long long q = n >> 2, r = n & 3;
    return q + (r == 3 || (r == 2 && (q & 1)));
}

// ---- MSE -------------------------------------------------------------------------------------------------------
constexpr int MSE_NT = 256, MSE_LOG_NT = 8;
constexpr int MSE_MAX_DEPTH_BELOW = 2;

struct MseArgs {
    const float* a;
    const float* b;
    long long n[3];                     // extents in visiting order, outermost first
    long long sa[3], sb[3];             // element strides in that order
    long long total;
    int U;
};

long long pw_split(long long s) { const long long h = s / 2; return h - h % 8; }

// U (depth of the first leaf) and the depth of the deepest unit subtree, from the distinct node sizes per level
bool pw_plan(long long n, int& U, int& below) {
    long long cur[64], nxt[64];
    int m = 1;
    cur[0] = n;
    U = 0;
    below = -1;
    for (int depth = 0; m > 0; ++depth) {
        bool any_leaf = false;
        int k = 0;
        for (int i = 0; i < m; ++i) {
            if (cur[i] <= 128) { any_leaf = true; continue; }
            const long long h = pw_split(cur[i]);
            for (long long c : {h, cur[i] - h}) {
                bool seen = false;
                for (int j = 0; j < k; ++j) seen |= nxt[j] == c;
                if (!seen) { if (k == 64) return false; nxt[k++] = c; }
            }
        }
        if (any_leaf && below < 0) { U = depth; below = 0; }
        else if (below >= 0) ++below;
        m = k;
        for (int i = 0; i < m; ++i) cur[i] = nxt[i];
    }
    return below <= MSE_MAX_DEPTH_BELOW;
}

// the elements from sequence position k on, as squared fp32 differences
struct MseWalk {
    long long c1, c2, oa, ob;
    __device__ MseWalk(const MseArgs& q, long long k) {
        c2 = k % q.n[2];
        const long long r = k / q.n[2];
        c1 = r % q.n[1];
        const long long c0 = r / q.n[1];
        oa = c0 * q.sa[0] + c1 * q.sa[1] + c2 * q.sa[2];
        ob = c0 * q.sb[0] + c1 * q.sb[1] + c2 * q.sb[2];
    }
    __device__ __forceinline__ float next(const MseArgs& q) {
        const float d = __fsub_rn(__ldg(q.a + oa), __ldg(q.b + ob));
        oa += q.sa[2];
        ob += q.sb[2];
        if (++c2 == q.n[2]) {
            c2 = 0;
            oa += q.sa[1] - q.n[2] * q.sa[2];
            ob += q.sb[1] - q.n[2] * q.sb[2];
            if (++c1 == q.n[1]) {
                c1 = 0;
                oa += q.sa[0] - q.n[1] * q.sa[1];
                ob += q.sb[0] - q.n[1] * q.sb[1];
            }
        }
        return __fmul_rn(d, d);
    }
};

// numpy's pairwise_sum of a leaf (at most 128 values)
__device__ __noinline__ float pw_leaf(const MseArgs& q, long long lo, int s) {
    MseWalk w(q, lo);
    if (s < 8) {
        float r = -0.0f;
        for (int i = 0; i < s; ++i) r = __fadd_rn(r, w.next(q));
        return r;
    }
    float r[8];
#pragma unroll
    for (int j = 0; j < 8; ++j) r[j] = w.next(q);
    int i = 8;
    for (; i < s - s % 8; i += 8)
#pragma unroll
        for (int j = 0; j < 8; ++j) r[j] = __fadd_rn(r[j], w.next(q));
    float res = __fadd_rn(__fadd_rn(__fadd_rn(r[0], r[1]), __fadd_rn(r[2], r[3])),
                          __fadd_rn(__fadd_rn(r[4], r[5]), __fadd_rn(r[6], r[7])));
    for (; i < s; ++i) res = __fadd_rn(res, w.next(q));
    return res;
}

template <int D>
__device__ float pw_node(const MseArgs& q, long long lo, long long s) {
    if constexpr (D == 0) {
        return pw_leaf(q, lo, (int)s);                   // pw_plan bounds the depth: s <= 128 here
    } else {
        if (s <= 128) return pw_leaf(q, lo, (int)s);
        const long long h = s / 2 - (s / 2) % 8;
        return __fadd_rn(pw_node<D - 1>(q, lo, h), pw_node<D - 1>(q, lo + h, s - h));
    }
}

__device__ __forceinline__ float mse_final(float sum, long long n) {
    return __double2float_rn(__ddiv_rn((double)__fadd_rn(0.0f, sum), (double)n));
}

// levels of the perfect tree over v[0, m): v[i] = v[2i] + v[2i+1] until one value is left
__device__ float tree_reduce(float* v, int m) {
    for (; m > 1; m >>= 1) {
        float t = 0.0f;
        if ((int)threadIdx.x < m / 2) t = __fadd_rn(v[2 * threadIdx.x], v[2 * threadIdx.x + 1]);
        __syncthreads();
        if ((int)threadIdx.x < m / 2) v[threadIdx.x] = t;
        __syncthreads();
    }
    return v[0];
}

__global__ void __launch_bounds__(MSE_NT) mse_unit_kernel(const __grid_constant__ MseArgs q, int log_per_cta, float* out,
                                                          float* d_mse) {
    __shared__ float v[MSE_NT];
    const long long j = ((long long)blockIdx.x << log_per_cta) + threadIdx.x;
    long long lo = 0, s = q.total;
    for (int l = q.U - 1; l >= 0; --l) {
        const long long h = s / 2 - (s / 2) % 8;
        if ((j >> l) & 1) { lo += h; s -= h; } else { s = h; }
    }
    v[threadIdx.x] = pw_node<MSE_MAX_DEPTH_BELOW>(q, lo, s);
    __syncthreads();
    const float r = tree_reduce(v, 1 << log_per_cta);
    if (threadIdx.x == 0) {
        if (d_mse) *d_mse = mse_final(r, q.total);
        else out[blockIdx.x] = r;
    }
}

__global__ void __launch_bounds__(MSE_NT) mse_tree_kernel(const float* __restrict__ in, int log_per_cta, float* out,
                                                          long long total, float* d_mse) {
    __shared__ float v[MSE_NT];
    v[threadIdx.x] = in[((long long)blockIdx.x << log_per_cta) + threadIdx.x];
    __syncthreads();
    const float r = tree_reduce(v, 1 << log_per_cta);
    if (threadIdx.x == 0) {
        if (d_mse) *d_mse = mse_final(r, total);
        else out[blockIdx.x] = r;
    }
}

bool strides_ok(const int64_t* s) { return s[0] >= 0 && s[1] >= 0 && s[2] >= 0; }
bool size_ok(int64_t H, int64_t W, int64_t lo) { return H >= lo && W >= lo && H <= 65535 && W <= 65535; }

// partial sums after the unit kernel: 2^(U-8) floats, then 2^(U-16), ... (two ping-pong buffers)
size_t mse_ws_floats(int U) { return U > MSE_LOG_NT ? (size_t)2 << (U - MSE_LOG_NT) : 0; }

}  // namespace

extern "C" {

int k4_op_resize_quarter(const float* d_src, int64_t H, int64_t W, const int64_t strides[3], float* d_dst,
                         k4_stream_t stream) {
    if (!d_src || !d_dst || !strides || !size_ok(H, W, 3) || !strides_ok(strides)) return K4_ERR_INVALID_ARG;
    if ((uintptr_t)d_src % sizeof(float) || (uintptr_t)d_dst % sizeof(float)) return K4_ERR_INVALID_ARG;
    const long long h = rz_out(H), w = rz_out(W), total = h * w * 3;
    resize_quarter_kernel<<<(unsigned)((total + RZ_NT - 1) / RZ_NT), RZ_NT, 0, (cudaStream_t)stream>>>(
        d_src, H, W, strides[0], strides[1], strides[2], h, w, d_dst);
    const cudaError_t e = cudaGetLastError();
    if (e != cudaSuccess) { k4_set_cuda_error(e, "k4_op_resize_quarter launch"); return K4_ERR_CUDA; }
    return K4_OK;
}

size_t k4_op_mse_f32_workspace_bytes(int64_t H, int64_t W) {
    int U, below;
    if (!size_ok(H, W, 1) || !pw_plan(3 * H * W, U, below)) return 0;
    return sizeof(float) * (mse_ws_floats(U) + 1);
}

int k4_op_mse_f32(const float* d_a, const float* d_b, int64_t H, int64_t W, const int64_t strides_a[3],
                  const int64_t strides_b[3], const int32_t order[3], float* d_mse, void* d_workspace,
                  size_t workspace_bytes, k4_stream_t stream) {
    if (!d_a || !d_b || !strides_a || !strides_b || !order || !d_mse || !d_workspace) return K4_ERR_INVALID_ARG;
    if (!size_ok(H, W, 1) || !strides_ok(strides_a) || !strides_ok(strides_b)) return K4_ERR_INVALID_ARG;
    for (int i = 0; i < 3; ++i)
        if (order[i] < 0 || order[i] > 2) return K4_ERR_INVALID_ARG;
    if ((1 << order[0] | 1 << order[1] | 1 << order[2]) != 7) return K4_ERR_INVALID_ARG;
    if ((uintptr_t)d_a % sizeof(float) || (uintptr_t)d_b % sizeof(float) || (uintptr_t)d_mse % sizeof(float) ||
        (uintptr_t)d_workspace % sizeof(float))
        return K4_ERR_INVALID_ARG;
    const size_t need = k4_op_mse_f32_workspace_bytes(H, W);
    if (need == 0) return K4_ERR_UNSUPPORTED;
    if (workspace_bytes < need) return K4_ERR_WORKSPACE;
    MseArgs q{};
    q.a = d_a;
    q.b = d_b;
    const long long ext[3] = {H, W, 3};
    for (int i = 0; i < 3; ++i) {
        q.n[i] = ext[order[i]];
        q.sa[i] = strides_a[order[i]];
        q.sb[i] = strides_b[order[i]];
    }
    q.total = 3 * H * W;
    int below;
    pw_plan(q.total, q.U, below);
    cudaStream_t s = (cudaStream_t)stream;
    float* buf[2] = {(float*)d_workspace, (float*)d_workspace + (mse_ws_floats(q.U) / 2)};
    int level = q.U;                                            // log2 of the values left to combine
    int lg = level < MSE_LOG_NT ? level : MSE_LOG_NT;
    level -= lg;
    mse_unit_kernel<<<1u << level, 1 << lg, 0, s>>>(q, lg, buf[0], level == 0 ? d_mse : nullptr);
    for (int p = 0; level > 0; ++p) {
        lg = level < MSE_LOG_NT ? level : MSE_LOG_NT;
        level -= lg;
        mse_tree_kernel<<<1u << level, 1 << lg, 0, s>>>(buf[p & 1], lg, buf[(p + 1) & 1], q.total,
                                                         level == 0 ? d_mse : nullptr);
    }
    const cudaError_t e = cudaGetLastError();
    if (e != cudaSuccess) { k4_set_cuda_error(e, "k4_op_mse_f32 launch"); return K4_ERR_CUDA; }
    return K4_OK;
}

}  // extern "C"
