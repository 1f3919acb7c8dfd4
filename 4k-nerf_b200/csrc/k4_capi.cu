// k4_capi.cu -- extern "C" surface of libk4nerf.so (include/k4nerf.h): scene creation (repacking a
// reference checkpoint's tensors for the fused kernels), argument marshalling, error plumbing.
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <cmath>
#include <new>

#include "k4_internal.cuh"
#include "k4_march_mma.cuh"
#include "k4_ws_cfgs.h"

// ------------------------------------------------------------------------------------------------
// errors
// ------------------------------------------------------------------------------------------------
static thread_local char g_cuda_err[512] = "";

void k4_set_cuda_error(cudaError_t e, const char* where) {
    snprintf(g_cuda_err, sizeof(g_cuda_err), "%s: %s (%s)", where, cudaGetErrorName(e), cudaGetErrorString(e));
}

extern "C" int k4_abi_version(void) { return K4_ABI_VERSION; }

extern "C" const char* k4_last_cuda_error(void) { return g_cuda_err; }

extern "C" const char* k4_status_string(int status) {
    switch (status) {
        case K4_OK: return "ok";
        case K4_ERR_INVALID_ARG: return "invalid argument";
        case K4_ERR_UNSUPPORTED: return "unsupported configuration";
        case K4_ERR_CUDA: return "CUDA error";
        case K4_ERR_WORKSPACE: return "workspace missing or too small";
        case K4_ERR_NO_DEVICE: return "no sm_90 device";
        default: return "unknown status";
    }
}

extern "C" int k4_device_check(void) {
    int dev = 0, major = 0;
    if (cudaGetDevice(&dev) != cudaSuccess) return K4_ERR_NO_DEVICE;
    if (cudaDeviceGetAttribute(&major, cudaDevAttrComputeCapabilityMajor, dev) != cudaSuccess) return K4_ERR_NO_DEVICE;
    return major == 9 ? K4_OK : K4_ERR_NO_DEVICE;
}

// ------------------------------------------------------------------------------------------------
// repack kernels (run once per scene)
// ------------------------------------------------------------------------------------------------
namespace {

// [C,X,Y,Z] planar -> [X,Y,Z,Cpad] channel last (zero padded)
__global__ void repack_k0_kernel(const float* __restrict__ src, float* __restrict__ dst,
                                 long long nvox, int C, int Cpad) {
    const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= nvox * Cpad) return;
    const long long v = i / Cpad;
    const int c = (int)(i - v * Cpad);
    dst[i] = (c < C) ? src[(long long)c * nvox + v] : 0.f;
}

// W [n_out][n_in] -> W^T [n_in][ldw] fp32 (zero padded), bias -> [ldw]
__global__ void transpose_w_kernel(const float* __restrict__ W, const float* __restrict__ b,
                                   float* __restrict__ WT, float* __restrict__ bp,
                                   int n_out, int n_in, int ldw) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n_in * ldw) {
        const int k = i / ldw, j = i - k * ldw;
        WT[i] = (j < n_out) ? W[(size_t)j * n_in + k] : 0.f;
    }
    if (i < ldw) bp[i] = (i < n_out) ? b[i] : 0.f;
}

// W [n_out][n_in] -> fp16 hi/lo blocks [npad][kstride] (k contiguous, zero padded)
__global__ void pack_w_f16_kernel(const float* __restrict__ W, __half* __restrict__ hi, __half* __restrict__ lo,
                                  int n_out, int n_in, int npad, int kstride) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= npad * kstride) return;
    const int n = i / kstride, k = i - n * kstride;
    float w = (n < n_out && k < n_in) ? W[(size_t)n * n_in + k] : 0.f;
    __half h = __float2half_rn(w);
    hi[i] = h;
    lo[i] = __float2half_rn(w - __half2float(h));
}

// wgmma operand tiles (canonical K-major, no swizzle; see tc_canon_off)
// The destination tile is pre-zeroed; model weight (n, k) lands at column colmap[k] (identity when colmap == nullptr):
// the config's row layout may hold more inputs than the model has (k4_ws_cfgs.h), those columns stay zero.
// output n of the layer goes to operand row n * rstride (the rows between stay as the caller zeroed them)
__global__ void pack_tc_weight_kernel(const float* __restrict__ W, unsigned char* __restrict__ dst,
                                      int n_out, int n_in, int kpad, const int* __restrict__ colmap, int rstride = 1) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n_out * n_in) return;
    const int n = i / n_in, k = i - n * n_in;
    const int kd = colmap ? colmap[k] : k;
    *reinterpret_cast<__half*>(dst + tc_canon_off(n * rstride, kd >> 3, kpad >> 3) + (kd & 7) * 2) = __float2half_rn(W[i]);
}

// ---- empty-space skipping: coarse occupancy of the mask and its Chebyshev distance field ----
__global__ void skip_coarse_kernel(const uint8_t* __restrict__ mask, uint8_t* __restrict__ dist, int mX, int mY, int mZ,
                                   int cX, int cY, int cZ) {
    const int c = blockIdx.x * blockDim.x + threadIdx.x;
    if (c >= cX * cY * cZ) return;
    const int cz = c % cZ, cy = (c / cZ) % cY, cx = c / (cZ * cY);
    bool any = false;
    for (int i = cx * K4_SKIP_B; i < min((cx + 1) * K4_SKIP_B, mX) && !any; ++i)
        for (int j = cy * K4_SKIP_B; j < min((cy + 1) * K4_SKIP_B, mY) && !any; ++j)
            for (int k = cz * K4_SKIP_B; k < min((cz + 1) * K4_SKIP_B, mZ); ++k)
                if (mask[((size_t)i * mY + j) * mZ + k]) { any = true; break; }
    dist[c] = any ? 0 : 255;
}
// pass p: an unset cell with a neighbour (3x3x3) of distance <= p-1 gets distance p.  In place: values written in
// this pass are p, never <= p-1, so the order of the threads does not matter.
__global__ void skip_dilate_kernel(uint8_t* __restrict__ dist, int cX, int cY, int cZ, int p) {
    const int c = blockIdx.x * blockDim.x + threadIdx.x;
    if (c >= cX * cY * cZ) return;
    if (dist[c] != 255) return;
    const int cz = c % cZ, cy = (c / cZ) % cY, cx = c / (cZ * cY);
    for (int i = max(cx - 1, 0); i <= min(cx + 1, cX - 1); ++i)
        for (int j = max(cy - 1, 0); j <= min(cy + 1, cY - 1); ++j)
            for (int k = max(cz - 1, 0); k <= min(cz + 1, cZ - 1); ++k)
                if (dist[((size_t)i * cY + j) * cZ + k] <= p - 1) { dist[c] = (uint8_t)p; return; }
}
__global__ void skip_cap_kernel(uint8_t* __restrict__ dist, int n) {
    const int c = blockIdx.x * blockDim.x + threadIdx.x;
    if (c < n && dist[c] == 255) dist[c] = K4_SKIP_MAXD + 1;
}
// bias tile [npad][16]: col 0 = fp16(b), col 1 = fp16(b - col0); multiplied by the ONES tile (cols 0,1 = 1)
// output j of the layer goes to row j * rstride of the npad-row tile; every other row is zero
__global__ void pack_tc_bias_kernel(const float* __restrict__ b, unsigned char* __restrict__ dst, int n_out, int npad, int rstride = 1) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= npad * 16) return;
    const int n = i / 16, k = i - n * 16;
    float v = 0.f;
    if (n % rstride == 0 && n / rstride < n_out && k < 2) {
        const float bb = b[n / rstride];
        const __half hi = __float2half_rn(bb);
        v = (k == 0) ? __half2float(hi) : (bb - __half2float(hi));
    }
    *reinterpret_cast<__half*>(dst + tc_canon_off(n, k >> 3, 2) + (k & 7) * 2) = __float2half_rn(v);
}
// layer 1's bias inside K (k4_ws_bias_col): W1 tile [npad][kpad] column col = fp16(b), col + 1 = fp16(b - col), the split
// of pack_tc_bias_kernel; the A rows hold 1.0 in both columns
__global__ void pack_tc_bias_col_kernel(const float* __restrict__ b, unsigned char* __restrict__ dst, int n_out, int kpad, int col) {
    const int n = blockIdx.x * blockDim.x + threadIdx.x;
    if (n >= n_out) return;
    const float bb = b[n];
    const __half hi = __float2half_rn(bb);
    __half* p = reinterpret_cast<__half*>(dst + tc_canon_off(n, col >> 3, kpad >> 3) + (col & 7) * 2);
    p[0] = hi;
    p[1] = __float2half_rn(bb - __half2float(hi));
}
__global__ void pack_tc_ones_kernel(unsigned char* __restrict__ dst) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= 128 * 16) return;
    const int n = i / 16, k = i - n * 16;
    *reinterpret_cast<__half*>(dst + tc_canon_off(n, k >> 3, 2) + (k & 7) * 2) = __float2half_rn(k < 2 ? 1.f : 0.f);
}

// get_rays / ndc_rays / get_rays_of_a_view (lib/dvgo.py:516-582), mode='center'
struct RayGenParams {
    float K[9];
    float c2w[12];
    int H, W, ndc, inverse_y, flip_x, flip_y;
    const int* rows;              // optional: image row of every output row (a rank's share of the frame)
    int n_rows;                   // output rows (== H when rows == nullptr)
};

__global__ void make_rays_kernel(const __grid_constant__ RayGenParams p, float* __restrict__ ro,
                                 float* __restrict__ rd, float* __restrict__ vd) {
    const long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (idx >= (long long)p.n_rows * p.W) return;
    const int ly = (int)(idx / p.W), x = (int)(idx - (long long)ly * p.W);
    const int y = p.rows ? __ldg(p.rows + ly) : ly;
    const int xs = p.flip_x ? (p.W - 1 - x) : x;
    const int ys = p.flip_y ? (p.H - 1 - y) : y;
    const float i = __fadd_rn((float)xs, 0.5f), j = __fadd_rn((float)ys, 0.5f);
    float d0 = __fdiv_rn(__fsub_rn(i, p.K[2]), p.K[0]);
    float d1 = __fdiv_rn(__fsub_rn(j, p.K[5]), p.K[4]);
    float d2 = 1.f;
    if (!p.inverse_y) { d1 = -d1; d2 = -1.f; }
    float dv[3];
#pragma unroll
    for (int r = 0; r < 3; ++r) {
        const float p0 = __fmul_rn(d0, p.c2w[4 * r + 0]);
        const float p1 = __fmul_rn(d1, p.c2w[4 * r + 1]);
        const float p2 = __fmul_rn(d2, p.c2w[4 * r + 2]);
        dv[r] = __fadd_rn(__fadd_rn(p0, p1), p2);
    }
    float ov[3] = {p.c2w[3], p.c2w[7], p.c2w[11]};
    const float nrm = __fsqrt_rn(__fadd_rn(__fadd_rn(__fmul_rn(dv[0], dv[0]), __fmul_rn(dv[1], dv[1])), __fmul_rn(dv[2], dv[2])));
    vd[3 * idx + 0] = __fdiv_rn(dv[0], nrm);
    vd[3 * idx + 1] = __fdiv_rn(dv[1], nrm);
    vd[3 * idx + 2] = __fdiv_rn(dv[2], nrm);
    if (p.ndc) {
        // ndc_rays(H, W, focal=K[0][0], near=1., rays_o, rays_d), lib/dvgo.py:557-574
        const float focal = p.K[0], near_ = 1.f;
        const float t = __fdiv_rn(-(__fadd_rn(near_, ov[2])), dv[2]);
        float o[3];
#pragma unroll
        for (int r = 0; r < 3; ++r) o[r] = __fadd_rn(ov[r], __fmul_rn(t, dv[r]));
        // python scalars: -1./(W/(2.*focal)) evaluated in double, then applied to fp32 tensors
        const float cw = (float)(-1.0 / ((double)p.W / (2.0 * (double)focal)));
        const float ch = (float)(-1.0 / ((double)p.H / (2.0 * (double)focal)));
        const float o0 = __fdiv_rn(__fmul_rn(cw, o[0]), o[2]);
        const float o1 = __fdiv_rn(__fmul_rn(ch, o[1]), o[2]);
        const float o2 = __fadd_rn(1.f, __fdiv_rn(__fmul_rn(2.f, near_), o[2]));
        const float q0 = __fsub_rn(__fdiv_rn(dv[0], dv[2]), __fdiv_rn(o[0], o[2]));
        const float q1 = __fsub_rn(__fdiv_rn(dv[1], dv[2]), __fdiv_rn(o[1], o[2]));
        const float n0 = __fmul_rn(cw, q0);
        const float n1 = __fmul_rn(ch, q1);
        const float n2 = __fdiv_rn(__fmul_rn(-2.f, near_), o[2]);
        ro[3 * idx + 0] = o0; ro[3 * idx + 1] = o1; ro[3 * idx + 2] = o2;
        rd[3 * idx + 0] = n0; rd[3 * idx + 1] = n1; rd[3 * idx + 2] = n2;
    } else {
        ro[3 * idx + 0] = ov[0]; ro[3 * idx + 1] = ov[1]; ro[3 * idx + 2] = ov[2];
        rd[3 * idx + 0] = dv[0]; rd[3 * idx + 1] = dv[1]; rd[3 * idx + 2] = dv[2];
    }
}

int scene_alloc(k4_scene* sc, void** p, size_t bytes) {
    if (sc->n_allocs >= 64) return K4_ERR_INVALID_ARG;
    if (bytes == 0) bytes = 16;
    K4_CUDA_TRY(cudaMalloc(p, bytes));
    sc->allocs[sc->n_allocs++] = *p;
    sc->bytes += bytes;
    return K4_OK;
}

inline int round_up(int v, int m) { return (v + m - 1) / m * m; }

}  // namespace

// ------------------------------------------------------------------------------------------------
// scene
// ------------------------------------------------------------------------------------------------
extern "C" int k4_scene_destroy(k4_scene* sc) {
    if (!sc) return K4_OK;
    for (int i = 0; i < sc->n_allocs; ++i) cudaFree(sc->allocs[i]);
    delete sc;
    return K4_OK;
}

extern "C" size_t k4_scene_device_bytes(const k4_scene* sc) { return sc ? sc->bytes : 0; }

extern "C" int k4_scene_best_mlp_mode(const k4_scene* sc) {
    if (!sc) return K4_ERR_INVALID_ARG;
    const K4Dev& v = sc->dev;
    if (v.depth == 0) return K4_MLP_FP32;
    if (k4_ws_supported(v)) return K4_MLP_TCGEN05_WS;
    if (MmaWarpCtx<K4_MLP_F16>::supported(v)) return K4_MLP_F16;
    return K4_MLP_FP32;
}

extern "C" int k4_scene_ws_config(const k4_scene* sc) { return sc ? sc->dev.tc_cfg : -1; }

extern "C" int k4_scene_create(const k4_scene_desc* d, k4_stream_t stream, k4_scene** out) {
    if (!d || !out) return K4_ERR_INVALID_ARG;
    *out = nullptr;
    if (d->kind != K4_KIND_DVGO && d->kind != K4_KIND_DMPIGO && d->kind != K4_KIND_DCVGO) return K4_ERR_INVALID_ARG;
    for (int a = 0; a < 3; ++a)
        if (d->world_size[a] < 2 || d->mask_size[a] < 1) return K4_ERR_INVALID_ARG;
    if (!d->d_density || !d->d_k0 || !d->d_mask) return K4_ERR_INVALID_ARG;
    if (d->k0_dim < 1 || d->k0_dim > 32) return K4_ERR_UNSUPPORTED;
    if (d->rgbnet_depth < 0 || d->rgbnet_depth > K4_MAX_MLP_LAYERS || d->rgbnet_depth == 1) return K4_ERR_INVALID_ARG;
    if (d->kind == K4_KIND_DMPIGO && (!d->d_act_shift_grid || d->mpi_depth < 2)) return K4_ERR_INVALID_ARG;
    if (d->viewbase_pe < 0 || d->viewbase_pe > 10 || d->spatial_pe < 0 || d->spatial_pe > 10) return K4_ERR_UNSUPPORTED;
    // the rgbnet's hidden activation: gauss / lkrelu exist in DirectMPIGO only (lib/dmpigo.py:89-95; DirectVoxGO and
    // DirectContractedVoxGO hard-code ReLU), the Gaussian needs a finite a > 0
    if (d->rgbnet_act != K4_ACT_RELU && d->rgbnet_act != K4_ACT_GAUSS && d->rgbnet_act != K4_ACT_LKRELU) return K4_ERR_INVALID_ARG;
    if (d->rgbnet_act != K4_ACT_RELU && d->kind != K4_KIND_DMPIGO) return K4_ERR_INVALID_ARG;
    if (d->rgbnet_act == K4_ACT_GAUSS && !(std::isfinite(d->rgbnet_act_param) && d->rgbnet_act_param > 0.f)) return K4_ERR_INVALID_ARG;
    const long long nvox = (long long)d->world_size[0] * d->world_size[1] * d->world_size[2];
    if (nvox >= (1ll << 31)) return K4_ERR_UNSUPPORTED;       // 32-bit voxel indices in the kernels
    int st = k4_device_check();
    if (st != K4_OK) return st;

    cudaStream_t s = (cudaStream_t)stream;
    k4_scene* sc = new (std::nothrow) k4_scene();
    if (!sc) return K4_ERR_INVALID_ARG;
    memset(sc, 0, sizeof(*sc));
    cudaGetDevice(&sc->device);
    K4Dev& v = sc->dev;
    v.kind = d->kind;
    v.X = d->world_size[0]; v.Y = d->world_size[1]; v.Z = d->world_size[2];
    v.C = d->k0_dim; v.Cpad = round_up(d->k0_dim, 4);
    // wgmma config this model runs on (k4_ws_cfgs.h): its k0 copy is padded to the config's channel count.
    // K4_WS_CONFIG=<id> (A-B / tests): that entry instead of the first covering one; one that does not cover the model
    // leaves the scene without a wgmma build.
    int want_cfg = -1;
    if (const char* e = getenv("K4_WS_CONFIG")) {      // a value that is not a whole non-negative number: no override
        char* end = nullptr;
        const long id = strtol(e, &end, 10);
        if (end != e && *end == '\0' && id >= 0 && id < 1000) want_cfg = (int)id;
    }
    const K4WsCfg* wcfg = (d->rgbnet_depth > 0)
        ? k4_ws_pick(d->kind, d->k0_dim, d->viewbase_pe, d->kind == K4_KIND_DMPIGO ? d->spatial_pe : 0, d->rgbnet_width,
                     d->kind == K4_KIND_DVGO ? (d->rgbnet_direct != 0) : 1, d->rgbnet_depth, want_cfg)
        : nullptr;
    if (wcfg && round_up(wcfg->C, 4) > v.Cpad) v.Cpad = round_up(wcfg->C, 4);
    v.tc_cfg = -1;
    v.mX = d->mask_size[0]; v.mY = d->mask_size[1]; v.mZ = d->mask_size[2];
    for (int a = 0; a < 3; ++a) {
        v.xyz_min[a] = d->xyz_min[a]; v.xyz_max[a] = d->xyz_max[a];
        v.xyz_len[a] = d->xyz_max[a] - d->xyz_min[a];           // fp32, as torch: (xyz_max - xyz_min)
        v.m_scale[a] = d->xyz2ijk_scale[a]; v.m_shift[a] = d->xyz2ijk_shift[a];
    }
    v.act_shift = d->act_shift; v.voxel_size = d->voxel_size; v.voxel_size_ratio = d->voxel_size_ratio;
    v.thres = d->fast_color_thres;
    v.max_world_size = d->max_world_size; v.mpi_depth = d->mpi_depth;
    v.depth = d->rgbnet_depth; v.width = d->rgbnet_width; v.direct = d->rgbnet_direct;
    v.viewpe = d->viewbase_pe; v.spape = d->spatial_pe;
    for (int a = 0; a < 3; ++a) { v.scene_center[a] = d->scene_center[a]; v.scene_radius[a] = d->scene_radius[a]; }
    v.bg_len = d->bg_len; v.one_plus_bg = (float)(1.0 + (double)d->bg_len); v.world_len = d->world_len;
    if (d->kind == K4_KIND_DCVGO) v.direct = 1;
    sc->act = d->rgbnet_depth > 0 ? d->rgbnet_act : K4_ACT_RELU;
    if (sc->act == K4_ACT_GAUSS) {
        const float a = d->rgbnet_act_param;
        const float aa = a * a;
        v.act_den = 2.f * aa;                                                  // torch: 2*self.a**2, in fp32
        v.act_c = (float)(-1.4426950408889634 / (2.0 * (double)a * (double)a));  // -log2(e) / (2 a^2)
    }

#define K4_TRY(x) do { st = (x); if (st != K4_OK) { k4_scene_destroy(sc); return st; } } while (0)
#define K4_CTRY(x) do { cudaError_t _e = (x); if (_e != cudaSuccess) { k4_set_cuda_error(_e, #x); k4_scene_destroy(sc); return K4_ERR_CUDA; } } while (0)

    float* p_density = nullptr; float* p_k0 = nullptr; uint8_t* p_mask = nullptr; float* p_act = nullptr;
    K4_TRY(scene_alloc(sc, (void**)&p_density, (size_t)nvox * 4));
    K4_CTRY(cudaMemcpyAsync(p_density, d->d_density, (size_t)nvox * 4, cudaMemcpyDeviceToDevice, s));
    K4_TRY(scene_alloc(sc, (void**)&p_k0, (size_t)nvox * v.Cpad * 4));
    {
        const long long n = nvox * v.Cpad;
        repack_k0_kernel<<<(unsigned)((n + 255) / 256), 256, 0, s>>>(d->d_k0, p_k0, nvox, v.C, v.Cpad);
        K4_CTRY(cudaGetLastError());
    }
    const size_t mbytes = (size_t)v.mX * v.mY * v.mZ;
    K4_TRY(scene_alloc(sc, (void**)&p_mask, mbytes));
    K4_CTRY(cudaMemcpyAsync(p_mask, d->d_mask, mbytes, cudaMemcpyDeviceToDevice, s));
    if (d->kind == K4_KIND_DMPIGO) {
        K4_TRY(scene_alloc(sc, (void**)&p_act, (size_t)d->mpi_depth * 4));
        K4_CTRY(cudaMemcpyAsync(p_act, d->d_act_shift_grid, (size_t)d->mpi_depth * 4, cudaMemcpyDeviceToDevice, s));
    }
    v.density = p_density; v.k0cl = p_k0; v.mask = p_mask; v.act_grid = p_act;

    // ---- empty-space skipping: distance field over K4_SKIP_B^3-voxel cells of the occupancy mask ----
    v.skip = nullptr; v.cX = v.cY = v.cZ = 0;
    {
        bool ok = d->kind != K4_KIND_DCVGO && getenv("K4_NO_SKIP") == nullptr;   // contracted sampling carries per-step state
        for (int a = 0; a < 3; ++a) {
            ok = ok && v.m_scale[a] > 0.f;
            v.m_iscale[a] = v.m_scale[a] > 0.f ? 1.f / v.m_scale[a] : 0.f;
        }
        if (ok) {
            v.cX = (v.mX + K4_SKIP_B - 1) / K4_SKIP_B; v.cY = (v.mY + K4_SKIP_B - 1) / K4_SKIP_B; v.cZ = (v.mZ + K4_SKIP_B - 1) / K4_SKIP_B;
            const int nc = v.cX * v.cY * v.cZ;
            uint8_t* p_skip = nullptr;
            K4_TRY(scene_alloc(sc, (void**)&p_skip, (size_t)nc));
            skip_coarse_kernel<<<(nc + 127) / 128, 128, 0, s>>>(p_mask, p_skip, v.mX, v.mY, v.mZ, v.cX, v.cY, v.cZ);
            int maxc = v.cX > v.cY ? v.cX : v.cY; if (v.cZ > maxc) maxc = v.cZ;
            const int passes = maxc < K4_SKIP_MAXD ? maxc : K4_SKIP_MAXD;
            for (int p = 1; p <= passes; ++p) skip_dilate_kernel<<<(nc + 127) / 128, 128, 0, s>>>(p_skip, v.cX, v.cY, v.cZ, p);
            skip_cap_kernel<<<(nc + 127) / 128, 128, 0, s>>>(p_skip, nc);
            K4_CTRY(cudaGetLastError());
            v.skip = p_skip;
        }
    }

    // ---- rgbnet ----
    v.dim0 = 0; v.k0_view_off = 0;
    if (v.depth > 0) {
        int dim0 = 3 + 3 * v.viewpe * 2;
        if (d->kind == K4_KIND_DVGO) {
            v.k0_view_off = v.direct ? 0 : 3;
            dim0 += v.C - v.k0_view_off;                          // lib/dvgo.py:94-101
        } else if (d->kind == K4_KIND_DCVGO) {
            dim0 += v.C;                                          // lib/dcvgo.py:105-106
        } else {
            dim0 += 3 + 3 * v.spape * 2 + v.C;                    // lib/dmpigo.py:85
        }
        v.dim0 = dim0;
        if (dim0 > K4_MAX_DIM0 || v.width > K4_MAX_WIDTH || v.width < 4) { k4_scene_destroy(sc); return K4_ERR_UNSUPPORTED; }
        for (int l = 0; l < v.depth; ++l) {
            if (!d->d_rgbnet_weight[l] || !d->d_rgbnet_bias[l]) { k4_scene_destroy(sc); return K4_ERR_INVALID_ARG; }
            v.n_in[l] = (l == 0) ? dim0 : v.width;
            v.n_out[l] = (l == v.depth - 1) ? 3 : v.width;
            v.ldw[l] = round_up(v.n_out[l], 4);
            float* wt = nullptr; float* bp = nullptr;
            K4_TRY(scene_alloc(sc, (void**)&wt, (size_t)v.n_in[l] * v.ldw[l] * 4));
            K4_TRY(scene_alloc(sc, (void**)&bp, (size_t)v.ldw[l] * 4));
            const int n = v.n_in[l] * v.ldw[l];
            transpose_w_kernel<<<(n + 255) / 256, 256, 0, s>>>(d->d_rgbnet_weight[l], d->d_rgbnet_bias[l], wt, bp,
                                                              v.n_out[l], v.n_in[l], v.ldw[l]);
            K4_CTRY(cudaGetLastError());
            v.wT[l] = wt; v.bias[l] = bp;
        }
        // tensor-core pack (only for the shapes the mma path is built for)
        if (v.depth == 3) {
            v.kpad[0] = round_up(dim0, 16); v.npad[0] = v.width;
            v.kpad[1] = v.width;            v.npad[1] = v.width;
            v.kpad[2] = v.width;            v.npad[2] = 8;
            if (MmaWarpCtx<K4_MLP_F16>::supported(v)) {
                MlpPackLayout L = mlp_pack_layout(v);
                unsigned char* hi = nullptr; unsigned char* lo = nullptr;
                K4_TRY(scene_alloc(sc, (void**)&hi, (size_t)L.part_bytes));
                K4_TRY(scene_alloc(sc, (void**)&lo, (size_t)L.part_bytes));
                K4_CTRY(cudaMemsetAsync(hi, 0, L.part_bytes, s));
                K4_CTRY(cudaMemsetAsync(lo, 0, L.part_bytes, s));
                for (int l = 0; l < 3; ++l) {
                    const int n = L.npad[l] * L.kstride[l];
                    __half* ph = reinterpret_cast<__half*>(hi + L.off_w[l]);
                    __half* pl = reinterpret_cast<__half*>(lo + L.off_w[l]);
                    pack_w_f16_kernel<<<(n + 255) / 256, 256, 0, s>>>(d->d_rgbnet_weight[l], ph, pl, v.n_out[l], v.n_in[l],
                                                                     L.npad[l], L.kstride[l]);
                    K4_CTRY(cudaGetLastError());
                    v.wh[l] = ph; v.wl[l] = pl;
                }
            }
            // wgmma operand blob, packed for the K4_WS_CFG_LIST entry that covers this model (k4_ws_cfgs.h)
            if (wcfg) {
                const K4WsCfg& c = *wcfg;
                const int kpad = k4_ws_kpad(c), w = c.W, nsp = k4_ws_nsp(c);
                // model input column -> row column of the config's layout
                int colmap[K4_MAX_DIM0];
                const int k0_in = v.C - v.k0_view_off;
                int k = 0;
                for (int j = 0; j < k0_in; ++j) colmap[k++] = j;
                if (d->kind == K4_KIND_DMPIGO) {          // [k0, p(3), sin(p f), cos(p f), view emb]  (lib/dmpigo.py:347-351,374)
                    const int pb = c.C;
                    for (int a = 0; a < 3; ++a) colmap[k++] = pb + a;
                    for (int a = 0; a < 3; ++a) for (int q = 0; q < v.spape; ++q) colmap[k++] = pb + 3 + a * c.spe + q;
                    for (int a = 0; a < 3; ++a) for (int q = 0; q < v.spape; ++q) colmap[k++] = pb + 3 + 3 * c.spe + a * c.spe + q;
                }
                for (int a = 0; a < 3; ++a) colmap[k++] = nsp + a;                              // viewdirs
                for (int a = 0; a < 3; ++a) for (int f = 0; f < v.viewpe; ++f) colmap[k++] = nsp + 3 + a * c.vpe + f;
                for (int a = 0; a < 3; ++a) for (int f = 0; f < v.viewpe; ++f) colmap[k++] = nsp + 3 + 3 * c.vpe + a * c.vpe + f;
                if (k != dim0) { k4_scene_destroy(sc); return K4_ERR_INVALID_ARG; }
                int* d_colmap = nullptr;
                K4_TRY(scene_alloc(sc, (void**)&d_colmap, sizeof(int) * K4_MAX_DIM0));
                K4_CTRY(cudaMemcpyAsync(d_colmap, colmap, sizeof(int) * dim0, cudaMemcpyHostToDevice, s));
                const TcBlobLayout BL = tc_blob_layout(kpad, w);
                unsigned char* blob = nullptr;
                K4_TRY(scene_alloc(sc, (void**)&blob, (size_t)BL.total));
                K4_CTRY(cudaMemsetAsync(blob, 0, BL.total, s));
                const int wm = v.width;
                pack_tc_weight_kernel<<<(wm * dim0 + 255) / 256, 256, 0, s>>>(d->d_rgbnet_weight[0], blob + BL.off_w1, wm, dim0, kpad, d_colmap);
                pack_tc_weight_kernel<<<(wm * wm + 255) / 256, 256, 0, s>>>(d->d_rgbnet_weight[1], blob + BL.off_w2, wm, wm, w, nullptr);
                // W3 / B3: output channel c at operand row (accumulator column) 2c, for mlp_batch_wgmma's epilogue
                pack_tc_weight_kernel<<<(3 * wm + 255) / 256, 256, 0, s>>>(d->d_rgbnet_weight[2], blob + BL.off_w3, 3, wm, w, nullptr, 2);
                if (k4_ws_bias_col(c) >= 0)
                    pack_tc_bias_col_kernel<<<(wm + 127) / 128, 128, 0, s>>>(d->d_rgbnet_bias[0], blob + BL.off_w1, wm, kpad, k4_ws_bias_col(c));
                else
                    pack_tc_bias_kernel<<<(w * 16 + 255) / 256, 256, 0, s>>>(d->d_rgbnet_bias[0], blob + BL.off_b1, wm, w);
                pack_tc_bias_kernel<<<(w * 16 + 255) / 256, 256, 0, s>>>(d->d_rgbnet_bias[1], blob + BL.off_b2, wm, w);
                pack_tc_bias_kernel<<<1, 256, 0, s>>>(d->d_rgbnet_bias[2], blob + BL.off_b3, 3, 16, 2);
                pack_tc_ones_kernel<<<8, 256, 0, s>>>(blob + BL.off_ones);
                K4_CTRY(cudaGetLastError());
                v.tc_blob = blob; v.tc_kpad = kpad; v.tc_width = w; v.tc_cfg = c.id; v.tc_colmap = d_colmap;
            }
        }
    }
#undef K4_TRY
#undef K4_CTRY
    *out = sc;
    return K4_OK;
}

// ------------------------------------------------------------------------------------------------
// render
// ------------------------------------------------------------------------------------------------
extern "C" size_t k4_render_workspace_bytes(const k4_scene*, int64_t) { return 256; }

// phases != NULL: the profiled ws marcher of k4_testing_march_phases (room for max_ctas CTAs, count to *n_ctas)
static int render_impl(const k4_scene* sc, const k4_render_args* a,
                       const float* d_rays_o, const float* d_rays_d, const float* d_viewdirs,
                       int64_t n_rays, const k4_render_out* out, const k4_frame_dst* fd,
                       void* d_workspace, size_t workspace_bytes, k4_stream_t stream,
                       unsigned long long* phases = nullptr, int max_ctas = 0, int* n_ctas = nullptr) {
    static const k4_render_out no_out = {nullptr, nullptr, nullptr, nullptr, nullptr, nullptr};
    if (!sc || !a || (!out && !fd)) return K4_ERR_INVALID_ARG;
    if (!out) out = &no_out;
    if (n_rays < 0) return K4_ERR_INVALID_ARG;
    if (n_rays == 0) return K4_OK;
    if (!d_rays_o || !d_rays_d) return K4_ERR_INVALID_ARG;
    if (!fd && (!out->d_rgb_marched || !out->d_alphainv_last)) return K4_ERR_INVALID_ARG;
    if (fd) {
        if (fd->n_dst < 1 || fd->n_dst > K4_MAX_PEERS || fd->world < 1 || fd->rank < 0 || fd->rank >= fd->world ||
            fd->frame_w < 1 || n_rays % fd->frame_w != 0) return K4_ERR_INVALID_ARG;
        for (int i = 0; i < fd->n_dst; ++i) if (!fd->d_frame[i]) return K4_ERR_INVALID_ARG;
        const long long r = n_rays / fd->frame_w - 1;                       // last local row -> its image row must fit
        const long long g = ((r >> 3) * fd->world + fd->rank) * 8 + (r & 7);
        if ((g + 1) * fd->frame_w > fd->n_full) return K4_ERR_INVALID_ARG;
    }
    if (sc->dev.depth > 0 && !d_viewdirs) return K4_ERR_INVALID_ARG;
    if (!d_workspace || workspace_bytes < k4_render_workspace_bytes(sc, n_rays)) return K4_ERR_WORKSPACE;
    if (!(a->stepsize > 0.f)) return K4_ERR_INVALID_ARG;
    if (a->mlp_mode < K4_MLP_FP32 || a->mlp_mode > K4_MLP_TCGEN05_WS) return K4_ERR_INVALID_ARG;
    if (a->image_w > 0 && (long long)a->image_w * a->image_h != n_rays) return K4_ERR_INVALID_ARG;
    cudaStream_t s = (cudaStream_t)stream;
    const K4Dev& v = sc->dev;

    K4RenderParams rp;
    memset(&rp, 0, sizeof(rp));
    rp.near_ = a->near_;
    rp.bg = a->bg;
    rp.render_depth = a->render_depth && (fd || out->d_depth);
    if (v.kind == K4_KIND_DVGO) {
        rp.far_ = 1e9f;                                            // lib/dvgo.py:307
        rp.stepdist = a->stepsize * v.voxel_size;                   // lib/dvgo.py:310 (fp32 product)
        rp.interval = a->stepsize * v.voxel_size_ratio;             // lib/dvgo.py:341 (fp32 product)
        rp.n_samples = (int)((float)(v.max_world_size - 1) / a->stepsize) + 1;   // lib/dvgo.py:311
    } else if (v.kind == K4_KIND_DCVGO) {
        if (!a->d_t_list || a->n_t < 2) return K4_ERR_INVALID_ARG;
        rp.far_ = a->far_;
        rp.stepdist = 0.f;
        rp.interval = a->stepsize * v.voxel_size_ratio;             // lib/dcvgo.py:279 (fp32 product)
        rp.n_samples = a->n_t;                                      // n_max = len(t)
        rp.t_list = a->d_t_list;
        rp.dist_thres = a->dist_thres;
    } else {
        if (!(a->near_ == 0.f && a->far_ == 1.f)) return K4_ERR_INVALID_ARG;      // lib/dmpigo.py:275
        rp.far_ = a->far_;
        rp.stepdist = 0.f;
        rp.interval = (float)((double)a->stepsize * (double)v.voxel_size_ratio);  // lib/dmpigo.py:306
        rp.n_samples = (int)((double)(v.mpi_depth - 1) / (double)a->stepsize) + 1;  // lib/dmpigo.py:278
        if (rp.n_samples < 2) return K4_ERR_INVALID_ARG;
    }
    rp.inv_nsamples = (float)(1.0 / (double)rp.n_samples);          // ATen: a / cpu_scalar == a * (1/b)
    rp.image_w = a->image_w; rp.image_h = a->image_h;
    rp.n_rays = n_rays;
    if (a->image_w > 0) rp.n_tiles = (long long)((a->image_w + 7) / 8) * ((a->image_h + 3) / 4);
    else rp.n_tiles = (n_rays + 31) / 32;
    rp.rays_o = d_rays_o; rp.rays_d = d_rays_d; rp.viewdirs = d_viewdirs;
    rp.rgb = out->d_rgb_marched; rp.depth = rp.render_depth ? out->d_depth : nullptr;
    rp.alphainv = out->d_alphainv_last;
    if (fd) {
        rp.n_dst = fd->n_dst; rp.f_rank = fd->rank; rp.f_world = fd->world; rp.f_w = fd->frame_w; rp.f_nfull = fd->n_full;
        for (int i = 0; i < fd->n_dst; ++i) rp.d_frame[i] = fd->d_frame[i];
    }
    rp.ray_stats = out->d_ray_stats; rp.t_minmax = out->d_t_minmax; rp.counters = out->d_counters;
    rp.tile_counter = reinterpret_cast<unsigned int*>(d_workspace);
    K4_CUDA_TRY(cudaMemsetAsync(d_workspace, 0, 16, s));
    if ((a->mlp_mode == K4_MLP_TCGEN05 || a->mlp_mode == K4_MLP_TCGEN05_WS) && v.depth > 0)   // K4_MLP_TCGEN05: an alias
        return k4_ws_supported(v) ? k4_launch_march_ws(sc, rp, s, phases, max_ctas, n_ctas) : K4_ERR_UNSUPPORTED;
    return k4_launch_march(sc, rp, a->mlp_mode, s);
}

extern "C" int k4_render_rays(const k4_scene* sc, const k4_render_args* a,
                              const float* d_rays_o, const float* d_rays_d, const float* d_viewdirs,
                              int64_t n_rays, const k4_render_out* out,
                              void* d_workspace, size_t workspace_bytes, k4_stream_t stream) {
    if (!out) return K4_ERR_INVALID_ARG;
    return render_impl(sc, a, d_rays_o, d_rays_d, d_viewdirs, n_rays, out, nullptr, d_workspace, workspace_bytes, stream);
}

extern "C" int k4_testing_march_phases(const k4_scene* sc, const k4_render_args* a,
                                       const float* d_rays_o, const float* d_rays_d, const float* d_viewdirs,
                                       int64_t n_rays, const k4_render_out* out, void* d_workspace, size_t workspace_bytes,
                                       uint64_t* d_phases, int32_t max_ctas, int32_t* n_ctas, k4_stream_t stream) {
    if (n_ctas) *n_ctas = 0;
    if (!sc || !a || !out || !d_phases || max_ctas < 1 || n_rays < 1) return K4_ERR_INVALID_ARG;
    if (a->mlp_mode != K4_MLP_TCGEN05_WS) return K4_ERR_INVALID_ARG;
    if (sc->dev.depth == 0) return K4_ERR_UNSUPPORTED;
    int n = 0;
    const int st = render_impl(sc, a, d_rays_o, d_rays_d, d_viewdirs, n_rays, out, nullptr, d_workspace, workspace_bytes, stream,
                               reinterpret_cast<unsigned long long*>(d_phases), max_ctas, &n);
    if (st == K4_OK && n_ctas) *n_ctas = n;
    return st;
}

extern "C" int k4_render_rays_frames(const k4_scene* sc, const k4_render_args* a,
                                     const float* d_rays_o, const float* d_rays_d, const float* d_viewdirs,
                                     int64_t n_rays, const k4_frame_dst* dst, const k4_render_out* out,
                                     void* d_workspace, size_t workspace_bytes, k4_stream_t stream) {
    if (!dst) return K4_ERR_INVALID_ARG;
    return render_impl(sc, a, d_rays_o, d_rays_d, d_viewdirs, n_rays, out, dst, d_workspace, workspace_bytes, stream);
}

// ---- the rgbnet of one MLP mode on caller-supplied rows (test suite) ----
// These kernels live here rather than in k4_march.cu so that the marcher's translation unit, and with it the code of
// the __noinline__ mlp_fp32 / MmaWarpCtx::flush it calls, is unchanged by them.
namespace {

// F16 / F16X3: one warp per group of 32 rows, driven through MmaWarpCtx as k4_march_kernel drives it: push_row of the
// group's rows (a full group flushes there), end_tile (flushes a partial group, hands back the per-lane accumulators).
template <int MODE, int ACT>
__global__ void __launch_bounds__(K4_MARCH_THREADS)
k4_test_rgbnet_mma_kernel(const __grid_constant__ K4Dev s, const float* __restrict__ xs, const float* __restrict__ diffs,
                          const float* __restrict__ ws, const int* __restrict__ owners, long long n, float* __restrict__ racc) {
    extern __shared__ __align__(16) unsigned char smem_raw[];
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    MmaWarpCtx<MODE, ACT> mma;
    mma.init(s, smem_raw, warp, lane);
    const long long n_groups = (n + 31) / 32;
    for (long long g = (long long)blockIdx.x * K4_MARCH_WARPS + warp; g < n_groups; g += (long long)gridDim.x * K4_MARCH_WARPS) {
        const long long r = g * 32 + lane;
        const bool shade = r < n;
        float x[64], d[3] = {0.f, 0.f, 0.f}, w = 0.f;
        int o = 0;
        if (shade) {
            for (int k = 0; k < s.kpad[0]; ++k) x[k] = k < s.dim0 ? xs[r * s.dim0 + k] : 0.f;
            if (diffs) { d[0] = diffs[3 * r]; d[1] = diffs[3 * r + 1]; d[2] = diffs[3 * r + 2]; }
            w = ws[r];
            o = owners[r] & 31;
        }
        mma.push_row(s, shade, w, x, diffs ? d : nullptr, o, lane);
        float cr, cg, cb;
        mma.end_tile(s, lane, cr, cg, cb);
        racc[3 * (g * 32 + lane) + 0] = cr; racc[3 * (g * 32 + lane) + 1] = cg; racc[3 * (g * 32 + lane) + 2] = cb;
    }
}

// FP32: thread (group g, owner j) walks the group's rows in order and accumulates the ones it owns, as k4_march_kernel
// accumulates a ray's samples
template <int ACT>
__global__ void k4_test_rgbnet_fp32_kernel(const __grid_constant__ K4Dev s, const float* __restrict__ xs, const float* __restrict__ diffs,
                                           const float* __restrict__ ws, const int* __restrict__ owners, long long n,
                                           float* __restrict__ racc) {
    const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    const long long g = i >> 5;
    const int j = (int)(i & 31);
    if (g * 32 >= n) return;
    float acc_r = 0.f, acc_g = 0.f, acc_b = 0.f;
    for (long long r = g * 32; r < n && r < g * 32 + 32; ++r) {
        if ((owners[r] & 31) != j) continue;
        float rgb[3];
        mlp_fp32<ACT>(s, xs + r * s.dim0, rgb);
        if (diffs) {
            rgb[0] = __fadd_rn(rgb[0], diffs[3 * r]); rgb[1] = __fadd_rn(rgb[1], diffs[3 * r + 1]);
            rgb[2] = __fadd_rn(rgb[2], diffs[3 * r + 2]);
        }
        rgb[0] = sigmoid_ref(rgb[0]); rgb[1] = sigmoid_ref(rgb[1]); rgb[2] = sigmoid_ref(rgb[2]);
        const float w = ws[r];
        acc_r = __fadd_rn(acc_r, __fmul_rn(w, rgb[0]));
        acc_g = __fadd_rn(acc_g, __fmul_rn(w, rgb[1]));
        acc_b = __fadd_rn(acc_b, __fmul_rn(w, rgb[2]));
    }
    racc[3 * i + 0] = acc_r; racc[3 * i + 1] = acc_g; racc[3 * i + 2] = acc_b;
}

template <int MODE, int ACT>
int launch_test_rgbnet_mma(const K4Dev& v, const k4_rgbnet_test_args* a, cudaStream_t st) {
    auto kern = k4_test_rgbnet_mma_kernel<MODE, ACT>;
    const size_t smem = MmaWarpCtx<MODE>::smem_bytes(v);
    if (smem > 48 * 1024) K4_CUDA_TRY(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    const long long n_groups = (a->n + 31) / 32;
    long long blocks = (n_groups + K4_MARCH_WARPS - 1) / K4_MARCH_WARPS;
    if (blocks > 1024) blocks = 1024;
    kern<<<(unsigned)blocks, K4_MARCH_THREADS, smem, st>>>(v, a->d_x, a->d_diffuse, a->d_w, a->d_owner, a->n, a->d_racc);
    K4_CUDA_TRY(cudaGetLastError());
    return K4_OK;
}

template <int ACT>
int testing_rgbnet_mma(const K4Dev& v, const k4_rgbnet_test_args* a, cudaStream_t st) {
    if (a->mode == K4_MLP_F16) return launch_test_rgbnet_mma<K4_MLP_F16, ACT>(v, a, st);
    if (a->mode == K4_MLP_F16X3) return launch_test_rgbnet_mma<K4_MLP_F16X3, ACT>(v, a, st);
    if (a->mode != K4_MLP_FP32) return K4_ERR_UNSUPPORTED;
    const long long threads = (a->n + 31) / 32 * 32;
    k4_test_rgbnet_fp32_kernel<ACT><<<(unsigned)((threads + 127) / 128), 128, 0, st>>>(v, a->d_x, a->d_diffuse, a->d_w, a->d_owner,
                                                                                      a->n, a->d_racc);
    K4_CUDA_TRY(cudaGetLastError());
    return K4_OK;
}

}  // namespace

extern "C" int k4_testing_ws_row_layout(int32_t config, int32_t* out) {
    int32_t v[4];
    if (!out) return K4_ERR_INVALID_ARG;
    const int st = k4_ws_row_layout(config, v);
    for (int i = 0; i < 4; ++i) out[i] = st == K4_OK ? v[i] : 0;
    return st;
}

extern "C" int k4_testing_rgbnet(const k4_scene* sc, const k4_rgbnet_test_args* a, int32_t* group_rows, k4_stream_t stream) {
    if (group_rows) *group_rows = 0;
    if (!sc || !a) return K4_ERR_INVALID_ARG;
    if (a->mode < K4_MLP_FP32 || a->mode > K4_MLP_TCGEN05_WS) return K4_ERR_INVALID_ARG;
    if (a->n < 1 || a->n > (1ll << 24)) return K4_ERR_INVALID_ARG;
    if (!a->d_x || !a->d_w || !a->d_owner || !a->d_racc) return K4_ERR_INVALID_ARG;
    const K4Dev& v = sc->dev;
    const bool diffuse = v.kind == K4_KIND_DVGO && !v.direct;
    if (diffuse != (a->d_diffuse != nullptr)) return K4_ERR_INVALID_ARG;
    const bool wgmma = a->mode == K4_MLP_TCGEN05 || a->mode == K4_MLP_TCGEN05_WS;
    if (v.depth == 0) return K4_ERR_UNSUPPORTED;
    if (wgmma && !k4_ws_supported(v)) return K4_ERR_UNSUPPORTED;
    if (a->mode == K4_MLP_F16 && !MmaWarpCtx<K4_MLP_F16>::supported(v)) return K4_ERR_UNSUPPORTED;
    if (a->mode == K4_MLP_F16X3 && !MmaWarpCtx<K4_MLP_F16X3>::supported(v)) return K4_ERR_UNSUPPORTED;
    cudaStream_t s = (cudaStream_t)stream;
    int st = wgmma ? k4_testing_rgbnet_ws(sc, a, s)
           : sc->act == K4_ACT_GAUSS ? testing_rgbnet_mma<K4_ACT_GAUSS>(v, a, s)
           : sc->act == K4_ACT_LKRELU ? testing_rgbnet_mma<K4_ACT_LKRELU>(v, a, s)
                                      : testing_rgbnet_mma<K4_ACT_RELU>(v, a, s);
    const cudaError_t e = cudaStreamSynchronize(s);
    if (st == K4_OK && e != cudaSuccess) { k4_set_cuda_error(e, "k4_testing_rgbnet"); st = K4_ERR_CUDA; }
    if (st == K4_OK && group_rows) *group_rows = wgmma ? 128 : 32;
    return st;
}

// ---- the empty-space-skipping field of a scene (test suite) ----
extern "C" int k4_testing_skip_field(const k4_scene* sc, uint8_t* d_out, int64_t n, int32_t cdims[3]) {
    if (cdims) cdims[0] = cdims[1] = cdims[2] = 0;
    if (!sc || !d_out || !cdims || n < 1) return K4_ERR_INVALID_ARG;
    const K4Dev& v = sc->dev;
    if (!v.skip) return K4_ERR_UNSUPPORTED;
    const long long nc = (long long)v.cX * v.cY * v.cZ;
    if (n < nc) return K4_ERR_INVALID_ARG;
    K4_CUDA_TRY(cudaMemcpy(d_out, v.skip, (size_t)nc, cudaMemcpyDeviceToDevice));
    cdims[0] = v.cX; cdims[1] = v.cY; cdims[2] = v.cZ;
    return K4_OK;
}

// ---- device memory shared between the ranks of a node (CUDA IPC; one process per GPU) ----
extern "C" int k4_peer_alloc(size_t bytes, void** d_ptr) {
    if (!d_ptr || bytes == 0) return K4_ERR_INVALID_ARG;
    *d_ptr = nullptr;
    void* p = nullptr;
    K4_CUDA_TRY(cudaMalloc(&p, bytes));
    cudaError_t e = cudaMemset(p, 0, bytes);
    if (e != cudaSuccess) { cudaFree(p); k4_set_cuda_error(e, "cudaMemset(peer buffer)"); return K4_ERR_CUDA; }
    *d_ptr = p;
    return K4_OK;
}
extern "C" int k4_peer_enable_all(void) {
    int dev = 0, n = 0;
    K4_CUDA_TRY(cudaGetDevice(&dev));
    K4_CUDA_TRY(cudaGetDeviceCount(&n));
    for (int d = 0; d < n; ++d) {
        if (d == dev) continue;
        int can = 0;
        if (cudaDeviceCanAccessPeer(&can, dev, d) != cudaSuccess || !can) { cudaGetLastError(); continue; }
        cudaError_t e = cudaDeviceEnablePeerAccess(d, 0);
        if (e != cudaSuccess && e != cudaErrorPeerAccessAlreadyEnabled) { k4_set_cuda_error(e, "cudaDeviceEnablePeerAccess"); cudaGetLastError(); return K4_ERR_CUDA; }
        cudaGetLastError();
    }
    return K4_OK;
}
extern "C" int k4_peer_free(void* d_ptr) {
    if (!d_ptr) return K4_OK;
    K4_CUDA_TRY(cudaFree(d_ptr));
    return K4_OK;
}
extern "C" int k4_peer_export(void* d_ptr, unsigned char handle[64]) {
    static_assert(sizeof(cudaIpcMemHandle_t) == 64, "CUDA IPC handle size");
    if (!d_ptr || !handle) return K4_ERR_INVALID_ARG;
    cudaIpcMemHandle_t h;
    K4_CUDA_TRY(cudaIpcGetMemHandle(&h, d_ptr));
    memcpy(handle, &h, 64);
    return K4_OK;
}
extern "C" int k4_peer_open(const unsigned char handle[64], void** d_ptr) {
    if (!d_ptr || !handle) return K4_ERR_INVALID_ARG;
    *d_ptr = nullptr;
    cudaIpcMemHandle_t h;
    memcpy(&h, handle, 64);
    void* p = nullptr;
    K4_CUDA_TRY(cudaIpcOpenMemHandle(&p, h, cudaIpcMemLazyEnablePeerAccess));
    *d_ptr = p;
    return K4_OK;
}
extern "C" int k4_peer_close(void* d_ptr) {
    if (!d_ptr) return K4_OK;
    K4_CUDA_TRY(cudaIpcCloseMemHandle(d_ptr));
    return K4_OK;
}

extern "C" int k4_make_rays_rows(const float* h_K, const float* h_c2w, int32_t H, int32_t W, int32_t ndc,
                                 int32_t inverse_y, int32_t flip_x, int32_t flip_y, const int32_t* d_rows, int32_t n_rows,
                                 float* d_rays_o, float* d_rays_d, float* d_viewdirs, k4_stream_t stream) {
    if (!h_K || !h_c2w || !d_rays_o || !d_rays_d || !d_viewdirs || H <= 0 || W <= 0 || n_rows < 0) return K4_ERR_INVALID_ARG;
    if (n_rows == 0) return K4_OK;
    RayGenParams p;
    memcpy(p.K, h_K, sizeof(p.K));
    memcpy(p.c2w, h_c2w, sizeof(p.c2w));
    p.H = H; p.W = W; p.ndc = ndc; p.inverse_y = inverse_y; p.flip_x = flip_x; p.flip_y = flip_y;
    p.rows = d_rows; p.n_rows = d_rows ? n_rows : H;
    const long long n = (long long)p.n_rows * W;
    make_rays_kernel<<<(unsigned)((n + 255) / 256), 256, 0, (cudaStream_t)stream>>>(p, d_rays_o, d_rays_d, d_viewdirs);
    K4_CUDA_TRY(cudaGetLastError());
    return K4_OK;
}

extern "C" int k4_make_rays(const float* h_K, const float* h_c2w, int32_t H, int32_t W, int32_t ndc,
                            int32_t inverse_y, int32_t flip_x, int32_t flip_y,
                            float* d_rays_o, float* d_rays_d, float* d_viewdirs, k4_stream_t stream) {
    return k4_make_rays_rows(h_K, h_c2w, H, W, ndc, inverse_y, flip_x, flip_y, nullptr, H, d_rays_o, d_rays_d, d_viewdirs, stream);
}
