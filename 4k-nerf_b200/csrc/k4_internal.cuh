// k4_internal.cuh -- structures shared by the translation units of libk4nerf.so (sm_90a only).
#pragma once
#include <cuda_runtime.h>
#include <cuda_fp16.h>
#include <stdint.h>
#include "../../include/k4nerf.h"

#define K4_SKIP_B 4               // occupancy voxels per skip cell edge
#define K4_SKIP_MAXD 48           // distance-field cap (cells); larger true distances are stored as the cap
#define K4_MAX_WIDTH 256          // widest hidden layer the fp32 path accepts
#define K4_MAX_DIM0 128           // widest MLP input the fp32 path accepts

// Device-side view of a scene; passed to kernels by value (__grid_constant__).
struct K4Dev {
    int kind;
    int X, Y, Z;                  // density / k0 grid size (z fastest)
    int C, Cpad;                  // k0 channels, padded to a multiple of 4 in the channel-last copy
    int mX, mY, mZ;               // occupancy mask size
    float xyz_min[3], xyz_max[3], xyz_len[3];
    float m_scale[3], m_shift[3];
    float act_shift, voxel_size, voxel_size_ratio, thres;
    int max_world_size, mpi_depth;
    int depth, width, direct, viewpe, spape;
    int dim0;                     // MLP input width (0 when depth == 0)
    int k0_view_off;              // first k0 channel fed to the MLP (3 when !direct, else 0)
    int n_in[K4_MAX_MLP_LAYERS], n_out[K4_MAX_MLP_LAYERS], ldw[K4_MAX_MLP_LAYERS];
    // K4_ACT_GAUSS, fp32 mode: 2*(a*a) in fp32, the denominator of torch's -x**2/(2*a**2).  This field and act_c below
    // sit in what was alignment padding, so no other field moves and the kernels without the activation keep their
    // parameter layout.  The activation itself is a template parameter of the kernels (k4_scene::act selects them).
    float act_den;
    const float* density;         // [X,Y,Z]
    const float* k0cl;            // [X,Y,Z,Cpad] channel last
    const uint8_t* mask;          // [mX,mY,mZ]
    const float* act_grid;        // [mpi_depth] or nullptr
    const float* wT[K4_MAX_MLP_LAYERS];    // fp32 [n_in][ldw] (transposed, ldw = n_out padded to 4)
    const float* bias[K4_MAX_MLP_LAYERS];  // fp32 [ldw]
    // tensor-core packs (fp16 hi / lo parts, [n_out_pad][k_pad] row major = "B^T", K contiguous)
    const __half* wh[K4_MAX_MLP_LAYERS];
    const __half* wl[K4_MAX_MLP_LAYERS];
    int kpad[K4_MAX_MLP_LAYERS], npad[K4_MAX_MLP_LAYERS];
    // wgmma pack: one blob of canonical K-major (no swizzle) operand tiles, see tc_blob_layout()
    const unsigned char* tc_blob;
    int tc_kpad, tc_width;
    int tc_cfg;                   // id of the K4_WS_CFG_LIST entry (k4_ws_cfgs.h) the blob is packed for, -1: none
    // empty-space skipping (k4_march_common.cuh skip_steps): Chebyshev distance field over K4_SKIP_B^3-voxel cells of
    // the occupancy mask, in cells: 0 = the cell holds an occupied voxel, d = every cell within d-1 is empty
    const uint8_t* skip;          // [cX,cY,cZ] or nullptr (skipping off)
    int cX, cY, cZ;
    float m_iscale[3];            // 1 / m_scale
    // DirectContractedVoxGO (lib/dcvgo.py)
    float scene_center[3], scene_radius[3], bg_len, one_plus_bg;
    int world_len;
    float act_c;                  // K4_ACT_GAUSS, tensor-core modes: -log2(e) / (2 a^2), from double (see act_den)
    const int* tc_colmap;        // [dim0]: column of every model input in the tc_cfg entry's row layout (k4_testing_rgbnet)
};

// ---- wgmma operand blob (built by k4_scene_create, staged by one TMA bulk copy) -------------------
// Canonical K-major SWIZZLE_NONE layout of a [rows][K] fp16 tile with K/8 16-byte chunks per row:
// byte offset of (row r, chunk kc) = (r/8)*(kchunks*128) + kc*128 + (r%8)*16, i.e. 8x16B "core
// matrices", LBO = 128 B between K chunks, SBO = kchunks*128 B between 8-row groups.
__host__ __device__ inline int tc_canon_off(int r, int kc, int kchunks) {
    return (r >> 3) * (kchunks * 128) + kc * 128 + (r & 7) * 16;
}
struct TcBlobLayout {
    int off_w1, off_w2, off_w3, off_b1, off_b2, off_b3, off_ones, total;
};
// W1 [W][kpad], W2 [W][W], W3 [16][W], bias tiles B1/B2 [W][16], B3 [16][16] (col 0 = fp16(b),
// col 1 = fp16(b - col0)), ONES [128][16] (cols 0,1 = 1): a layer's bias is one extra K=16 MMA -- but for layer 1 of a
// config with two spare K columns (k4_ws_bias_col), whose bias hi / lo sit in those columns of W1 (B1 stays zero).
// Output channel c of the last layer is row 2c of W3 and B3 (the other rows are zero), for the epilogue of mlp_batch_wgmma.
__host__ __device__ inline TcBlobLayout tc_blob_layout(int kpad, int w) {
    TcBlobLayout L;
    int o = 0;
    L.off_w1 = o; o += w * kpad * 2;
    L.off_w2 = o; o += w * w * 2;
    L.off_w3 = o; o += 16 * w * 2;
    L.off_b1 = o; o += w * 16 * 2;
    L.off_b2 = o; o += w * 16 * 2;
    L.off_b3 = o; o += 16 * 16 * 2;
    L.off_ones = o; o += 128 * 16 * 2;
    L.total = o;
    return L;
}

struct k4_scene {
    K4Dev dev;
    int device;
    size_t bytes;
    void* allocs[64];
    int n_allocs;
    int act;                      // K4_ACT_* of the rgbnet's hidden layers: which kernel instantiations run the scene
};
static_assert(sizeof(K4Dev) == 704, "K4Dev grew: the kernels' parameter layout would move");

struct K4RenderParams {
    float near_, far_, stepdist, interval, bg, inv_nsamples;
    const float* t_list;          // DCVGO: per-step ray parameter (device, n_samples entries)
    float dist_thres;             // DCVGO: cumdist_thres threshold (lib/dcvgo.py:283)
    int n_samples;                // MPI: samples per ray; DVGO: depth normaliser only
    int render_depth;
    int image_w, image_h;         // >0: 2-D 8x4 tiles
    long long n_rays;
    long long n_tiles;
    const float* rays_o;
    const float* rays_d;
    const float* viewdirs;
    float* rgb;
    float* depth;
    float* alphainv;
    int* ray_stats;
    float* t_minmax;
    unsigned long long* counters;
    unsigned int* tile_counter;
    // k4_render_rays_frames (multi-GPU frame output): n_dst > 0 -> rgb / depth / alphainv above are unused and the ray of
    // local row r, column c is stored at ray index g = (((r >> 3) * f_world + f_rank) * 8 + (r & 7)) * f_w + c of every
    // frame d_frame[0 .. n_dst) (the local one and the peer-mapped ones): rgb at 3g, depth at 3 f_nfull + g, alphainv
    // at 4 f_nfull + g
    int n_dst, f_rank, f_world, f_w;
    long long f_nfull;
    float* d_frame[K4_MAX_PEERS];
};

// error plumbing (k4_capi.cu)
void k4_set_cuda_error(cudaError_t e, const char* where);
#define K4_CUDA_TRY(expr)                                            \
    do {                                                             \
        cudaError_t _e = (expr);                                     \
        if (_e != cudaSuccess) { k4_set_cuda_error(_e, #expr); return K4_ERR_CUDA; } \
    } while (0)

// launchers
int k4_launch_march(const k4_scene* sc, const K4RenderParams& rp, int mlp_mode, cudaStream_t st);
bool k4_ws_supported(const K4Dev& v);
// k4_testing_ws_row_layout: the compile-time row layout of K4_WS_CFG_LIST entry `id` (k4_march_ws.cu)
int k4_ws_row_layout(int id, int32_t out[4]);
// the warp-specialised wgmma marcher; K4_ERR_UNSUPPORTED if the shape has no wgmma build.  phases != NULL runs the profiled kernel (k4_testing_march_phases), which
// writes the phase counters of at most max_ctas CTAs there; *n_ctas (may be NULL) receives the CTA count
int k4_launch_march_ws(const k4_scene* sc, K4RenderParams rp, cudaStream_t st, unsigned long long* phases = nullptr,
                       int max_ctas = 0, int* n_ctas = nullptr);
// k4_testing_rgbnet for the wgmma modes (arguments already checked; k4_capi.cu runs the other modes)
int k4_testing_rgbnet_ws(const k4_scene* sc, const k4_rgbnet_test_args* a, cudaStream_t st);

// A 3x3 / pad 1 convolution with bias and ReLU on the decoder's wgmma kernels (k4_sr.cu), for LPIPS's VGG16
// (k4_lpips.cu), with every value carried as an fp16 pair hi = fp16(x), lo = fp16(x - hi).  k4_conv3x3_pack packs
// w [cout][cin][3][3] and b [cout] (fp32, device) into one allocation: cout / 64 blocks of 64 output channels, K = 3 cin
// (the weights w_hi, w_hi, w_lo against the activations' hi, lo, hi copies).  k4_conv3x3_relu_split reads src, fp16
// NHWC with cin_pad channels per pixel ([hi | lo | hi] of cin channels each, then zeros), and writes dst, fp16 NHWC
// with 3 cout channels: [hi | lo | hi] of max(conv + b, 0) (fp32 accumulation).  Caller's stream, no host sync.
struct K4Conv3x3Pack {
    void* blob;
    unsigned char* wpack;         // [cout / 64][ws_bytes]: conv3x3_ws_kernel packs
    float* bias;                  // [cout]
    size_t ws_bytes;
    int cin, cin_pad, cout;       // cin_pad = 3 cin rounded up to 32
};
int k4_conv3x3_pack(const float* w, const float* b, int cout, int cin, cudaStream_t s, K4Conv3x3Pack* c);
void k4_conv3x3_free(K4Conv3x3Pack* c);
int k4_conv3x3_relu_split(const K4Conv3x3Pack& c, const __half* src, int H, int W, __half* dst, cudaStream_t s);
