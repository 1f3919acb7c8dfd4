/*
 * k4nerf.h -- C ABI of libk4nerf.so, the H100 (sm_90a) implementation of the 4K-NeRF rendering
 * hot path.  This header is the drop-in boundary (SURVEY.md section 8b): plain pointers and sizes,
 * no torch types.  The reference has no C ABI of its own; every entry point below names the
 * reference interface it replaces (file:line under /root/reference).  The Python host mirror of
 * the reference API (k4nerf.dvgo.DirectVoxGO etc.) is a thin ctypes caller of these functions;
 * INTEGRATION.md shows the binding a reference maintainer would add.
 *
 * Conventions
 *  - every function returns K4_OK (0) or a negative k4_status; nothing throws, nothing exits;
 *  - all pointers named d_* / inside descriptors are DEVICE pointers on the current device unless
 *    the name says host (h_*); fp32 unless stated;
 *  - the caller allocates and owns all outputs and the workspace; no hidden allocation, no hidden
 *    host synchronisation on the render calls (the reference syncs twice per call:
 *    lib/cuda/render_utils_kernel.cu:212 and :635);
 *  - all work is enqueued on the given stream (pass torch.cuda.current_stream().cuda_stream);
 *  - re-entrant across streams; a k4_scene is immutable after creation.
 */
#ifndef K4NERF_H_
#define K4NERF_H_

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define K4_ABI_VERSION 1

#if defined(__GNUC__)
#define K4_API __attribute__((visibility("default")))
#else
#define K4_API
#endif

typedef enum k4_status {
    K4_OK = 0,
    K4_ERR_INVALID_ARG = -1,   /* NULL pointer, bad shape, bad enum                     */
    K4_ERR_UNSUPPORTED = -2,   /* valid in the reference but not built here (see DESIGN) */
    K4_ERR_CUDA = -3,          /* a CUDA runtime call failed; see k4_last_cuda_error()   */
    K4_ERR_WORKSPACE = -4,     /* workspace NULL or smaller than k4_render_workspace_bytes */
    K4_ERR_NO_DEVICE = -5      /* no sm_90 device / library built for another arch       */
} k4_status;

typedef void* k4_stream_t;                 /* cudaStream_t */
typedef struct k4_scene k4_scene;          /* opaque: device-resident, repacked scene     */
typedef struct k4_srnet k4_srnet;          /* opaque: device-resident VC-Decoder weights  */

enum { K4_KIND_DVGO = 0,                   /* DirectVoxGO,            lib/dvgo.py:23-448   */
       K4_KIND_DMPIGO = 1,                 /* DirectMPIGO,            lib/dmpigo.py:18-427 */
       K4_KIND_DCVGO = 2 };                /* DirectContractedVoxGO,  lib/dcvgo.py:27-382  */

enum { K4_MLP_FP32 = 0,                    /* fp32 FFMA, sequential accumulation (exact mode)   */
       K4_MLP_F16 = 1,                     /* tensor cores, fp16 operands, fp32 accumulate       */
       K4_MLP_F16X3 = 2,                   /* tensor cores, error-compensated 3-term fp16 split  */
       K4_MLP_TCGEN05 = 3,                 /* alias of K4_MLP_TCGEN05_WS, kept for compatibility */
       K4_MLP_TCGEN05_WS = 4 };            /* wgmma, fp16 operands, MLP in its own warpgroups    */

/* The colour MLP's hidden activation (DirectMPIGO's fine_model_and_render.act_type, lib/dmpigo.py:89-95): the
 * module after every hidden nn.Linear.  DirectVoxGO and DirectContractedVoxGO always use K4_ACT_RELU.
 *   K4_ACT_RELU    max(x, 0)
 *   K4_ACT_GAUSS   exp(-x^2 / (2 a^2)), GaussianActivation (lib/act.py), a = k4_scene_desc.rgbnet_act_param
 *   K4_ACT_LKRELU  x > 0 ? x : 0.01 x (nn.LeakyReLU())
 * Every mode evaluates the activation in fp32 on the layer's fp32 result.  fp32 mode follows torch's expression
 * order (gauss: expf(-(x*x) / (2*(a*a))), division and expf as torch does them); the tensor-core modes take
 * ex2.approx(x*x*c) with c = -log2(e) / (2 a^2) rounded once from double, and round the activated value to fp16 as
 * they round a ReLU'd one. */
enum { K4_ACT_RELU = 0, K4_ACT_GAUSS = 1, K4_ACT_LKRELU = 2 };

#define K4_MAX_MLP_LAYERS 8
#define K4_MAX_PEERS 8            /* GPUs of one NVLink / NVSwitch node */

/*
 * Scene description = the tensors of a reference checkpoint's `model_state_dict` plus the derived
 * scalars its constructor computes (SURVEY.md section 5 "Checkpoint"):
 *   density.grid [1,1,X,Y,Z], k0.grid [1,C,X,Y,Z] (planar, z fastest: lib/grid.py:115),
 *   mask_cache.mask [mX,mY,mZ] bool + xyz2ijk_scale/shift (lib/grid.py:290-293),
 *   act_shift (DVGO scalar lib/dvgo.py:46 | MPI grid [1,1,1,1,D] lib/dmpigo.py:48-58),
 *   rgbnet.{0,1.0,...}.{weight,bias} (lib/dvgo.py:116-124; weight [out,in] row major).
 * k4_scene_create copies/repacks everything it needs; the caller may free its tensors afterwards.
 */
typedef struct k4_scene_desc {
    int32_t kind;                 /* K4_KIND_*                                                  */
    int32_t world_size[3];        /* X, Y, Z                                                    */
    int32_t k0_dim;               /* C (3 when rgbnet_depth == 0)                               */
    int32_t mask_size[3];         /* mX, mY, mZ                                                 */
    float xyz_min[3];
    float xyz_max[3];
    float xyz2ijk_scale[3];
    float xyz2ijk_shift[3];
    float act_shift;              /* DVGO: density bias (lib/dvgo.py:46); MPI: ignored          */
    float voxel_size;             /* DVGO: lib/dvgo.py:155; MPI: ignored                        */
    float voxel_size_ratio;       /* lib/dvgo.py:158 | lib/dmpigo.py:164                        */
    float fast_color_thres;       /* lib/dvgo.py:38                                             */
    int32_t max_world_size;       /* DVGO: world_size.max() (depth normalisation, dvgo.py:311)  */
    int32_t mpi_depth;            /* MPI: number of planes (lib/dmpigo.py:159)                  */
    int32_t rgbnet_depth;         /* number of Linear layers; 0 = no MLP, rgb = sigmoid(k0)     */
    int32_t rgbnet_width;
    int32_t rgbnet_direct;        /* DVGO only (lib/dvgo.py:382-386,409-412)                    */
    int32_t viewbase_pe;          /* number of view-direction frequencies                       */
    int32_t spatial_pe;           /* MPI only: number of positional frequencies                 */
    int32_t rgbnet_act;           /* K4_ACT_*; MPI only, every other kind must keep K4_ACT_RELU  */
    const float* d_density;       /* [X*Y*Z]                                                    */
    const float* d_k0;            /* [C*X*Y*Z] planar, reference layout                         */
    const uint8_t* d_mask;        /* [mX*mY*mZ] bytes, non-zero = occupied                      */
    const float* d_act_shift_grid;/* MPI: [mpi_depth]; DVGO: NULL                               */
    const float* d_rgbnet_weight[K4_MAX_MLP_LAYERS]; /* [out,in] row major                      */
    const float* d_rgbnet_bias[K4_MAX_MLP_LAYERS];   /* [out]                                   */
    /* DirectContractedVoxGO only (lib/dcvgo.py:46-55,226-248): xyz_min/max above are -+(1+bg_len)  */
    float scene_center[3];        /* (xyz_min + xyz_max) / 2 of the foreground cube              */
    float scene_radius[3];        /* (xyz_max - xyz_min) / 2                                     */
    float bg_len;                 /* thickness of the contracted background shell                */
    int32_t world_len;            /* world_size[0]                                               */
    float rgbnet_act_param;       /* K4_ACT_GAUSS: the Gaussian's a (finite, > 0); ignored otherwise */
} k4_scene_desc;

/* render_kwargs of the reference forward (run_sr.py:1311-1320; lib/dvgo.py:327) + kernel knobs. */
typedef struct k4_render_args {
    float near_;                  /* render_kwargs['near']                                      */
    float far_;                   /* render_kwargs['far'] (DVGO forces 1e9, lib/dvgo.py:307)    */
    float stepsize;               /* render_kwargs['stepsize']                                  */
    float bg;                     /* render_kwargs['bg']                                        */
    int32_t render_depth;         /* render_kwargs['render_depth']                              */
    int32_t mlp_mode;             /* K4_MLP_*                                                   */
    int32_t image_w;              /* >0: rays are a row-major HxW image -> 8x4 pixel tiles/warp */
    int32_t image_h;
    /* DirectContractedVoxGO only: the per-step ray parameters `t` of sample_ray (lib/dcvgo.py:241-248,
     * a function of world_len, bg_len and stepsize only; the host computes them with the reference's
     * own torch expressions) and the cumdist_thres threshold (lib/dcvgo.py:283) */
    const float* d_t_list;
    int32_t n_t;
    float dist_thres;
} k4_render_args;

typedef struct k4_render_out {
    float* d_rgb_marched;         /* [N,3]  == rgb_feature (aliased in the reference, dvgo.py:425-427) */
    float* d_depth;               /* [N] or NULL                                                */
    float* d_alphainv_last;       /* [N]                                                        */
    int32_t* d_ray_stats;         /* optional [N,4]: N_steps, S_m, S_d, S_c per ray (parity)    */
    float* d_t_minmax;            /* optional [N,2]: t_min, t_max per ray (parity)              */
    unsigned long long* d_counters; /* optional [4]: total S_m, S_d, S_c, MLP batches           */
} k4_render_out;

K4_API int k4_abi_version(void);
K4_API const char* k4_status_string(int status);
K4_API const char* k4_last_cuda_error(void);       /* thread-local text of the last CUDA failure */
K4_API int k4_device_check(void);                  /* K4_OK iff the current device is sm_90      */

/* Replaces: utils.load_model -> model.to(device) (lib/utils.py:62-66) for the marcher's tensors. */
K4_API int k4_scene_create(const k4_scene_desc* desc, k4_stream_t stream, k4_scene** out_scene);
K4_API int k4_scene_destroy(k4_scene* scene);
K4_API size_t k4_scene_device_bytes(const k4_scene* scene);
/* The fastest K4_MLP_* mode built for this scene's rgbnet shape: K4_MLP_TCGEN05_WS for every 3-layer MLP that one of
 * the instantiated wgmma configurations covers (csrc/k4_ws_cfgs.h: k0 <= 16 channels, <= 6 view / <= 5 position
 * frequencies, width <= 128, rgbnet_direct either way), else the mma.sync / fp32 kernels.  k4_scene_ws_config: the
 * id of that configuration, -1 if none. */
K4_API int k4_scene_best_mlp_mode(const k4_scene* scene);
K4_API int k4_scene_ws_config(const k4_scene* scene);

/* Scratch needed by k4_render_rays for n_rays (a few bytes of scheduler state). */
K4_API size_t k4_render_workspace_bytes(const k4_scene* scene, int64_t n_rays);

/*
 * Replaces: DirectVoxGO.forward (lib/dvgo.py:327-448) / DirectMPIGO.forward (lib/dmpigo.py:292-427)
 * at inference, i.e. the whole chain sample_pts_on_rays -> maskcache_lookup -> grid_sample ->
 * raw2alpha -> alpha2weight -> grid_sample -> rgbnet -> segment_coo in ONE launch.
 * d_rays_o/d_rays_d/d_viewdirs: [N,3] contiguous fp32 (the reference CHECK_CONTIGUOUS contract,
 * lib/cuda/render_utils.cpp:46-48).  Any N >= 0.
 */
K4_API int k4_render_rays(const k4_scene* scene, const k4_render_args* args,
                   const float* d_rays_o, const float* d_rays_d, const float* d_viewdirs,
                   int64_t n_rays, const k4_render_out* out,
                   void* d_workspace, size_t workspace_bytes, k4_stream_t stream);

/*
 * Multi-GPU frames (SURVEY.md section 8e; the reference has no multi-GPU path -- run_sr.py:99-128 renders every frame on
 * one device): the same fused launch for ONE RANK'S ROWS of a frame that is sharded in 8-row blocks dealt round-robin
 * over `world` ranks, with the exchange fused into the kernel: every ray's results are stored straight into the
 * image-order frame of EVERY rank -- d_frame[i] are the local frame and the peers' frames mapped with k4_peer_open
 * (NVLink P2P stores) -- instead of a local band buffer followed by an all-gather and a transpose.  The rays passed are
 * the rank's rows in order (k4_make_rays_rows), n_rays = rows * frame_w; local row r is image row
 * ((r / 8) * world + rank) * 8 + r % 8.  A frame is 5 * n_full floats: rgb [n_full,3] | depth [n_full] | alphainv
 * [n_full], n_full >= the padded image (world * ceil(ceil(H/8) / world) * 8 rows).  `out` may be NULL or carry the
 * optional parity outputs (d_ray_stats / d_t_minmax / d_counters, local ray order).  The stores are complete when the
 * launch has completed on this rank's stream; the caller orders the ranks (any barrier that follows it in stream order).
 */
typedef struct k4_frame_dst {
    int32_t n_dst;                /* frames to write: 1 .. K4_MAX_PEERS                                  */
    int32_t rank, world;          /* block-cyclic position of the rows of this call                      */
    int32_t frame_w;              /* W                                                                   */
    int64_t n_full;               /* rays per (padded) frame                                             */
    float* d_frame[K4_MAX_PEERS];
} k4_frame_dst;
K4_API int k4_render_rays_frames(const k4_scene* scene, const k4_render_args* args,
                   const float* d_rays_o, const float* d_rays_d, const float* d_viewdirs,
                   int64_t n_rays, const k4_frame_dst* dst, const k4_render_out* out,
                   void* d_workspace, size_t workspace_bytes, k4_stream_t stream);

/* Device memory other processes of the node can map (one process per GPU): k4_peer_alloc = cudaMalloc + zero fill
 * (pool / async allocations cannot be exported), k4_peer_export fills the 64-byte CUDA IPC handle to send to the other
 * ranks (any transport: torch.distributed.all_gather_object), k4_peer_open maps another PROCESS's allocation into the
 * current device's address space with peer access enabled, k4_peer_close unmaps it. */
K4_API int k4_peer_enable_all(void);                 /* peer access from the current device to every device that allows it */
K4_API int k4_peer_alloc(size_t bytes, void** d_ptr);
K4_API int k4_peer_free(void* d_ptr);
K4_API int k4_peer_export(void* d_ptr, unsigned char handle[64]);
K4_API int k4_peer_open(const unsigned char handle[64], void** d_ptr);
K4_API int k4_peer_close(void* d_ptr);

/*
 * Replaces: get_rays_of_a_view (lib/dvgo.py:516-582) feeding the chunk loop of render_viewpoints
 * (run_sr.py:99-128): pixel-centre rays of an HxW pinhole view generated on the device.
 * h_K: 9 floats row major, h_c2w: 12 floats (3x4) row major, both HOST pointers.
 * d_rays_o/d_rays_d/d_viewdirs: [H*W,3] outputs.
 */
K4_API int k4_make_rays(const float* h_K, const float* h_c2w, int32_t H, int32_t W, int32_t ndc,
                 int32_t inverse_y, int32_t flip_x, int32_t flip_y,
                 float* d_rays_o, float* d_rays_d, float* d_viewdirs, k4_stream_t stream);

/* Same for a subset of the image rows (multi-GPU: a rank generates only ITS rows of the frame, SURVEY.md
 * section 8e): d_rows = DEVICE array of n_rows image-row indices (NULL = all H rows in order);
 * outputs are [n_rows*W,3] in the order of d_rows.  Values are identical to the same pixels of k4_make_rays. */
K4_API int k4_make_rays_rows(const float* h_K, const float* h_c2w, int32_t H, int32_t W, int32_t ndc,
                 int32_t inverse_y, int32_t flip_x, int32_t flip_y, const int32_t* d_rows, int32_t n_rows,
                 float* d_rays_o, float* d_rays_d, float* d_viewdirs, k4_stream_t stream);

/* ------------------------------------------------------------------------------------------------
 * VC-Decoder: SFTNet (lib/sr_esrnet.py:400-465), the SFT-RRDB decoder that turns the marcher's
 * rgb_feature + depth images into the output frame (run_sr.py:1353-1387): x4, the 4K upsampler, or x1, the
 * refinement network of the 1x configurations (no upsampling; conv_hr and conv_last run at the input resolution).
 *
 * h_params: HOST array of DEVICE pointers to the fp32 parameters (weight, bias alternating) of the
 * convolutions in this fixed order -- the reference module's registration order:
 *   conv_first; CondNet.0, CondNet.2, CondNet.4, CondNet.6;
 *   for i in blocks: for j in rdb1..rdb3: conv1..conv5,
 *                                          sft0.{SFT_scale_conv0, SFT_scale_conv1, SFT_shift_conv0, SFT_shift_conv1},
 *                                          sft1.{same four};
 *                    body.i.sft0.{same four};
 *   sftbody.{same four}; then
 *     scale 4: conv_body; conv_up1; conv_up2; conv_hr; conv_last.
 *     scale 1: conv_body; conv_hr; conv_last.
 * n_params = 2 * (1 + 4 + 43 * num_block + 4 + (scale == 4 ? 5 : 3)): 229 convolutions for 5 blocks at x4, 227 at x1;
 * a count that does not match the scale returns K4_ERR_INVALID_ARG.
 * Only SFTNet(n_in_colors=3, scale=4 or 1, num_feat=64, num_block<=32, num_grow_ch=32, num_cond=1..64, dswise=False)
 * (run_sr.py:1353) is built; other configurations, scale 2 and num_cond > 64 included, return K4_ERR_UNSUPPORTED, and
 * num_cond < 1 returns K4_ERR_INVALID_ARG.  num_cond is CondNet.0's input width (weight [64][num_cond][3][3]): 1 for the
 * depth condition, 63 for the view-direction embedding, 64 for depth followed by the embedding (run_sr.py:895-912).
 */
typedef struct k4_srnet_desc {
    int32_t n_in_colors, scale, num_feat, num_block, num_grow_ch, num_cond;
    int32_t n_params;                  /* = 2 * number of convolutions */
    int32_t reserved0;
    const float* const* h_params;
} k4_srnet_desc;

K4_API int k4_srnet_create(const k4_srnet_desc* desc, k4_stream_t stream, k4_srnet** out_net);
K4_API int k4_srnet_destroy(k4_srnet* net);
/* Device workspace of one h x w tile for `net`'s scale (x1 needs less than x4); net == NULL gives the x4 size, which
 * covers every built scale. */
K4_API size_t k4_srnet_workspace_bytes(const k4_srnet* net, int32_t h, int32_t w);

/* Replaces: SFTNet.forward(x, cond) (lib/sr_esrnet.py:446-465) for one tile.
 * d_x [3,h,w], d_cond [num_cond,h,w] planar fp32 (the reference's NCHW, batch 1); d_out [3,s*h,s*w] fp32 with s the
 * net's scale (4 or 1).  The same d_cond layout holds for k4_srnet_forward_roi and k4_srnet_forward_roi_peers.
 * Tiling (SFTNet.tile_process, lib/sr_esrnet.py:467-527) is host logic above this call. */
K4_API int k4_srnet_forward(const k4_srnet* net, const float* d_x, const float* d_cond, int32_t h, int32_t w,
                            float* d_out, void* d_workspace, size_t workspace_bytes, k4_stream_t stream);

/* The same forward when only a block of the tile's output is wanted -- what SFTNet.tile_process does with every tile
 * (lib/sr_esrnet.py:509-523 crops the 10-pixel pad away and copies the rest into the frame) and what the multi-GPU
 * decoder does with a tile's row parts.  keep_* select LR rows [keep_y0,keep_y1) x columns [keep_x0,keep_x1) of the
 * h x w input; their x scale pixels (x4: 4x4 per LR pixel; x1: the block 1:1) are written straight to
 * d_out[c*out_plane_stride + Y*out_row_stride + X] with (Y, X) relative to the block's first pixel (pass a pointer into
 * the frame and the frame's strides).  Every layer computes only
 * the rows inside the remaining receptive field of the kept rows; the values are bit-identical to k4_srnet_forward's. */
K4_API int k4_srnet_forward_roi(const k4_srnet* net, const float* d_x, const float* d_cond, int32_t h, int32_t w,
                                int32_t keep_y0, int32_t keep_y1, int32_t keep_x0, int32_t keep_x1,
                                float* d_out, int64_t out_plane_stride, int64_t out_row_stride,
                                void* d_workspace, size_t workspace_bytes, k4_stream_t stream);

/* k4_srnet_forward_roi whose last convolution stores the kept block into n_extra MORE frames as well (h_extra: HOST array
 * of device pointers with d_out's meaning and strides -- the same window of the other ranks' frames, mapped with
 * k4_peer_open): the multi-GPU decoder's exchange fused into the kernel that produces the pixels, instead of an
 * all-gather of packed blocks and an assembly pass.  n_extra <= K4_MAX_PEERS - 1. */
K4_API int k4_srnet_forward_roi_peers(const k4_srnet* net, const float* d_x, const float* d_cond, int32_t h, int32_t w,
                                      int32_t keep_y0, int32_t keep_y1, int32_t keep_x0, int32_t keep_x1,
                                      float* d_out, int64_t out_plane_stride, int64_t out_row_stride,
                                      int32_t n_extra, float* const* h_extra,
                                      void* d_workspace, size_t workspace_bytes, k4_stream_t stream);

/* ------------------------------------------------------------------------------------------------
 * Op-level surface: the 13 functions of the reference extension `render_utils_cuda`
 * (lib/cuda/render_utils.cpp:170-184), bit-identical results, caller-allocated outputs, no host sync.
 * Needed for training compatibility (lib/dvgo.py:453-511 autograd shims), not for inference.
 * All pointers are device pointers; masks are bytes (torch.bool); ids are int64.
 *   reference function                      entry point(s)
 *   infer_t_minmax            (.cpp:50)     k4_op_infer_t_minmax
 *   infer_n_samples           (.cpp:60)     k4_op_infer_n_samples
 *   infer_ray_start_dir       (.cpp:68)     k4_op_infer_ray_start_dir
 *   sample_pts_on_rays        (.cpp:76)     the three above + cumsum (host side) + k4_op_fill_ray_step_ids + k4_op_sample_pts
 *   sample_ndc_pts_on_rays    (.cpp:92)     k4_op_sample_ndc_pts
 *   sample_bg_pts_on_rays     (.cpp:104)    k4_op_sample_bg_pts
 *   maskcache_lookup          (.cpp:112)    k4_op_maskcache_lookup       (out must be pre-zeroed, as .cu:405)
 *   raw2alpha[_nonuni]        (.cpp:124,131) k4_op_raw2alpha             (interval_v = NULL | per-point intervals)
 *   raw2alpha[_nonuni]_backward (.cpp:138,146) k4_op_raw2alpha_backward
 *   alpha2weight              (.cpp:154)    k4_op_alpha2weight           (outputs pre-filled 0/1/1/0/0 as .cu:624-628)
 *   alpha2weight_backward     (.cpp:162)    k4_op_alpha2weight_backward  (grad pre-zeroed as .cu:684)
 */
K4_API int k4_op_infer_t_minmax(const float* d_rays_o, const float* d_rays_d, const float* d_xyz_min, const float* d_xyz_max,
                                float near_, float far_, int64_t n_rays, float* d_t_min, float* d_t_max, k4_stream_t stream);
K4_API int k4_op_infer_n_samples(const float* d_rays_d, const float* d_t_min, const float* d_t_max, float stepdist, int64_t n_rays,
                                 int64_t* d_n_samples, k4_stream_t stream);
K4_API int k4_op_infer_ray_start_dir(const float* d_rays_o, const float* d_rays_d, const float* d_t_min, int64_t n_rays,
                                     float* d_rays_start, float* d_rays_dir, k4_stream_t stream);
K4_API int k4_op_fill_ray_step_ids(const int64_t* d_n_steps_cumsum, int64_t n_rays, int64_t total, int64_t* d_ray_id,
                                   int64_t* d_step_id, k4_stream_t stream);
K4_API int k4_op_sample_pts(const float* d_rays_start, const float* d_rays_dir, const float* d_xyz_min, const float* d_xyz_max,
                            const int64_t* d_ray_id, const int64_t* d_step_id, float stepdist, int64_t total, float* d_pts,
                            uint8_t* d_mask_outbbox, k4_stream_t stream);
K4_API int k4_op_sample_ndc_pts(const float* d_rays_o, const float* d_rays_d, const float* d_xyz_min, const float* d_xyz_max,
                                int32_t N_samples, int64_t n_rays, float* d_pts, uint8_t* d_mask_outbbox, k4_stream_t stream);
K4_API int k4_op_sample_bg_pts(const float* d_rays_o, const float* d_rays_d, const float* d_t_max, float bg_preserve,
                               int32_t N_samples, int64_t n_rays, float* d_pts, k4_stream_t stream);
K4_API int k4_op_maskcache_lookup(const uint8_t* d_world, const float* d_xyz, uint8_t* d_out, const float* d_scale,
                                  const float* d_shift, int32_t sz_i, int32_t sz_j, int32_t sz_k, int64_t n_pts, k4_stream_t stream);
K4_API int k4_op_raw2alpha(const float* d_density, float shift, float interval, const float* d_interval_v, int64_t n_pts,
                           float* d_exp, float* d_alpha, k4_stream_t stream);
K4_API int k4_op_raw2alpha_backward(const float* d_exp, const float* d_grad_back, float interval, const float* d_interval_v,
                                    int64_t n_pts, float* d_grad, k4_stream_t stream);
K4_API int k4_op_alpha2weight(const float* d_alpha, const int64_t* d_ray_id, int64_t n_rays, int64_t n_pts, float* d_weight,
                              float* d_T, float* d_alphainv_last, int64_t* d_i_start, int64_t* d_i_end, k4_stream_t stream);
K4_API int k4_op_alpha2weight_backward(const float* d_alpha, const float* d_weight, const float* d_T, const float* d_alphainv_last,
                                       const int64_t* d_i_start, const int64_t* d_i_end, int64_t n_rays,
                                       const float* d_grad_weights, const float* d_grad_last, float* d_grad, k4_stream_t stream);

/* ------------------------------------------------------------------------------------------------
 * Grid maintenance and optimiser steps either side of the render path during training
 * (SURVEY.md section 8 f-4).  Device pointers unless prefixed h_; caller's stream; no host sync.
 *   reference                                                       entry point
 *   total_variation_cuda.total_variation_add_grad (lib/cuda/total_variation.cpp:16-20; param
 *       [1,C,I,J,K] contiguous, grad updated in place; !dense_mode skips grad==0)   k4_op_total_variation_add_grad
 *   adam_upd_cuda.adam_upd / masked_adam_upd / adam_upd_with_perlr (lib/cuda/adam_upd.cpp:37-75;
 *       d_perlr != NULL selects the per-voxel-lr variant, else skip_zero_grad the masked one;
 *       `step` is the 1-based step count after the increment, lib/masked_adam.py:57)  k4_op_adam_upd
 *   update_occupancy_cache (lib/dvgo.py:224-233, lib/dmpigo.py:212-224): alpha of the trilinear density
 *       at the occupancy grid's points (d_lx/ly/lz = the three torch.linspace vectors), then
 *       mask &= max_pool3d(alpha, 3, stride 1, pad 1) > thres              k4_op_grid_alpha, k4_op_maxpool3_thres_and
 *   DenseGrid.scale_volume_grid (lib/grid.py:130-135: F.interpolate(mode='trilinear',
 *       align_corners=True) of a [1,C,X,Y,Z] grid to [1,C,X2,Y2,Z2])        k4_op_resample_trilinear
 */
K4_API int k4_op_total_variation_add_grad(const float* d_param, float* d_grad, float wx, float wy, float wz, int32_t dense_mode,
                                          int64_t n, int32_t sz_i, int32_t sz_j, int32_t sz_k, k4_stream_t stream);
K4_API int k4_op_adam_upd(float* d_param, const float* d_grad, float* d_exp_avg, float* d_exp_avg_sq, const float* d_perlr,
                          int64_t n, int32_t step, float beta1, float beta2, float lr, float eps, int32_t skip_zero_grad,
                          k4_stream_t stream);
K4_API int k4_op_grid_alpha(const float* d_density, int32_t X, int32_t Y, int32_t Z, const float* h_xyz_min, const float* h_xyz_max,
                            const float* d_lx, const float* d_ly, const float* d_lz, int32_t mX, int32_t mY, int32_t mZ,
                            float shift, float interval, float* d_alpha, k4_stream_t stream);
K4_API int k4_op_maxpool3_thres_and(const float* d_alpha, int32_t mX, int32_t mY, int32_t mZ, float thres, uint8_t* d_mask,
                                    k4_stream_t stream);
/* ub360_utils_cuda.cumdist_thres (lib/cuda/ub360_utils.cpp:20-22; dist [n_rays, n_pts] -> bool mask, bit-identical) */
K4_API int k4_op_cumdist_thres(const float* d_dist, float thres, int64_t n_rays, int64_t n_pts, uint8_t* d_mask, k4_stream_t stream);
K4_API int k4_op_resample_trilinear(const float* d_src, int32_t C, int32_t X, int32_t Y, int32_t Z, float* d_dst, int32_t X2,
                                    int32_t Y2, int32_t Z2, k4_stream_t stream);

/* DenseGrid.forward with autograd (lib/grid.py:117-128): trilinear lookup of world points in a planar [1,C,X,Y,Z]
 * grid -- ((xyz-min)/(max-min)).flip(-1)*2-1, ATen grid_sampler_3d (bilinear, zeros, align_corners=True) and the
 * [C,M]->[M,C] transpose in one launch -- and its backward: the scatter of the output gradient [M,C] into the grid
 * gradient [C,X,Y,Z] (ACCUMULATED with atomics: the caller zero-fills), which the reference obtains from ATen's
 * grid_sampler_3d_backward.  h_xyz_min/max: 3 host floats each.  d_xyz [M,3], d_out / d_grad_out [M,C]. */
K4_API int k4_op_grid_sample(const float* d_grid, int32_t C, int32_t X, int32_t Y, int32_t Z, const float* h_xyz_min,
                             const float* h_xyz_max, const float* d_xyz, int64_t M, float* d_out, k4_stream_t stream);
K4_API int k4_op_grid_sample_backward(const float* d_grad_out, int32_t C, int32_t X, int32_t Y, int32_t Z, const float* h_xyz_min,
                                      const float* h_xyz_max, const float* d_xyz, int64_t M, float* d_grad_grid, k4_stream_t stream);

/* The distortion loss over a flat sample list (csrc/k4_distloss.cu): d_w / d_m [n_samples] fp32, d_ray_id
 * [n_samples] int64 non-decreasing and >= 0; a segment is a maximal run of equal ids, n = max(ray_id) + 1 (rays
 * without samples do not count).  With the exclusive in-segment prefixes W<i, WM<i (of w and w*m) and suffixes W>i, WM>i:
 *   L       = (sum_i 2 w_i (m_i W<i - WM<i) + interval/3 sum_i w_i^2) / n
 *   dL/dw_i = g/n (2 m_i (W<i - W>i) + 2 (WM>i - WM<i) + 2/3 interval w_i)
 *   torch_efficient_distloss.flatten_eff_distloss(w, m, interval, ray_id)      k4_op_distloss_forward + _backward
 *   ub360_utils_cuda.segment_cumsum(w, s, ray_id) (the op lib/dcvgo.py:390 calls): exclusive prefixes [n_samples],
 *       totals [n_rays] (0 for a ray without samples; ids >= n_rays are not written)   k4_op_segment_cumsum
 * interval is d_interval[0] when d_interval != NULL (a device scalar), else the host value.  The workspace holds
 * k4_op_distloss_workspace_bytes(n_samples) bytes, 16-byte aligned; the backward reads what the forward with the same
 * inputs left there (n and the per-tile carries), so the forward's workspace must be kept until the backward runs.
 * d_grad_loss is the upstream gradient g, a device scalar; divide_by_n = 0 leaves out the 1/n factor (lib/dcvgo.py:406).
 * The loss and the gradient are bitwise reproducible (fixed summation order).  Caller's stream, no host sync.
 * n_samples < 1, a NULL pointer or workspace: K4_ERR_INVALID_ARG; a workspace smaller than the size: K4_ERR_WORKSPACE. */
K4_API size_t k4_op_distloss_workspace_bytes(int64_t n_samples);
K4_API int k4_op_distloss_forward(const float* d_w, const float* d_m, const int64_t* d_ray_id, int64_t n_samples, float interval,
                                  const float* d_interval, float* d_loss, void* d_workspace, size_t workspace_bytes,
                                  k4_stream_t stream);
K4_API int k4_op_distloss_backward(const float* d_w, const float* d_m, const int64_t* d_ray_id, int64_t n_samples, float interval,
                                   const float* d_interval, const float* d_grad_loss, int32_t divide_by_n,
                                   const void* d_workspace, size_t workspace_bytes, float* d_grad_w, k4_stream_t stream);
K4_API int k4_op_segment_cumsum(const float* d_w, const float* d_s, const int64_t* d_ray_id, int64_t n_samples, int64_t n_rays,
                                float* d_w_prefix, float* d_w_total, float* d_ws_prefix, float* d_ws_total, void* d_workspace,
                                size_t workspace_bytes, k4_stream_t stream);

/* One scene-training step's render and loss, fused (csrc/k4_train_march.cu): the training forward of DirectVoxGO /
 * DirectMPIGO (lib/dvgo.py:327-448, lib/dmpigo.py:292-427) and run_sr.py's composite loss (run_sr.py:521-546, without
 * nearclip) in one forward kernel, and its gradient in one backward kernel that re-marches every ray.  The parameters are
 * read live, in their own layouts: density [X,Y,Z] (of [1,1,X,Y,Z]), k0 planar [C,X,Y,Z], mask [mX,mY,mZ] bytes, the MPI
 * act_shift [mpi_depth], rgbnet weights [out,in] and biases [out].  Loss terms (a weight of 0 skips its term):
 *   main          w_main * mean((rgb_marched - target)^2)
 *   entropy_last  w_entropy * mean over rays of the entropy of clamp(alphainv_last, 1e-6, 1 - 1e-6)
 *   distortion    w_distortion * flatten_eff_distloss(weights, s, 1 / n_samples, ray_id), divided by the largest shaded
 *                 ray id + 1 (DirectMPIGO only)
 *   rgbper        w_rgbper * sum over shaded samples of weight * |rgb - target|^2, divided by n_rays
 * d_loss [1] receives their sum, d_loss_terms [4] each weighted term (0 when skipped); both are bitwise reproducible.
 * d_bkgd [n_rays,3] (may be NULL: the scalar bg) is the background under rand_bkgd.  The backward ADDS dL/d(parameter),
 * times the device scalar *d_grad_loss, into the d_grad_* arrays (same layouts as the parameters; a NULL one is not
 * computed); the caller zero-fills them.  It reads what the forward left in the workspace
 * (k4_train_march_workspace_bytes(n_rays) bytes, 16-byte aligned).  Caller's stream, no host synchronisation.
 * A NULL pointer, n_rays < 1 or a bad enum / size: K4_ERR_INVALID_ARG; DirectContractedVoxGO, an rgbnet depth other
 * than 0 or 3, k0_dim > 32, width > 128, an MLP input wider than 128, a pe above 10: K4_ERR_UNSUPPORTED; both before
 * any CUDA call. */
typedef struct k4_train_march_args {
    int32_t kind;                 /* K4_KIND_DVGO / K4_KIND_DMPIGO                                   */
    int32_t rgbnet_act;           /* K4_ACT_* of the hidden layers (DirectMPIGO's act_type)          */
    int64_t n_rays;
    int32_t world_size[3];        /* density / k0 grid X, Y, Z                                       */
    int32_t k0_dim;
    int32_t mask_size[3];
    int32_t mpi_depth;
    float xyz_min[3], xyz_max[3];
    float xyz2ijk_scale[3], xyz2ijk_shift[3];
    float act_shift;              /* DirectVoxGO                                                     */
    float voxel_size;             /* DirectVoxGO: stepdist = stepsize * voxel_size (fp32)            */
    float interval;               /* float(stepsize * voxel_size_ratio), as the training forward     */
    float fast_color_thres;
    float near_, stepsize, bg;
    int32_t max_world_size;
    int32_t rgbnet_depth;         /* 0 (colour grid) or 3                                            */
    int32_t rgbnet_width;
    int32_t rgbnet_direct;
    int32_t viewbase_pe, spatial_pe;
    float rgbnet_act_param;       /* K4_ACT_GAUSS: GaussianActivation.a                              */
    float w_main, w_entropy, w_distortion, w_rgbper;
    const float* d_rays_o;        /* [n_rays,3] each                                                 */
    const float* d_rays_d;
    const float* d_viewdirs;
    const float* d_target;
    const float* d_bkgd;
    const float* d_density;
    const float* d_k0;
    const uint8_t* d_mask;
    const float* d_act_shift_grid;
    const float* d_rgbnet_weight[3];
    const float* d_rgbnet_bias[3];
    float* d_rgb_marched;         /* [n_rays,3]  forward outputs                                     */
    float* d_alphainv_last;       /* [n_rays]                                                        */
    float* d_loss;                /* [1]                                                             */
    float* d_loss_terms;          /* [4]: main, entropy_last, distortion, rgbper                     */
    float* d_grad_density;        /* backward outputs (accumulated)                                  */
    float* d_grad_k0;
    float* d_grad_weight[3];
    float* d_grad_bias[3];
} k4_train_march_args;

K4_API size_t k4_train_march_workspace_bytes(int64_t n_rays);
K4_API int k4_train_march_forward(const k4_train_march_args* args, void* d_workspace, size_t workspace_bytes, k4_stream_t stream);
K4_API int k4_train_march_backward(const k4_train_march_args* args, const float* d_grad_loss, const void* d_workspace,
                                   size_t workspace_bytes, k4_stream_t stream);

/* ------------------------------------------------------------------------------------------------
 * Evaluation metrics (csrc/k4_metrics.cu).
 *
 * Replaces: utils.rgb_ssim (lib/utils.py:88-134), the SSIM that render_viewpoints scores frames with (eval_ssim).
 * d_img0, d_img1: two H x W x 3 images of `dtype` (K4_DTYPE_F32 or K4_DTYPE_F64, both the same), element (y, x, c) at
 * y * strides[0] + x * strides[1] + c * strides[2] (host arrays of element strides; any value, 0 included, so permuted,
 * cropped and expanded views are read in place).  h_win: HOST array of the filter_size window taps, c1 = (k1 max_val)^2,
 * c2 = (k2 max_val)^2, as utils.rgb_ssim computes them.  Per channel, a separable 'valid' blur with the reversed taps
 * along rows, then columns, gives the means m0 / m1, variances v0 / v1 (clipped at 0) and covariance cov (clipped to
 * sign(cov) min(sqrt(v0 v1), |cov|)) of every window; the map value is
 *   ((2 m0 m1 + c1)(2 cov + c2)) / ((m0^2 + m1^2 + c1)(v0 + v1 + c2)).
 * Every operation is in fp64.  d_map (may be NULL): fp64 [H-f+1, W-f+1, 3] contiguous; d_mean: one device double, the
 * map's mean.  The workspace holds k4_op_rgb_ssim_workspace_bytes(H, W, filter_size) bytes (0 for an invalid shape),
 * 8-byte aligned; the mean is summed from per-tile sums in an order fixed by (H, W, filter_size), so it is bitwise
 * reproducible.  Caller's stream, no host sync.
 * A NULL pointer (other than d_map), filter_size outside 1 .. K4_SSIM_MAX_FILTER, H or W below filter_size, or another
 * dtype: K4_ERR_INVALID_ARG; a workspace smaller than the size: K4_ERR_WORKSPACE.
 */
#define K4_SSIM_MAX_FILTER 31
enum { K4_DTYPE_F32 = 0, K4_DTYPE_F64 = 1 };
/* Replaces: utils.rgb_ssim (lib/utils.py:88-134) -- the workspace of k4_op_rgb_ssim. */
K4_API size_t k4_op_rgb_ssim_workspace_bytes(int64_t H, int64_t W, int32_t filter_size);
/* Replaces: utils.rgb_ssim (lib/utils.py:88-134). */
K4_API int k4_op_rgb_ssim(const void* d_img0, const void* d_img1, int32_t dtype, int64_t H, int64_t W, const int64_t strides0[3],
                          const int64_t strides1[3], const double* h_win, int32_t filter_size, double c1, double c2,
                          double* d_map, double* d_mean, void* d_workspace, size_t workspace_bytes, k4_stream_t stream);

/* ------------------------------------------------------------------------------------------------
 * The joint stage's validation scores (csrc/k4_val.cu; DESIGN.md section 3.11).
 *
 * k4_op_resize_quarter replaces cv2.resize(img, None, fx=1/4, fy=1/4) (INTER_LINEAR, run_sr.py:1136) of an fp32
 * H x W x 3 image, bit for bit with cv2 4.13's IPP build.  d_src: element (y, x, c) at y * strides[0] + x * strides[1] +
 * c * strides[2] (HOST array of element strides, each >= 0).  d_dst: fp32 [h, w, 3] contiguous, h = cvRound(H / 4),
 * w = cvRound(W / 4) (halves round to even).  Per axis of n pixels, output k interpolates pixels 4k+1 and 4k+2 with
 * t = 0.5, or, when 4k + 3 > n, pixels n-2 and n-1 with t = 1, as a + (b - a) t with one rounding per operation; along
 * columns first, then rows.  With H or W equal to 3, rows first, and a pair past the edge reads pixel n-1 alone.
 * A NULL or misaligned pointer, a negative stride, or H or W outside 3 .. 65535: K4_ERR_INVALID_ARG, before any CUDA
 * call.  Caller's stream, no host sync, no allocation.
 *
 * k4_op_mse_f32 replaces np.mean(np.square(a - b)) of two float32 H x W x 3 arrays (run_sr.py:1132), bit for bit:
 * d = a - b and d * d in fp32, their sum in numpy's pairwise order (loops_utils.h's pairwise_sum over all 3 H W values),
 * added to 0, and *d_mse = float32(float64(sum) / (3 H W)) as numpy's mean computes it.  d_a, d_b and their strides as
 * k4_op_resize_quarter's source.  order: HOST int32[3], the axes (0 = y, 1 = x, 2 = c) from the outermost to the
 * innermost in the order numpy visits the difference's elements (its memory order: {0, 1, 2} for C-contiguous
 * operands, {2, 0, 1} when both are [3, H, W] planes viewed as [H, W, 3]).  The workspace holds
 * k4_op_mse_f32_workspace_bytes(H, W) bytes, 4-byte aligned (0: an invalid shape).  The sum's tree depends on 3 H W
 * only and is evaluated without atomics, so the result is bitwise reproducible.  Caller's stream, no host sync.
 * A NULL or misaligned pointer, a negative stride, H or W outside 1 .. 65535, or an order that is not a permutation of
 * {0, 1, 2}: K4_ERR_INVALID_ARG; a workspace smaller than the size: K4_ERR_WORKSPACE; both before any CUDA call.
 */
/* Replaces: cv2.resize(rgb, dsize=None, fx=1/4, fy=1/4) (run_sr.py:1136). */
K4_API int k4_op_resize_quarter(const float* d_src, int64_t H, int64_t W, const int64_t strides[3], float* d_dst,
                                k4_stream_t stream);
/* Replaces: np.mean(np.square(rgb_srsave - rgb_srgt_val[idx])) (run_sr.py:1132) -- the workspace of k4_op_mse_f32. */
K4_API size_t k4_op_mse_f32_workspace_bytes(int64_t H, int64_t W);
/* Replaces: np.mean(np.square(rgb_srsave - rgb_srgt_val[idx])) (run_sr.py:1132). */
K4_API int k4_op_mse_f32(const float* d_a, const float* d_b, int64_t H, int64_t W, const int64_t strides_a[3],
                         const int64_t strides_b[3], const int32_t order[3], float* d_mse, void* d_workspace,
                         size_t workspace_bytes, k4_stream_t stream);

/* ------------------------------------------------------------------------------------------------
 * LPIPS (csrc/k4_lpips.cu).
 *
 * Replaces: utils.rgb_lpips (lib/utils.py:137-149), lpips.LPIPS(net='vgg' | 'alex', version='0.1') called with
 * normalize=True, the perceptual metric of render_viewpoints' eval_lpips_vgg / eval_lpips_alex.
 *
 * k4_lpips_create: h_params is a HOST array of n_params DEVICE pointers to fp32 parameters, in this fixed order (the
 * keys of lpips.LPIPS(...).state_dict()):
 *   K4_LPIPS_VGG  (n_params 31): net.slice1.{0,2}, net.slice2.{5,7}, net.slice3.{10,12,14}, net.slice4.{17,19,21},
 *                 net.slice5.{24,26,28}, each .weight [cout][cin][3][3] then .bias [cout]; then lin0 .. lin4
 *                 .model.1.weight ([1][C][1][1], C = 64, 128, 256, 512, 512).
 *   K4_LPIPS_ALEX (n_params 15): net.slice1.0, net.slice2.3, net.slice3.6, net.slice4.8, net.slice5.10, each .weight
 *                 then .bias; then lin0 .. lin4 .model.1.weight (C = 64, 192, 384, 256, 256).
 * The scaling layer's shift (-.030, -.088, -.188) and scale (.458, .448, .450) are lpips' constants, built in.  The
 * parameters are copied (the call synchronises `stream`, so they may be freed on return).  A NULL pointer, another
 * net or another n_params: K4_ERR_INVALID_ARG, before any CUDA call.
 *
 * k4_lpips_forward: d_img0, d_img1: two H x W x 3 fp32 images in [0, 1], element (y, x, c) at y * strides[0] +
 * x * strides[1] + c * strides[2] (HOST arrays of element strides, so [H, W, 3] and [3, H, W] tensors and views are read
 * in place).  *d_out (one device double) receives the score: the sum over the five taps of the mean over the tap's
 * pixels of sum_c lin[c] (f0 / (|f0| + 1e-10) - f1 / (|f1| + 1e-10))^2, |f| the L2 norm of a pixel's channel vector.
 * VGG's convolutions run on the tensor cores with every activation and weight an fp16 pair hi + lo (three fp16 GEMM
 * terms, fp32 accumulation: fp32-class), AlexNet's in fp32; the head is fp64, summed in an order fixed by (net, H, W),
 * so the score is bitwise reproducible.  Caller's stream, no host sync.  The workspace holds
 * k4_lpips_workspace_bytes(net, H, W) bytes (0 for a size the trunk cannot take: VGG needs H, W >= 16, AlexNet
 * H, W >= 31; both at most 16384), 256-byte aligned.  A NULL pointer, a size outside those bounds or a misaligned
 * pointer: K4_ERR_INVALID_ARG; a workspace smaller than the size: K4_ERR_WORKSPACE; both before any CUDA call.
 */
enum { K4_LPIPS_VGG = 0, K4_LPIPS_ALEX = 1 };
typedef struct k4_lpips k4_lpips;
/* Replaces: lpips.LPIPS(net=..., version='0.1') (lib/utils.py:138-142). */
K4_API int k4_lpips_create(int32_t net, const float* const* h_params, int32_t n_params, k4_stream_t stream, k4_lpips** out_net);
K4_API int k4_lpips_destroy(k4_lpips* net);
/* Replaces: utils.rgb_lpips (lib/utils.py:144-149) -- the workspace of k4_lpips_forward. */
K4_API size_t k4_lpips_workspace_bytes(const k4_lpips* net, int64_t H, int64_t W);
/* Replaces: utils.rgb_lpips (lib/utils.py:144-149). */
K4_API int k4_lpips_forward(const k4_lpips* net, const float* d_img0, const float* d_img1, const int64_t strides0[3],
                            const int64_t strides1[3], int64_t H, int64_t W, double* d_out, void* d_workspace,
                            size_t workspace_bytes, k4_stream_t stream);

/* ------------------------------------------------------------------------------------------------
 * Video streams of run_sr.py --render_video (csrc/k4_video.cu).
 *
 * k4_op_masked_quantiles replaces the depth video's range, run_sr.py:1459-1461:
 *   depths_vis = depths * (1 - bgmaps) + bgmaps;  dmin, dmax = np.percentile(depths_vis[bgmaps < 0.1], q=[5, 95])
 * d_depth, d_bgmap: n x H x W fp32, element (f, y, x) at f * strides[0] + y * strides[1] + x * strides[2] (host arrays of
 * element strides, so [n, H, W, 1] arrays and views are read in place).  depths_vis is formed in fp32 with one rounding
 * per operation, the selection is bgmap < 0.1f.  h_q: HOST array of the two quantiles as fractions, q / 100 as numpy's
 * percentile computes it (np.true_divide(q, np.float32(100)), fp64), each in [0, 1].  d_quantiles (2 device doubles)
 * receives np.percentile's 'linear' values bit for bit: the order statistics are exact (a radix select on the fp32
 * keys: integer counts only) and the interpolation is numpy's _lerp.  A NaN among the selected values gives NaN, as
 * numpy.  d_count (one device int64) receives the number of selected values; with 0 the quantiles are NaN (numpy
 * raises).  -0.0 orders before +0.0 (numpy treats them as equal, so a quantile that falls on a tie between them may
 * carry either sign there).  The workspace holds k4_op_masked_quantiles_workspace_bytes(n, H, W) bytes (0 for an
 * invalid shape), 16-byte aligned.  Caller's stream, no host sync; the result is bitwise reproducible.
 * A NULL pointer, n, H or W below 1, n * H above 2^31 - 1, a quantile outside [0, 1] or NaN, or a misaligned pointer:
 * K4_ERR_INVALID_ARG; a workspace smaller than the size: K4_ERR_WORKSPACE.
 *
 * k4_op_depth_video_u8 replaces run_sr.py:1462-1463's frames:
 *   to8b(plt.get_cmap('rainbow')(1 - np.clip((depths_vis - dmin) / (dmax - dmin), 0, 1)).squeeze()[..., :3])
 * with render_video_flipy / render_video_rot90 (render.py's _post) applied.  d_range: the two device doubles dmin, dmax
 * (k4_op_masked_quantiles' d_quantiles).  The normalisation is fp64, as numpy 2 computes float32 - float64.  Colormap
 * index: i = trunc(256 x), 256 -> 255; NaN x (dmax == dmin at depths_vis == dmin, or NaN data) is the colormap's 'bad'
 * colour, (0, 0, 0).  h_lut: HOST u8 [256][3], to8b of the colormap's rgb table.  d_out: u8 [n, H', W', 3] contiguous,
 * H' x W' = H x W for even rot90 and W x H for odd; frame f is rot90(flip(frame f, axis 0) if flip_y, rot90 mod 4).
 * n, H or W outside 1 .. 65535, flip_y not 0 / 1, a NULL or misaligned pointer: K4_ERR_INVALID_ARG.
 *
 * k4_op_frame_u8 replaces utils.to8b (lib/utils.py:20) of one rendered frame, (255 * np.clip(x, 0, 1)).astype(uint8)
 * with the product in fp32, with the same flip / rot90.  d_rgb: H x W x 3 fp32, element (y, x, c) at y * strides[0] +
 * x * strides[1] + c * strides[2], e.g. a [3, H, W] decoder output read as permute(1, 2, 0).  NaN gives 0.
 * d_out: u8 [H', W', 3] contiguous.  H or W outside 1 .. 65535, flip_y not 0 / 1, a NULL or misaligned pointer:
 * K4_ERR_INVALID_ARG.
 */
/* Replaces: np.percentile(depths_vis[bgmaps < 0.1], q=[5, 95]) (run_sr.py:1460) -- the workspace of
 * k4_op_masked_quantiles. */
K4_API size_t k4_op_masked_quantiles_workspace_bytes(int64_t n, int64_t H, int64_t W);
/* Replaces: depths_vis = depths * (1-bgmaps) + bgmaps; np.percentile(depths_vis[bgmaps < 0.1], q=[5, 95])
 * (run_sr.py:1459-1460). */
K4_API int k4_op_masked_quantiles(const float* d_depth, const float* d_bgmap, int64_t n, int64_t H, int64_t W,
                                  const int64_t depth_strides[3], const int64_t bgmap_strides[3], const double h_q[2],
                                  double* d_quantiles, int64_t* d_count, void* d_workspace, size_t workspace_bytes,
                                  k4_stream_t stream);
/* Replaces: to8b(plt.get_cmap('rainbow')(1 - np.clip((depths_vis - dmin) / (dmax - dmin), 0, 1)).squeeze()[..., :3])
 * (run_sr.py:1461-1463), flipped / rotated as render_viewpoints' render_video_flipy / render_video_rot90. */
K4_API int k4_op_depth_video_u8(const float* d_depth, const float* d_bgmap, int64_t n, int64_t H, int64_t W,
                                const int64_t depth_strides[3], const int64_t bgmap_strides[3], const double* d_range,
                                const uint8_t* h_lut, int32_t flip_y, int32_t rot90, uint8_t* d_out, k4_stream_t stream);
/* Replaces: utils.to8b (lib/utils.py:20) of the video frames (run_sr.py:1457-1458), flipped / rotated. */
K4_API int k4_op_frame_u8(const float* d_rgb, int64_t H, int64_t W, const int64_t strides[3], int32_t flip_y, int32_t rot90,
                          uint8_t* d_out, k4_stream_t stream);

/* The passes of k4_op_masked_quantiles one by one, for frames spread over several GPUs (or any set of shares).  The
 * select's three passes each read a histogram of integer counts, and integer counts add exactly, so per pass p = 0, 1, 2:
 *   1. every share zeroes an int64 histogram of K4_MASKED_QUANTILES_HIST_LEN entries and adds its frames into it with
 *      k4_op_masked_quantiles_hist(p, ...);
 *   2. the caller sums the shares' histograms element by element (e.g. one all-reduce);
 *   3. every share runs k4_op_masked_quantiles_select(p, ...) on the sum.
 * Every share then holds the same state for pass p + 1, and after pass 2 d_quantiles and d_count are bit for bit
 * k4_op_masked_quantiles' over all the shares' frames, in the same layout.  The histogram's last two entries hold the
 * count and the NaN count of pass 0 (zero in passes 1 and 2).  The workspace holds the per-pass state:
 * k4_op_masked_quantiles_pass_workspace_bytes() bytes, 16-byte aligned, kept by the caller from pass 0 to pass 2; it needs
 * no initialisation.
 * k4_op_masked_quantiles_hist ADDS into d_hist (int64 counts, 8-byte aligned).  n == 0 (a share without frames) is valid
 * and launches nothing; d_depth and d_bgmap may then be NULL.  The select takes the same h_q on every pass (pass 0 reads
 * it) and writes d_quantiles / d_count in pass 2.  Caller's stream, no host sync.
 * A pass outside 0 .. 2, a NULL pointer, n below 0, H or W below 1, n * H above 2^31 - 1, a quantile outside [0, 1] or
 * NaN, or a misaligned pointer: K4_ERR_INVALID_ARG; a workspace smaller than the size: K4_ERR_WORKSPACE. */
#define K4_MASKED_QUANTILES_HIST_LEN (4 * 2048 + 2)
/* Replaces: np.percentile(depths_vis[bgmaps < 0.1], q=[5, 95]) (run_sr.py:1460) over frames spread over GPUs -- the
 * per-pass state of k4_op_masked_quantiles_hist / _select. */
K4_API size_t k4_op_masked_quantiles_pass_workspace_bytes(void);
/* Replaces: np.percentile(depths_vis[bgmaps < 0.1], q=[5, 95]) (run_sr.py:1459-1460) over frames spread over GPUs --
 * one share's histogram of pass `pass`. */
K4_API int k4_op_masked_quantiles_hist(int32_t pass, const float* d_depth, const float* d_bgmap, int64_t n, int64_t H,
                                       int64_t W, const int64_t depth_strides[3], const int64_t bgmap_strides[3],
                                       int64_t* d_hist, const void* d_workspace, size_t workspace_bytes,
                                       k4_stream_t stream);
/* Replaces: np.percentile(depths_vis[bgmaps < 0.1], q=[5, 95]) (run_sr.py:1460) over frames spread over GPUs -- the
 * select of pass `pass` on the summed histogram. */
K4_API int k4_op_masked_quantiles_select(int32_t pass, const int64_t* d_hist, const double h_q[2], double* d_quantiles,
                                         int64_t* d_count, void* d_workspace, size_t workspace_bytes, k4_stream_t stream);

/* ------------------------------------------------------------------------------------------------
 * Testing.  Entry points for the test suite, not for renderers: they replace no reference interface and may change
 * with the kernels they expose.
 *
 * k4_testing_conv3x3: ONE VC-Decoder convolution layer, packed by the same weight packers k4_srnet_create uses and run
 * by the same dispatcher as k4_srnet_forward, so that a test can compare a single layer with a reference.
 *   d_weight [cout][cin][3][3], d_bias [cout] fp32; cout <= 64, cin <= 192.  Inputs are padded to cin_pad = 32 *
 *   ceil(cin / 32) channels (the decoder's NHWC layouts); the layer computes npad = 16 | 32 | 64 output channels
 *   (cout rounded up), the ones beyond cout with zero weights and bias.
 *   d_src: fp16 NHWC, channels [src_c0, src_c0 + cin_pad) of src_cstride per pixel (both multiples of 8), H x W pixels.
 *   upsample2x: "nearest x2, then conv" in its sub-pixel form; the output is 2H x 2W (modes 0-4 only).
 *   Output rows [y_lo, y_hi) of the H x W iteration grid (the source grid when upsample2x), 0 <= y_lo < y_hi <= H.
 *   mode (the epilogues of csrc/k4_sr.cu, pixels p of the output grid, fp32 per-pixel buffers have 64 channels):
 *     0 dst_h[p][dst_c0 + c] = fp16(act(conv + b)), act = LeakyReLU(lrelu) if lrelu > 0
 *     1 dst_f = (conv + b) * scale + add_f
 *     2 dst_h = fp16((conv + b) + add_f)
 *     3 dst_f = dst_f2 = conv + b                          (dst_f2 may be NULL)
 *     4 d_out_nchw[c * out_plane_stride + (y - crop_y0) * out_row_stride + (x - crop_x0)] = conv + b for c < n_valid and
 *       (y, x) inside [crop_y0, crop_y1) x [crop_x0, crop_x1)
 *     5 dst_h = fp16(sft(act(conv + b)))                                            (cout 32 or 64)
 *     6 t = (conv + b) * scale [+ add_f]; dst_f [, dst_f2] = t; dst_h2 = fp16(sft(t))           (cout 32 or 64)
 *     7 t as in 6; u = sft(t) * scale2 + add_f2; dst_f = u; dst_h2 = fp16(sft2(u))               (cout 64)
 *   sft(x) = x * (scale + 1) + shift of an SFT layer with condition d_cond16 (fp16 [H*W][32]); h_sft / h_sft2: HOST
 *   arrays of the 8 device pointers of its 1x1 convolutions in k4_srnet_desc order (scale_conv0 w, b, scale_conv1 w, b,
 *   shift_conv0 w, b, shift_conv1 w, b).
 *   kernel: K4_CONV_KERNEL_AUTO picks what k4_srnet_forward would (environment switches included); any other value
 *   forces that kernel, which runs or the call returns K4_ERR_UNSUPPORTED.  *kernel_used (may be NULL) receives the
 *   kernel that ran.  Arguments are checked before any CUDA call (K4_ERR_INVALID_ARG).  The call synchronises `stream`.
 */
enum { K4_CONV_KERNEL_AUTO = 0,            /* the decoder's own choice                           */
       K4_CONV_KERNEL_WS_TMA = 1,          /* conv3x3_ws_kernel, TMA producer                    */
       K4_CONV_KERNEL_WS_CPASYNC = 2,      /* conv3x3_ws_kernel, cp.async producer               */
       K4_CONV_KERNEL_K64 = 3 };           /* conv3x3_k64_kernel (cin_pad 64, npad 16 or 64)     */

typedef struct k4_conv_test_args {
    const float* d_weight;
    const float* d_bias;
    int32_t cout, cin;
    const void* d_src;                     /* fp16 */
    int32_t src_cstride, src_c0;
    int32_t H, W;
    int32_t upsample2x;
    int32_t mode;
    float lrelu, scale, scale2;
    int32_t y_lo, y_hi;
    void* d_dst_h;                         /* fp16 */
    int32_t dst_cstride, dst_c0;
    float* d_dst_f;
    float* d_dst_f2;
    const float* d_add_f;
    const float* d_add_f2;
    void* d_dst_h2;                        /* fp16 */
    int32_t dst2_cstride, dst2_c0;
    float* d_out_nchw;
    int32_t n_valid, reserved0;
    int64_t out_plane_stride, out_row_stride;
    int32_t crop_y0, crop_y1, crop_x0, crop_x1;
    const void* d_cond16;                  /* fp16 */
    const float* const* h_sft;
    const float* const* h_sft2;
    int32_t kernel;
    int32_t reserved1;
} k4_conv_test_args;
K4_API int k4_testing_conv3x3(const k4_conv_test_args* args, int32_t* kernel_used, k4_stream_t stream);

/*
 * k4_testing_condnet / k4_testing_sft: the decoder's per-pixel MLPs -- CondNet and one SFT layer as its own pass -- packed
 * by the packers k4_srnet_create uses and run by the decoder's own launchers, so that a test can compare them element
 * by element with a reference.
 *   kernel: K4_SR_KERNEL_AUTO picks what k4_srnet_forward would (K4_CONDNET_FP32, read per call; K4_SFT_FP32, latched at
 *   the first SFT pass of a process); MMA / FP32 force condnet_mma_kernel / sft_mma_kernel or condnet_kernel /
 *   sft_kernel, which run every valid shape.  *kernel_used (may be NULL) receives the kernel that ran, -1 on error.
 *   Arguments are checked before any CUDA call (K4_ERR_INVALID_ARG).  The calls synchronise `stream`.
 *
 * k4_testing_condnet: CondNet (conv3x3 num_cond -> 64, LeakyReLU 0.2, 1x1 64 -> 64, LeakyReLU, 1x1 64 -> 64, LeakyReLU,
 * 1x1 64 -> 32) on rows [y_lo, y_hi) of an H x W condition map, zero padded at the map's border.
 *   num_cond: 0 .. 64, 0 meaning 1 (other values: K4_ERR_INVALID_ARG).  MMA is condnet_mma_kernel at num_cond 1 and
 *   condnet_wide_mma_kernel above.
 *   h_condnet: HOST array of the 8 device pointers in k4_srnet_desc order (CondNet.0 w [64][num_cond][3][3], b [64], .2 w
 *   [64][64], b, .4 w [64][64], b, .6 w [32][64], b [32]).  d_cond_in fp32 [num_cond][H][W].  d_cond_out fp32 [H*W][32]
 *   and d_cond16 (fp16 [H*W][32], the operand of the fused SFT epilogues, NULL to skip) receive the window's rows only.
 *
 * k4_testing_sft: one SFT layer, y = x * (scale + 1) + shift, on pixels [p0, p0 + P) of per-pixel buffers.
 *   h_sft: HOST array of the layer's 8 device pointers (the h_sft convention of k4_conv_test_args); cout 32 or 64.
 *   d_cond fp32 [..][32].  Input: d_x_f (fp32 [..][64], channels [0, cout)) or d_x_h (fp16, channels [xh_c0, xh_c0 +
 *   cout) of xh_cstride, both even), not both.  Output: d_dst_h (fp16, channels [dst_c0, dst_c0 + cout) of dst_cstride,
 *   both multiples of 8; may be d_x_h) or d_dst_f (fp32 [..][64]) = y * res_scale + d_res_f, where d_res_f may equal
 *   d_dst_f (the RRDB tail), not both.
 */
enum { K4_SR_KERNEL_AUTO = 0,              /* the decoder's own choice                           */
       K4_SR_KERNEL_MMA = 1,               /* condnet_mma_kernel / sft_mma_kernel (mma.sync)     */
       K4_SR_KERNEL_FP32 = 2 };            /* condnet_kernel / sft_kernel (fp32 FFMA)            */

typedef struct k4_condnet_test_args {
    const float* const* h_condnet;
    const float* d_cond_in;
    int32_t H, W;
    int32_t y_lo, y_hi;
    float* d_cond_out;
    void* d_cond16;                        /* fp16, or NULL */
    int32_t kernel;
    int32_t num_cond;                      /* condition channels, 0 .. 64 (0: 1) */
} k4_condnet_test_args;
K4_API int k4_testing_condnet(const k4_condnet_test_args* args, int32_t* kernel_used, k4_stream_t stream);

typedef struct k4_sft_test_args {
    const float* const* h_sft;
    int32_t cout;
    int32_t kernel;
    const float* d_cond;
    const float* d_x_f;
    const void* d_x_h;                     /* fp16 */
    int32_t xh_cstride, xh_c0;
    void* d_dst_h;                         /* fp16 */
    int32_t dst_cstride, dst_c0;
    float* d_dst_f;
    const float* d_res_f;
    float res_scale;
    int32_t reserved0;
    int64_t p0, P;
} k4_sft_test_args;
K4_API int k4_testing_sft(const k4_sft_test_args* args, int32_t* kernel_used, k4_stream_t stream);

/*
 * k4_testing_srnet_forward_upto: k4_srnet_forward_roi (same arguments, same code) that returns after its first
 * `stop_after` steps, so that a test can read the workspace as the real forward left it after any layer.  A step is one
 * layer as the forward enqueues it: the NCHW -> NHWC input conversion, CondNet, one convolution (with the SFT layers
 * fused into its epilogue, if any; conv_up1 / conv_up2 are one step of four phase launches each) or one standalone SFT
 * pass.  The steps that ran are enqueued on `stream` (not synchronised), exactly as the full forward enqueues them.
 *   steps[0 .. min(*n_steps, max_steps)) receive the descriptors of the steps that ran, in order; *n_steps their count
 *   (stop_after, or all steps when stop_after is larger).  *ws receives the byte offsets of the workspace buffers of
 *   an h x w tile of `net` (the layout every k4_srnet_forward* call uses).
 *   Arguments are checked before any CUDA call (K4_ERR_INVALID_ARG, *n_steps 0).
 */
enum { K4_SR_STEP_INPUT = 0,               /* in16 = fp16 NHWC32 of d_x                          */
       K4_SR_STEP_CONDNET = 1,             /* cond32 (and cond16 when SFT is fused)              */
       K4_SR_STEP_CONV_FIRST = 2,
       K4_SR_STEP_RDB_CONV = 3,            /* conv `conv` (0..4) of dense block `dense` of RRDB `block` */
       K4_SR_STEP_SFT0 = 4,                /* standalone SFT passes: sft0 / sft1 of a dense block, */
       K4_SR_STEP_SFT1 = 5,
       K4_SR_STEP_SFT_RRDB = 6,            /*   the RRDB tail's sft0 (with its residual),        */
       K4_SR_STEP_SFT_BODY = 7,            /*   sftbody                                          */
       K4_SR_STEP_CONV_BODY = 8,
       K4_SR_STEP_UP1 = 9,
       K4_SR_STEP_UP2 = 10,
       K4_SR_STEP_HR = 11,
       K4_SR_STEP_LAST = 12 };

typedef struct k4_sr_step {
    int32_t kind;                          /* K4_SR_STEP_*                                       */
    int32_t block, dense, conv;            /* RRDB, dense block in it, conv in that (-1: none)   */
    int32_t fused;                         /* 1: SFT layer(s) applied in this convolution's epilogue */
} k4_sr_step;

typedef struct k4_sr_ws_layout {
    uint64_t in16, cond32, cond16, feat, trunk_a, trunk_b, cat, cat2, sbody, bf, up1, up2, hr, total;   /* byte offsets */
} k4_sr_ws_layout;

K4_API int k4_testing_srnet_forward_upto(const k4_srnet* net, const float* d_x, const float* d_cond, int32_t h, int32_t w,
                                         int32_t keep_y0, int32_t keep_y1, int32_t keep_x0, int32_t keep_x1,
                                         float* d_out, int64_t out_plane_stride, int64_t out_row_stride,
                                         void* d_workspace, size_t workspace_bytes, int32_t stop_after,
                                         k4_sr_step* steps, int32_t max_steps, int32_t* n_steps, k4_sr_ws_layout* ws,
                                         k4_stream_t stream);

/*
 * k4_testing_rgbnet: the scene's packed rgbnet on rows the caller supplies, run by the marchers' own device code for one
 * K4_MLP_* mode, so that a test can compare the colour MLP sample by sample with a reference.
 *   d_x [n][dim0]: model-layout MLP inputs, the vectors the reference's rgbnet receives (rgb_feat: the k0 channels fed to
 *   the MLP, the MPI position code, the view embedding; lib/dvgo.py:407-412, lib/dmpigo.py:374).  d_diffuse [n][3]: the
 *   diffuse logits k0[0:3] of a DirectVoxGO model with rgbnet_direct=False, NULL for every other model.  d_w [n]: sample
 *   weights.  d_owner [n]: the row's owner inside its group.
 *   Rows form groups of G consecutive rows (*group_rows receives G; the last group may be partial):
 *     K4_MLP_TCGEN05_WS     G = 128 (also for its alias K4_MLP_TCGEN05): one warpgroup batch of mlp_batch_wgmma; the
 *                           rows are written into a ring tile through
 *                           the column map of the scene's K4_WS_CFG_LIST entry, as fp16 with saturation
 *     K4_MLP_F16 / _F16X3   G = 32: one warp's MmaWarpCtx, rows appended as the marcher appends them, flushed at 32 rows
 *                           and at the end of the group
 *     K4_MLP_FP32           G = 32: mlp_fp32, accumulated per owner in row order
 *   Owners are in [0, G); only their low log2(G) bits are read.
 *   d_racc [ceil(n / G)][G][3]: racc[g][j][c] = sum over the rows of group g with owner j of w * sigmoid(logit_c (+ diffuse_c)),
 *   what the marchers accumulate into a ray.
 *   A mode the scene's shape has no build for returns K4_ERR_UNSUPPORTED; nothing falls back to another mode.  Arguments
 *   are checked before any CUDA call (K4_ERR_INVALID_ARG).  The call synchronises `stream`.
 */
typedef struct k4_rgbnet_test_args {
    int32_t mode;                          /* K4_MLP_*                                           */
    int32_t reserved0;
    int64_t n;                             /* rows, 1 .. 2^24                                    */
    const float* d_x;
    const float* d_diffuse;
    const float* d_w;
    const int32_t* d_owner;
    float* d_racc;
} k4_rgbnet_test_args;
K4_API int k4_testing_rgbnet(const k4_scene* scene, const k4_rgbnet_test_args* args, int32_t* group_rows, k4_stream_t stream);

/*
 * k4_testing_ws_row_layout: the A-row layout the warp-specialised marcher's kernels are compiled with for the
 * K4_WS_CFG_LIST entry `config` (csrc/k4_ws_cfgs.h), so that a test can check it without a GPU.  out[4] (host):
 *   out[0]  the config's inputs per row (its dim0: the padded per-sample features, then the view embedding)
 *   out[1]  K of layer 1 (dim0 rounded up to 16)
 *   out[2]  the first of the two columns that hold fp16 1.0 in every row and layer 1's bias hi / lo in W1, so that the
 *           bias rides inside layer 1's K; -1 where they do not fit below out[1] and layer 1 adds its bias with one more
 *           MMA against a tile of ones
 *   out[3]  1 if the marcher's row store writes those ones with every row, 0 if they are written once per ring
 * An id that is not in the list returns K4_ERR_INVALID_ARG with out zeroed.  Needs no device.
 */
K4_API int k4_testing_ws_row_layout(int32_t config, int32_t* out);

/*
 * k4_testing_march_phases: k4_render_rays in mode K4_MLP_TCGEN05_WS, run by the profiled instantiation of the
 * warp-specialised marcher.  It computes what the production kernel computes and, besides, where each warpgroup's SM
 * cycles go: thread 0 of every warpgroup reads the SM clock at each phase boundary and charges the cycles since the
 * previous boundary to the phase that ended, so a warpgroup's phases add up to its elapsed cycles.
 *   d_phases [n_ctas][4][K4_PHASE_SLOTS] uint64: CTA c, warpgroup g (0, 1 marchers; 2, 3 the MLP groups of marchers
 *   0, 1), slots K4_PH_* below.  max_ctas: CTAs d_phases has room for; the launch has min(SM count, ceil(tiles / 2))
 *   CTAs, and a launch that needs more returns K4_ERR_INVALID_ARG before it starts.  *n_ctas receives the CTA count.
 *   Every other argument has k4_render_rays' meaning; args->mlp_mode must be K4_MLP_TCGEN05_WS.  Arguments are checked
 *   before any CUDA call (K4_ERR_INVALID_ARG), except the CTA count, which needs the device's SM count.  Does not
 *   synchronise `stream`.
 */
enum { K4_PHASE_SLOTS = 8 };
enum { K4_PH_ELAPSED = 0,                  /* every warpgroup: cycles from the staged weights to its exit              */
       /* marcher warpgroups */
       K4_PH_M_SETUP = 1,                  /*   tile fetch, ray setup, exit                                            */
       K4_PH_M_MARCH = 2,                  /*   stepping, gathers, appending rows to the ring                          */
       K4_PH_M_RENDEZVOUS = 3,             /*   warpgroup barriers between marching rounds and before a submit         */
       K4_PH_M_WAIT_DONE = 4,              /*   submit: waiting until the MLP group has consumed the previous batch    */
       K4_PH_M_DRAIN = 5,                  /*   tile end: waiting until every batch of the tile is consumed            */
       K4_PH_M_STORE = 6,                  /*   tile end: storing the rays                                             */
       K4_PH_M_BATCHES = 7,                /*   count: batches submitted                                               */
       /* MLP warpgroups */
       K4_PH_L_WAIT_FULL = 1,              /*   waiting for a batch (FULL), or for the exit                            */
       K4_PH_L_L1 = 2,                     /*   waiting for layer 1's MMAs (issue to retire)                           */
       K4_PH_L_L2 = 3,
       K4_PH_L_L3 = 4,
       K4_PH_L_REPACK = 5,                 /*   accumulators -> ReLU'd fp16 operands of the next layer                 */
       K4_PH_L_EPILOGUE = 6,               /*   sigmoid, weight and shared-memory atomics into the rays                */
       K4_PH_L_BATCHES = 7 };              /*   count: batches consumed                                                */
K4_API int k4_testing_march_phases(const k4_scene* scene, const k4_render_args* args,
                                   const float* d_rays_o, const float* d_rays_d, const float* d_viewdirs,
                                   int64_t n_rays, const k4_render_out* out, void* d_workspace, size_t workspace_bytes,
                                   uint64_t* d_phases, int32_t max_ctas, int32_t* n_ctas, k4_stream_t stream);

/*
 * k4_testing_skip_field: a copy of the scene's empty-space-skipping field, so that a test can compare it with an
 * independent distance transform.  The field covers the occupancy mask in cells of 4 x 4 x 4 mask voxels (the last cell
 * of an axis may be partial): cdims[a] = ceil(mask_size[a] / 4).  Cell (i, j, k) is stored at d_out[(i * cdims[1] + j) *
 * cdims[2] + k] and holds the Chebyshev distance, in cells, to the nearest cell that contains an occupied voxel: 0 for
 * such a cell, and 49 for every cell with no occupied cell within 48 cells (also every cell of an empty mask).
 *   d_out: device buffer of n bytes, n >= cdims[0] * cdims[1] * cdims[2].  cdims (host) receives the cell dimensions.
 *   A scene without the field returns K4_ERR_UNSUPPORTED with cdims zeroed: DirectContractedVoxGO, a scene created with
 *   K4_NO_SKIP set, and one whose mask has a single voxel on some axis (xyz2ijk_scale 0 there: every point maps to that
 *   voxel, and the skip geometry needs 1 / scale).  Arguments are checked before any CUDA call (K4_ERR_INVALID_ARG).  The copy
 *   is a synchronous cudaMemcpy: the call returns when d_out holds the field.
 */
K4_API int k4_testing_skip_field(const k4_scene* scene, uint8_t* d_out, int64_t n, int32_t cdims[3]);

/*
 * k4_testing_lpips_stage: one image through k4_lpips_forward's trunk up to `stage`, so that a test can compare each
 * layer with a reference.  Stage 0 is the scaled input (2x - 1, then the scaling layer); stage s >= 1 is the output of
 * the trunk's s-th operation, in the order of torchvision's features: VGG16 17 (conv + ReLU, or 2x2 max-pool), AlexNet
 * 7 (conv + ReLU, or 3x3 / 2 max-pool).  out_shape (host) receives the stored (h, w, c); d_out (NULL: only the shape)
 * receives the stage as h x w x c contiguous: for VGG fp16 with c = 3 C, the pairs hi = fp16(x), lo = fp16(x - hi) of
 * the C channels as [hi | lo | hi] (stage 0: 32 channels, hi, lo, hi of the image's 3, then zeros), for AlexNet fp32
 * with c = C.
 * Image, strides, size and workspace as k4_lpips_forward (one image's half of the workspace is used).  Arguments are
 * checked before any CUDA call (K4_ERR_INVALID_ARG, K4_ERR_WORKSPACE).  Caller's stream, no host sync.
 */
K4_API int k4_testing_lpips_stage(const k4_lpips* net, const float* d_img, const int64_t strides[3], int64_t H, int64_t W,
                                  int32_t stage, void* d_out, int64_t out_shape[3], void* d_workspace, size_t workspace_bytes,
                                  k4_stream_t stream);

/*
 * k4_testing_png_code_lengths: the length-limited Huffman code lengths k4_png_encode gives a histogram (package-merge,
 * the encoder's own device routine in one CTA, as for its literal / length, distance and code-length codes), so that a
 * test can compare them with an optimal length-limited code on histograms no frame produces.
 *   d_freq: device int32 [n] counts, 1 <= n <= 286; a count <= 0 gets length 0.  maxbits: 1..15.
 *   d_len: device uint8 [n], receives the lengths.  Counts the routine cannot code -- more non-zero counts than
 *   2^maxbits, or a total of 2^31 - 1 or more -- give 0xff for every length.
 * Arguments are checked before any CUDA call (K4_ERR_INVALID_ARG).  Caller's stream, no host sync.
 */
K4_API int k4_testing_png_code_lengths(const int32_t* d_freq, int32_t n, int32_t maxbits, uint8_t* d_len,
                                       k4_stream_t stream);

/*
 * PNG files of uint8 RGB frames on the device, for run_sr.py --render_test's imageio.imwrite of every frame
 * (csrc/k4_png.cu; DESIGN.md section 3.10).
 *   d_rgb: u8 [H, W, 3] contiguous (frame_u8 / render_frame_4k(out_u8=True)'s layout).
 *   d_out: receives the whole file (signature, IHDR, one IDAT, IEND); out_capacity >= k4_png_encode_bound(H, W).
 *   d_len: one device int64 (8-byte aligned), receives the file's length in bytes.
 *   d_workspace: k4_png_workspace_bytes(H, W) bytes, 256-byte aligned.
 * Each row is filtered with the least sum of |byte as int8| of the five PNG filters (ties to the lowest type); the
 * filtered stream is cut into segments of K4_PNG_SEG bytes, each one dynamic-Huffman block (code lengths <= 15) with
 * back-references up to 32 KiB before its start, or one stored block when that is not larger; a dynamic segment
 * other than the last ends with an empty stored block (a sync flush).  The output is a fixed function of the frame.
 * The bound is the all-stored file: H (1 + 3 W) + 5 ceil(H (1 + 3 W) / K4_PNG_SEG) + 63 bytes.  Frames whose bound
 * exceeds 2^31 - 1 (one IDAT chunk) give 0 from both size functions.
 * A NULL pointer, H or W < 1, too large a frame, out_capacity below the bound, too small or misaligned a workspace:
 * K4_ERR_INVALID_ARG before any CUDA call.  Caller's stream, no host sync, no allocation.
 */
#define K4_PNG_SEG 32768
K4_API size_t k4_png_encode_bound(int64_t H, int64_t W);
K4_API size_t k4_png_workspace_bytes(int64_t H, int64_t W);
K4_API int k4_png_encode(const uint8_t* d_rgb, int64_t H, int64_t W, uint8_t* d_out, size_t out_capacity, int64_t* d_len,
                         void* d_workspace, size_t workspace_bytes, k4_stream_t stream);

#ifdef __cplusplus
}
#endif
#endif /* K4NERF_H_ */
