"""ctypes binding of libk4nerf.so -- the exact declarations of include/k4nerf.h."""
import ctypes as C
import os

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_HERE, 'libk4nerf.so')

K4_OK = 0
K4_KIND_DVGO, K4_KIND_DMPIGO, K4_KIND_DCVGO = 0, 1, 2
K4_MLP_FP32, K4_MLP_F16, K4_MLP_F16X3, K4_MLP_TCGEN05, K4_MLP_TCGEN05_WS = 0, 1, 2, 3, 4
K4_ACT_RELU, K4_ACT_GAUSS, K4_ACT_LKRELU = 0, 1, 2
K4_MAX_MLP_LAYERS = 8
K4_MAX_PEERS = 8
MLP_MODES = {'fp32': K4_MLP_FP32, 'f16': K4_MLP_F16, 'f16x3': K4_MLP_F16X3, 'tcgen05': K4_MLP_TCGEN05,
             'tc': K4_MLP_TCGEN05, 'ws': K4_MLP_TCGEN05_WS}


class SceneDesc(C.Structure):
    _fields_ = [
        ('kind', C.c_int32), ('world_size', C.c_int32 * 3), ('k0_dim', C.c_int32), ('mask_size', C.c_int32 * 3),
        ('xyz_min', C.c_float * 3), ('xyz_max', C.c_float * 3),
        ('xyz2ijk_scale', C.c_float * 3), ('xyz2ijk_shift', C.c_float * 3),
        ('act_shift', C.c_float), ('voxel_size', C.c_float), ('voxel_size_ratio', C.c_float),
        ('fast_color_thres', C.c_float),
        ('max_world_size', C.c_int32), ('mpi_depth', C.c_int32),
        ('rgbnet_depth', C.c_int32), ('rgbnet_width', C.c_int32), ('rgbnet_direct', C.c_int32),
        ('viewbase_pe', C.c_int32), ('spatial_pe', C.c_int32), ('rgbnet_act', C.c_int32),
        ('d_density', C.c_void_p), ('d_k0', C.c_void_p), ('d_mask', C.c_void_p), ('d_act_shift_grid', C.c_void_p),
        ('d_rgbnet_weight', C.c_void_p * K4_MAX_MLP_LAYERS), ('d_rgbnet_bias', C.c_void_p * K4_MAX_MLP_LAYERS),
        ('scene_center', C.c_float * 3), ('scene_radius', C.c_float * 3), ('bg_len', C.c_float), ('world_len', C.c_int32),
        ('rgbnet_act_param', C.c_float),
    ]


class RenderArgs(C.Structure):
    _fields_ = [
        ('near_', C.c_float), ('far_', C.c_float), ('stepsize', C.c_float), ('bg', C.c_float),
        ('render_depth', C.c_int32), ('mlp_mode', C.c_int32), ('image_w', C.c_int32), ('image_h', C.c_int32),
        ('d_t_list', C.c_void_p), ('n_t', C.c_int32), ('dist_thres', C.c_float),
    ]


class RenderOut(C.Structure):
    _fields_ = [
        ('d_rgb_marched', C.c_void_p), ('d_depth', C.c_void_p), ('d_alphainv_last', C.c_void_p),
        ('d_ray_stats', C.c_void_p), ('d_t_minmax', C.c_void_p), ('d_counters', C.c_void_p),
    ]


class FrameDst(C.Structure):
    _fields_ = [
        ('n_dst', C.c_int32), ('rank', C.c_int32), ('world', C.c_int32), ('frame_w', C.c_int32),
        ('n_full', C.c_int64), ('d_frame', C.c_void_p * K4_MAX_PEERS),
    ]


class SrnetDesc(C.Structure):
    _fields_ = [
        ('n_in_colors', C.c_int32), ('scale', C.c_int32), ('num_feat', C.c_int32), ('num_block', C.c_int32),
        ('num_grow_ch', C.c_int32), ('num_cond', C.c_int32), ('n_params', C.c_int32), ('reserved0', C.c_int32),
        ('h_params', C.POINTER(C.c_void_p)),
    ]


K4_CONV_KERNEL_AUTO, K4_CONV_KERNEL_WS_TMA, K4_CONV_KERNEL_WS_CPASYNC, K4_CONV_KERNEL_K64 = 0, 1, 2, 3


class ConvTestArgs(C.Structure):
    """k4_conv_test_args: one decoder convolution for the test suite (k4_testing_conv3x3)."""
    _fields_ = [
        ('d_weight', C.c_void_p), ('d_bias', C.c_void_p), ('cout', C.c_int32), ('cin', C.c_int32),
        ('d_src', C.c_void_p), ('src_cstride', C.c_int32), ('src_c0', C.c_int32), ('H', C.c_int32), ('W', C.c_int32),
        ('upsample2x', C.c_int32), ('mode', C.c_int32), ('lrelu', C.c_float), ('scale', C.c_float), ('scale2', C.c_float),
        ('y_lo', C.c_int32), ('y_hi', C.c_int32),
        ('d_dst_h', C.c_void_p), ('dst_cstride', C.c_int32), ('dst_c0', C.c_int32),
        ('d_dst_f', C.c_void_p), ('d_dst_f2', C.c_void_p), ('d_add_f', C.c_void_p), ('d_add_f2', C.c_void_p),
        ('d_dst_h2', C.c_void_p), ('dst2_cstride', C.c_int32), ('dst2_c0', C.c_int32),
        ('d_out_nchw', C.c_void_p), ('n_valid', C.c_int32), ('reserved0', C.c_int32),
        ('out_plane_stride', C.c_int64), ('out_row_stride', C.c_int64),
        ('crop_y0', C.c_int32), ('crop_y1', C.c_int32), ('crop_x0', C.c_int32), ('crop_x1', C.c_int32),
        ('d_cond16', C.c_void_p), ('h_sft', C.POINTER(C.c_void_p)), ('h_sft2', C.POINTER(C.c_void_p)),
        ('kernel', C.c_int32), ('reserved1', C.c_int32),
    ]


K4_SR_KERNEL_AUTO, K4_SR_KERNEL_MMA, K4_SR_KERNEL_FP32 = 0, 1, 2


class CondnetTestArgs(C.Structure):
    """k4_condnet_test_args: CondNet on a row window for the test suite (k4_testing_condnet)."""
    _fields_ = [
        ('h_condnet', C.POINTER(C.c_void_p)), ('d_cond_in', C.c_void_p), ('H', C.c_int32), ('W', C.c_int32),
        ('y_lo', C.c_int32), ('y_hi', C.c_int32), ('d_cond_out', C.c_void_p), ('d_cond16', C.c_void_p),
        ('kernel', C.c_int32), ('num_cond', C.c_int32),
    ]


class SftTestArgs(C.Structure):
    """k4_sft_test_args: one SFT layer as its own pass for the test suite (k4_testing_sft)."""
    _fields_ = [
        ('h_sft', C.POINTER(C.c_void_p)), ('cout', C.c_int32), ('kernel', C.c_int32), ('d_cond', C.c_void_p),
        ('d_x_f', C.c_void_p), ('d_x_h', C.c_void_p), ('xh_cstride', C.c_int32), ('xh_c0', C.c_int32),
        ('d_dst_h', C.c_void_p), ('dst_cstride', C.c_int32), ('dst_c0', C.c_int32),
        ('d_dst_f', C.c_void_p), ('d_res_f', C.c_void_p), ('res_scale', C.c_float), ('reserved0', C.c_int32),
        ('p0', C.c_int64), ('P', C.c_int64),
    ]


# k4_testing_srnet_forward_upto: the decoder forward's steps (K4_SR_STEP_*) and the workspace layout of a tile
SR_STEP_KINDS = ('input', 'condnet', 'conv_first', 'rdb_conv', 'sft0', 'sft1', 'sft_rrdb', 'sft_body', 'conv_body', 'up1',
                 'up2', 'hr', 'last')


class SrStep(C.Structure):
    _fields_ = [('kind', C.c_int32), ('block', C.c_int32), ('dense', C.c_int32), ('conv', C.c_int32), ('fused', C.c_int32)]


class SrWsLayout(C.Structure):
    _fields_ = [(k, C.c_uint64) for k in ('in16', 'cond32', 'cond16', 'feat', 'trunk_a', 'trunk_b', 'cat', 'cat2', 'sbody',
                                           'bf', 'up1', 'up2', 'hr', 'total')]


# k4_testing_march_phases: counters per warpgroup and their slots (marchers: K4_PH_M_*, MLP groups: K4_PH_L_*)
K4_PHASE_SLOTS = 8
MARCHER_PHASES = {1: 'setup', 2: 'march', 3: 'rendezvous', 4: 'wait_done', 5: 'drain', 6: 'store'}
MLP_PHASES = {1: 'wait_full', 2: 'l1', 3: 'l2', 4: 'l3', 5: 'repack', 6: 'epilogue'}


class RgbnetTestArgs(C.Structure):
    """k4_rgbnet_test_args: a scene's rgbnet on caller rows for the test suite (k4_testing_rgbnet)."""
    _fields_ = [
        ('mode', C.c_int32), ('reserved0', C.c_int32), ('n', C.c_int64),
        ('d_x', C.c_void_p), ('d_diffuse', C.c_void_p), ('d_w', C.c_void_p), ('d_owner', C.c_void_p), ('d_racc', C.c_void_p),
    ]


EXPORTS = {
    'k4_abi_version': (C.c_int, []),
    'k4_status_string': (C.c_char_p, [C.c_int]),
    'k4_last_cuda_error': (C.c_char_p, []),
    'k4_device_check': (C.c_int, []),
    'k4_scene_create': (C.c_int, [C.POINTER(SceneDesc), C.c_void_p, C.POINTER(C.c_void_p)]),
    'k4_scene_destroy': (C.c_int, [C.c_void_p]),
    'k4_scene_device_bytes': (C.c_size_t, [C.c_void_p]),
    'k4_scene_best_mlp_mode': (C.c_int, [C.c_void_p]),
    'k4_scene_ws_config': (C.c_int, [C.c_void_p]),
    'k4_testing_ws_row_layout': (C.c_int, [C.c_int32, C.POINTER(C.c_int32)]),
    'k4_render_workspace_bytes': (C.c_size_t, [C.c_void_p, C.c_int64]),
    'k4_render_rays': (C.c_int, [C.c_void_p, C.POINTER(RenderArgs), C.c_void_p, C.c_void_p, C.c_void_p,
                                 C.c_int64, C.POINTER(RenderOut), C.c_void_p, C.c_size_t, C.c_void_p]),
    'k4_render_rays_frames': (C.c_int, [C.c_void_p, C.POINTER(RenderArgs), C.c_void_p, C.c_void_p, C.c_void_p,
                                        C.c_int64, C.POINTER(FrameDst), C.POINTER(RenderOut), C.c_void_p, C.c_size_t, C.c_void_p]),
    'k4_peer_enable_all': (C.c_int, []),
    'k4_peer_alloc': (C.c_int, [C.c_size_t, C.POINTER(C.c_void_p)]),
    'k4_peer_free': (C.c_int, [C.c_void_p]),
    'k4_peer_export': (C.c_int, [C.c_void_p, C.c_char_p]),
    'k4_peer_open': (C.c_int, [C.c_char_p, C.POINTER(C.c_void_p)]),
    'k4_peer_close': (C.c_int, [C.c_void_p]),
    'k4_srnet_create': (C.c_int, [C.POINTER(SrnetDesc), C.c_void_p, C.POINTER(C.c_void_p)]),
    'k4_srnet_destroy': (C.c_int, [C.c_void_p]),
    'k4_srnet_workspace_bytes': (C.c_size_t, [C.c_void_p, C.c_int32, C.c_int32]),
    'k4_srnet_forward': (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_int32, C.c_int32, C.c_void_p, C.c_void_p,
                                   C.c_size_t, C.c_void_p]),
    'k4_srnet_forward_roi': (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_int32, C.c_int32, C.c_int32, C.c_int32, C.c_int32, C.c_int32,
                                       C.c_void_p, C.c_int64, C.c_int64, C.c_void_p, C.c_size_t, C.c_void_p]),
    'k4_srnet_forward_roi_peers': (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_int32, C.c_int32, C.c_int32, C.c_int32, C.c_int32,
                                             C.c_int32, C.c_void_p, C.c_int64, C.c_int64, C.c_int32, C.POINTER(C.c_void_p),
                                             C.c_void_p, C.c_size_t, C.c_void_p]),
    'k4_op_infer_t_minmax': (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_float, C.c_float, C.c_int64, C.c_void_p, C.c_void_p, C.c_void_p]),
    'k4_op_infer_n_samples': (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_float, C.c_int64, C.c_void_p, C.c_void_p]),
    'k4_op_infer_ray_start_dir': (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_int64, C.c_void_p, C.c_void_p, C.c_void_p]),
    'k4_op_fill_ray_step_ids': (C.c_int, [C.c_void_p, C.c_int64, C.c_int64, C.c_void_p, C.c_void_p, C.c_void_p]),
    'k4_op_sample_pts': (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_float, C.c_int64, C.c_void_p, C.c_void_p, C.c_void_p]),
    'k4_op_sample_ndc_pts': (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_int32, C.c_int64, C.c_void_p, C.c_void_p, C.c_void_p]),
    'k4_op_sample_bg_pts': (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_float, C.c_int32, C.c_int64, C.c_void_p, C.c_void_p]),
    'k4_op_maskcache_lookup': (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_int32, C.c_int32, C.c_int32, C.c_int64, C.c_void_p]),
    'k4_op_raw2alpha': (C.c_int, [C.c_void_p, C.c_float, C.c_float, C.c_void_p, C.c_int64, C.c_void_p, C.c_void_p, C.c_void_p]),
    'k4_op_raw2alpha_backward': (C.c_int, [C.c_void_p, C.c_void_p, C.c_float, C.c_void_p, C.c_int64, C.c_void_p, C.c_void_p]),
    'k4_op_alpha2weight': (C.c_int, [C.c_void_p, C.c_void_p, C.c_int64, C.c_int64, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p]),
    'k4_op_alpha2weight_backward': (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_int64, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p]),
    'k4_op_total_variation_add_grad': (C.c_int, [C.c_void_p, C.c_void_p, C.c_float, C.c_float, C.c_float, C.c_int32, C.c_int64, C.c_int32, C.c_int32, C.c_int32, C.c_void_p]),
    'k4_op_adam_upd': (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_int64, C.c_int32, C.c_float, C.c_float, C.c_float, C.c_float, C.c_int32, C.c_void_p]),
    'k4_op_grid_alpha': (C.c_int, [C.c_void_p, C.c_int32, C.c_int32, C.c_int32, C.POINTER(C.c_float), C.POINTER(C.c_float), C.c_void_p, C.c_void_p, C.c_void_p,
                                   C.c_int32, C.c_int32, C.c_int32, C.c_float, C.c_float, C.c_void_p, C.c_void_p]),
    'k4_op_maxpool3_thres_and': (C.c_int, [C.c_void_p, C.c_int32, C.c_int32, C.c_int32, C.c_float, C.c_void_p, C.c_void_p]),
    'k4_op_cumdist_thres': (C.c_int, [C.c_void_p, C.c_float, C.c_int64, C.c_int64, C.c_void_p, C.c_void_p]),
    'k4_op_resample_trilinear': (C.c_int, [C.c_void_p, C.c_int32, C.c_int32, C.c_int32, C.c_int32, C.c_void_p, C.c_int32, C.c_int32, C.c_int32, C.c_void_p]),
    'k4_op_grid_sample': (C.c_int, [C.c_void_p, C.c_int32, C.c_int32, C.c_int32, C.c_int32, C.POINTER(C.c_float), C.POINTER(C.c_float),
                                    C.c_void_p, C.c_int64, C.c_void_p, C.c_void_p]),
    'k4_op_grid_sample_backward': (C.c_int, [C.c_void_p, C.c_int32, C.c_int32, C.c_int32, C.c_int32, C.POINTER(C.c_float), C.POINTER(C.c_float),
                                             C.c_void_p, C.c_int64, C.c_void_p, C.c_void_p]),
    'k4_op_distloss_workspace_bytes': (C.c_size_t, [C.c_int64]),
    'k4_op_distloss_forward': (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_int64, C.c_float, C.c_void_p, C.c_void_p,
                                         C.c_void_p, C.c_size_t, C.c_void_p]),
    'k4_op_distloss_backward': (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_int64, C.c_float, C.c_void_p, C.c_void_p,
                                          C.c_int32, C.c_void_p, C.c_size_t, C.c_void_p, C.c_void_p]),
    'k4_op_segment_cumsum': (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_int64, C.c_int64, C.c_void_p, C.c_void_p,
                                       C.c_void_p, C.c_void_p, C.c_void_p, C.c_size_t, C.c_void_p]),
    'k4_op_rgb_ssim_workspace_bytes': (C.c_size_t, [C.c_int64, C.c_int64, C.c_int32]),
    'k4_op_rgb_ssim': (C.c_int, [C.c_void_p, C.c_void_p, C.c_int32, C.c_int64, C.c_int64, C.POINTER(C.c_int64),
                                 C.POINTER(C.c_int64), C.POINTER(C.c_double), C.c_int32, C.c_double, C.c_double, C.c_void_p,
                                 C.c_void_p, C.c_void_p, C.c_size_t, C.c_void_p]),
    'k4_make_rays_rows':(C.c_int, [C.POINTER(C.c_float), C.POINTER(C.c_float), C.c_int32, C.c_int32, C.c_int32,
                                    C.c_int32, C.c_int32, C.c_int32, C.c_void_p, C.c_int32, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p]),
    'k4_make_rays': (C.c_int, [C.POINTER(C.c_float), C.POINTER(C.c_float), C.c_int32, C.c_int32, C.c_int32,
                               C.c_int32, C.c_int32, C.c_int32, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p]),
    'k4_testing_conv3x3': (C.c_int, [C.POINTER(ConvTestArgs), C.POINTER(C.c_int32), C.c_void_p]),
    'k4_testing_condnet': (C.c_int, [C.POINTER(CondnetTestArgs), C.POINTER(C.c_int32), C.c_void_p]),
    'k4_testing_sft': (C.c_int, [C.POINTER(SftTestArgs), C.POINTER(C.c_int32), C.c_void_p]),
    'k4_testing_srnet_forward_upto': (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_int32, C.c_int32, C.c_int32, C.c_int32,
                                                C.c_int32, C.c_int32, C.c_void_p, C.c_int64, C.c_int64, C.c_void_p, C.c_size_t,
                                                C.c_int32, C.POINTER(SrStep), C.c_int32, C.POINTER(C.c_int32),
                                                C.POINTER(SrWsLayout), C.c_void_p]),
    'k4_testing_rgbnet': (C.c_int, [C.c_void_p, C.POINTER(RgbnetTestArgs), C.POINTER(C.c_int32), C.c_void_p]),
    'k4_testing_march_phases': (C.c_int, [C.c_void_p, C.POINTER(RenderArgs), C.c_void_p, C.c_void_p, C.c_void_p, C.c_int64,
                                          C.POINTER(RenderOut), C.c_void_p, C.c_size_t, C.c_void_p, C.c_int32,
                                          C.POINTER(C.c_int32), C.c_void_p]),
    'k4_testing_skip_field': (C.c_int, [C.c_void_p, C.c_void_p, C.c_int64, C.POINTER(C.c_int32)]),
}

if not os.path.exists(LIB_PATH):
    raise RuntimeError(
        f'{LIB_PATH} is missing: build it with `python 4k-nerf_b200/csrc/build.py` '
        '(k4nerf has no CPU or PyTorch fallback for the rendering hot path)')

lib = C.CDLL(LIB_PATH)
for _name, (_res, _args) in EXPORTS.items():
    _fn = getattr(lib, _name)           # AttributeError here == the library does not match the header
    _fn.restype = _res
    _fn.argtypes = _args

if lib.k4_abi_version() != 1:
    raise RuntimeError('libk4nerf.so ABI version mismatch')


class K4Error(RuntimeError):
    pass


def check(status, what=''):
    if status != K4_OK:
        msg = lib.k4_status_string(status).decode()
        if status == -3:
            msg += ': ' + lib.k4_last_cuda_error().decode()
        raise K4Error(f'{what}: {msg}' if what else msg)
