"""render_viewpoints with the reference's two signatures (run.py:66-171, run_sr.py:74-182).

Differences that do not change results: rays are generated on the device (k4_make_rays), the whole
frame is ONE fused launch instead of 8192-ray chunks (the chunk loop only bounds the reference's
intermediate memory, run_sr.py:121-124), SSIM is computed on the device (utils.rgb_ssim of CUDA tensors), and
LPIPS, which needs pretrained weights this project does not ship, raises if requested.
"""
import numpy as np
import torch

from . import dvgo
from .utils import rgb_ssim, to8b


@torch.no_grad()
def _render_frames(model, render_poses, HW, Ks, ndc, render_kwargs, render_factor, flip_x, flip_y):
    if render_factor != 0:
        HW = np.copy(HW)
        Ks = np.copy(Ks)
        HW = (HW / render_factor).astype(int)
        Ks[:, :2, :3] /= render_factor
    frames = []
    for i, c2w in enumerate(render_poses):
        H, W = int(HW[i][0]), int(HW[i][1])
        K = Ks[i]
        rays_o, rays_d, viewdirs = dvgo.get_rays_of_a_view(
            H, W, K, torch.as_tensor(np.asarray(c2w), dtype=torch.float32), ndc,
            inverse_y=render_kwargs['inverse_y'], flip_x=flip_x, flip_y=flip_y)
        ret = model.render_rays(rays_o.view(-1, 3), rays_d.view(-1, 3), viewdirs.view(-1, 3),
                                render_kwargs, image_hw=(H, W))
        frames.append({
            'rgb_marched': ret['rgb_marched'].view(H, W, 3),
            'rgb_feature': ret['rgb_marched'].view(H, W, 3),
            'depth': ret['depth'].view(H, W, 1) if 'depth' in ret else None,
            'alphainv_last': ret['alphainv_last'].view(H, W, 1),
            'viewdirs': viewdirs.view(-1, 3),
        })
    return frames


def _post(rgbs, depths, bgmaps, render_video_flipy, render_video_rot90):
    if render_video_flipy:
        for i in range(len(rgbs)):
            rgbs[i] = np.flip(rgbs[i], axis=0); depths[i] = np.flip(depths[i], axis=0); bgmaps[i] = np.flip(bgmaps[i], axis=0)
    if render_video_rot90 != 0:
        for i in range(len(rgbs)):
            rgbs[i] = np.rot90(rgbs[i], k=render_video_rot90, axes=(0, 1))
            depths[i] = np.rot90(depths[i], k=render_video_rot90, axes=(0, 1))
            bgmaps[i] = np.rot90(bgmaps[i], k=render_video_rot90, axes=(0, 1))


def _write_png(filename, rgb8):
    """imageio.imwrite of the reference (run.py:165, run_sr.py:175), with the writers this environment may have instead."""
    try:
        import imageio
        imageio.imwrite(filename, rgb8)
        return
    except ImportError:
        pass
    try:
        from PIL import Image
        Image.fromarray(rgb8).save(filename)
        return
    except ImportError:
        pass
    import cv2
    cv2.imwrite(filename, rgb8[..., ::-1])


def _ssim_on_device(rgb, gt):
    """``rgb_ssim(rgb, gt, max_val=1)`` of a clamped frame still on the device (run.py:134-135): the ground truth is
    uploaded, the frame is not copied back for it."""
    return rgb_ssim(rgb, torch.as_tensor(gt, device=rgb.device), max_val=1)


def _report(psnrs, ssims):
    """run.py:141-145 / run_sr.py:153-157."""
    if len(psnrs):
        print('Testing psnr', np.mean(psnrs), '(avg)')
        if len(ssims):
            print('Testing ssim', np.mean(ssims), '(avg)')


def _dump(rgbs, savedir, dump_images, global_step):
    """run.py:161-165 / run_sr.py:171-175: ``e<global_step>_<index>.png`` of the (flipped / rotated) 8-bit frames."""
    if savedir is None or not dump_images:
        return
    import os
    for i, rgb in enumerate(rgbs):
        _write_png(os.path.join(savedir, 'e{}_{:03d}.png'.format(global_step, i)), to8b(np.ascontiguousarray(rgb)))


@torch.no_grad()
def render_viewpoints(model, render_poses, HW, Ks, ndc, render_kwargs,
                      gt_imgs=None, savedir=None, dump_images=False,
                      render_factor=0, render_video_flipy=False, render_video_rot90=0,
                      eval_ssim=False, eval_lpips_alex=False, eval_lpips_vgg=False, global_step=0,
                      arr_index=None, img_enc=None, flip_x=None, flip_y=None):
    """run.py:66-171 contract: returns ``(rgbs, depths, bgmaps, psnrs, ssims, lpips_vgg)``; ``savedir`` +
    ``dump_images`` write ``e<global_step>_<i>.png`` like the reference.

    The reference reads ``cfg.data.flip_x/flip_y`` from a module global (run.py:96); here they come
    from ``render_kwargs`` unless passed explicitly.  The reference's defaults evaluate SSIM and LPIPS-VGG when ground
    truth is given (here both default to off): ``eval_ssim`` scores the frame on the GPU (``utils.rgb_ssim``), LPIPS needs the
    ``lpips`` package and its pretrained VGG / AlexNet weights and raises."""
    assert len(render_poses) == len(HW) and len(HW) == len(Ks)
    if eval_lpips_alex or eval_lpips_vgg:
        raise NotImplementedError('LPIPS evaluation needs the lpips package and its pretrained weights')
    if arr_index is not None or img_enc is not None:
        raise NotImplementedError('img_enc conditioning needs lib/img_encoder, which the reference does not ship')
    flip_x = render_kwargs.get('flip_x', False) if flip_x is None else flip_x
    flip_y = render_kwargs.get('flip_y', False) if flip_y is None else flip_y
    frames = _render_frames(model, render_poses, HW, Ks, ndc, render_kwargs, render_factor, flip_x, flip_y)
    rgbs, depths, bgmaps, psnrs, ssims = [], [], [], [], []
    for i, f in enumerate(frames):
        rgb_d = f['rgb_marched'].clamp(0, 1)
        rgb = rgb_d.cpu().numpy()
        rgbs.append(rgb)
        depths.append(f['depth'].cpu().numpy() if f['depth'] is not None else None)
        bgmaps.append(f['alphainv_last'].cpu().numpy())
        if gt_imgs is not None and render_factor == 0:
            psnrs.append(-10. * np.log10(np.mean(np.square(rgb - gt_imgs[i]))))
            if eval_ssim:
                ssims.append(_ssim_on_device(rgb_d, gt_imgs[i]))          # run.py:134-135
    _report(psnrs, ssims)
    _post(rgbs, depths, bgmaps, render_video_flipy, render_video_rot90)
    _dump(rgbs, savedir, dump_images, global_step)
    return np.array(rgbs), np.array(depths), np.array(bgmaps), psnrs, ssims, []


@torch.no_grad()
def render_viewpoints_sr(model, render_poses, HW, Ks, ndc, render_kwargs,
                         gt_imgs=None, savedir=None, dump_images=False,
                         render_factor=0, render_video_flipy=False, render_video_rot90=0,
                         eval_ssim=False, eval_lpips_alex=False, eval_lpips_vgg=False, global_step=0,
                         arr_index=None, img_enc=None, flip_x=None, flip_y=None):
    """run_sr.py:74-182 contract: returns ``(rgbs, depths, bgmaps, psnrs, viewdirs_all, rgb_features)``
    where ``rgb_features`` is the UNclamped render fed to the VC-Decoder (run_sr.py:131)."""
    assert len(render_poses) == len(HW) and len(HW) == len(Ks)
    if arr_index is not None or img_enc is not None:
        raise NotImplementedError('img_enc conditioning needs lib/img_encoder, which the reference does not ship')
    flip_x = render_kwargs.get('flip_x', False) if flip_x is None else flip_x
    flip_y = render_kwargs.get('flip_y', False) if flip_y is None else flip_y
    frames = _render_frames(model, render_poses, HW, Ks, ndc, render_kwargs, render_factor, flip_x, flip_y)
    if eval_lpips_alex or eval_lpips_vgg:
        raise NotImplementedError('LPIPS evaluation needs the lpips package and its pretrained weights')
    rgbs, rgb_features, depths, bgmaps, psnrs, ssims, viewdirs_all = [], [], [], [], [], [], []
    for i, f in enumerate(frames):
        rgb_d = f['rgb_marched'].clamp(0, 1)
        rgb = rgb_d.cpu().numpy()
        rgbs.append(rgb)
        rgb_features.append(f['rgb_feature'].cpu().numpy())
        depths.append(f['depth'].cpu().numpy())
        bgmaps.append(f['alphainv_last'].cpu().numpy())
        viewdirs_all.append(f['viewdirs'])
        if gt_imgs is not None and render_factor == 0:
            psnrs.append(-10. * np.log10(np.mean(np.square(rgb - gt_imgs[i]))))
            if eval_ssim:
                ssims.append(_ssim_on_device(rgb_d, gt_imgs[i]))          # run_sr.py:146-147 (printed, not returned)
    _report(psnrs, ssims)
    _post(rgbs, depths, bgmaps, render_video_flipy, render_video_rot90)
    _dump(rgbs, savedir, dump_images, global_step)
    return np.array(rgbs), np.array(depths), np.array(bgmaps), psnrs, viewdirs_all, np.array(rgb_features)


@torch.no_grad()
def render_frame_4k(model, net_sr, H, W, K, c2w, ndc, render_kwargs, test_tile=510, out_u8=False,
                    flip_x=False, flip_y=False):
    """One full 4K-NeRF frame, device resident (SURVEY.md section 8 f-1): rays generated on the
    device, one fused marcher launch at HxW, ``rgb_feature`` + ``depth`` handed to the VC-Decoder
    without the numpy round trip of run_sr.py:130-133,1362-1367, x``s`` decode (``s = net_sr.scale``: 4, or 1 for the
    1x configs) with the reference's tile geometry (``--test_tile``), optional ``to8b`` quantisation (lib/utils.py:20)
    on the device.

    The decoder's condition is :func:`k4nerf.sr_esrnet.sft_condition` of ``net_sr.num_cond``: the depth, the view
    embedding of the frame's ``viewdirs``, or both.

    Returns ``(sr [3,s*H,s*W] float32 in [0,1] or uint8 [s*H,s*W,3], lr dict)`` -- same values as
    ``render_viewpoints_sr`` followed by ``SFTNet.tile_process`` and ``clamp(0,1)``."""
    from .sr_esrnet import sft_condition
    rays_o, rays_d, viewdirs = dvgo.get_rays_of_a_view(
        H, W, K, torch.as_tensor(np.asarray(c2w), dtype=torch.float32), ndc,
        inverse_y=render_kwargs['inverse_y'], flip_x=flip_x, flip_y=flip_y)
    kw = dict(render_kwargs)
    kw['render_depth'] = True
    lr = model.render_rays(rays_o.view(-1, 3), rays_d.view(-1, 3), viewdirs.view(-1, 3), kw, image_hw=(H, W))
    x = lr['rgb_marched'].view(H, W, 3).permute(2, 0, 1).unsqueeze(0).contiguous()    # unclamped, as run_sr.py:131
    cond = sft_condition(net_sr.num_cond, lr['depth'], viewdirs, H, W)
    sr = net_sr.tile_process(x, cond, tile_size=test_tile if test_tile else max(H, W), to_cpu=False)
    sr = sr.squeeze(0).clamp_(0, 1)
    if out_u8:
        sr = (sr * 255).to(torch.uint8).permute(1, 2, 0).contiguous()     # to8b: (255*clip(x,0,1)).astype(uint8)
    return sr, lr


@torch.no_grad()
def render_frame_4k_sharded(model, net_sr, H, W, K, c2w, ndc, render_kwargs, test_tile=510, out_u8=False,
                            flip_x=False, flip_y=False, group=None):
    """:func:`render_frame_4k` across the ranks of ``group`` (one process per GPU, scene and decoder
    replicated; SURVEY.md section 8e / config 5): every rank marches its 8-row blocks of the LR frame
    (one all-gather of the packed ``[rgb|depth|alphainv]`` rows), then decodes its share of the
    reference tiles / tile row-parts (one all-gather of the decoded blocks, x``net_sr.scale``).  Every rank returns the
    full frame; values are identical to the single-GPU :func:`render_frame_4k`.  The LR dict's tensors are views of the
    cached :class:`k4nerf.dist.CyclicFrame` buffer (no allocation per frame): valid until the next call with the same
    (H, W, group).  A view-conditioned decoder (``net_sr.num_cond`` 63 / 64) needs the whole frame's ``viewdirs``: every
    rank generates them itself (they depend on ``K`` and ``c2w`` only), so nothing more is exchanged."""
    from . import dist as kdist
    from .sr_esrnet import sft_condition
    kw = dict(render_kwargs)
    kw['render_depth'] = True
    dev = next(model.parameters()).device
    cache = model.__dict__.setdefault('_k4_cyclic_frames', {})
    key = (H, W, dev, id(group))
    frame = cache.get(key)
    if frame is None:
        frame = cache[key] = kdist.CyclicFrame(H, W, dev, group)
    c2w_t = torch.as_tensor(np.asarray(c2w), dtype=torch.float32)
    make = lambda rows: tuple(t.view(-1, 3) for t in dvgo.get_rays_of_a_view(
        H, W, K, c2w_t, ndc, inverse_y=render_kwargs['inverse_y'], flip_x=flip_x, flip_y=flip_y, rows=rows, device=dev))
    fn = lambda ro, rd, vd, hw, out: model.render_rays(ro, rd, vd, kw, image_hw=hw, out=out)
    lr = frame.render(make, fn)          # rank's rays only -> fused march into the packed buffer -> one all-gather -> transpose
    x = lr['rgb_marched'].view(H, W, 3).permute(2, 0, 1).unsqueeze(0).contiguous()
    viewdirs = None
    if net_sr.num_cond != 1:
        viewdirs = dvgo.get_rays_of_a_view(H, W, K, c2w_t, ndc, inverse_y=render_kwargs['inverse_y'], flip_x=flip_x,
                                           flip_y=flip_y, device=dev)[2]
    cond = sft_condition(net_sr.num_cond, lr['depth'], viewdirs, H, W).contiguous()
    sr = net_sr.tile_process_sharded(x, cond, tile_size=test_tile if test_tile else max(H, W), group=group)
    sr = sr.squeeze(0).clamp_(0, 1)
    if out_u8:
        sr = (sr * 255).to(torch.uint8).permute(1, 2, 0).contiguous()
    return sr, lr
