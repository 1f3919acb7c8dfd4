"""render_viewpoints with the reference's two signatures (run.py:66-171, run_sr.py:74-182).

Differences that do not change results: rays are generated on the device (k4_make_rays), the whole
frame is ONE fused launch instead of 8192-ray chunks (the chunk loop only bounds the reference's
intermediate memory, run_sr.py:121-124), and SSIM and LPIPS are computed on the device (utils.rgb_ssim and
utils.rgb_lpips of CUDA tensors).
"""
import numpy as np
import torch

from . import dvgo
from .utils import rgb_lpips, rgb_ssim, to8b


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


def _score(rgb, gt, eval_ssim, eval_lpips_alex, eval_lpips_vgg, ssims, lpips_alex, lpips_vgg):
    """run.py:136-141 / run_sr.py:146-151 on a clamped frame still on the device: the ground truth is uploaded once."""
    if not (eval_ssim or eval_lpips_alex or eval_lpips_vgg):
        return
    gt = torch.as_tensor(gt, device=rgb.device)
    if eval_ssim:
        ssims.append(rgb_ssim(rgb, gt, max_val=1))
    if eval_lpips_alex:
        lpips_alex.append(rgb_lpips(rgb, gt, net_name='alex', device=rgb.device))
    if eval_lpips_vgg:
        lpips_vgg.append(rgb_lpips(rgb, gt, net_name='vgg', device=rgb.device))


def _report(psnrs, ssims, lpips_vgg, lpips_alex):
    """run.py:143-147 / run_sr.py:153-157."""
    if len(psnrs):
        print('Testing psnr', np.mean(psnrs), '(avg)')
        if len(ssims):
            print('Testing ssim', np.mean(ssims), '(avg)')
        if len(lpips_vgg):
            print('Testing lpips (vgg)', np.mean(lpips_vgg), '(avg)')
        if len(lpips_alex):
            print('Testing lpips (alex)', np.mean(lpips_alex), '(avg)')


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
    truth is given (here both default to off): ``eval_ssim`` and ``eval_lpips_vgg`` / ``eval_lpips_alex`` score the
    frame on the GPU (``utils.rgb_ssim``, ``utils.rgb_lpips``; LPIPS loads the ``lpips`` package's pretrained weights)."""
    assert len(render_poses) == len(HW) and len(HW) == len(Ks)
    if arr_index is not None or img_enc is not None:
        raise NotImplementedError('img_enc conditioning needs lib/img_encoder, which the reference does not ship')
    flip_x = render_kwargs.get('flip_x', False) if flip_x is None else flip_x
    flip_y = render_kwargs.get('flip_y', False) if flip_y is None else flip_y
    frames = _render_frames(model, render_poses, HW, Ks, ndc, render_kwargs, render_factor, flip_x, flip_y)
    rgbs, depths, bgmaps, psnrs, ssims, lpips_alex, lpips_vgg = [], [], [], [], [], [], []
    for i, f in enumerate(frames):
        rgb_d = f['rgb_marched'].clamp(0, 1)
        rgb = rgb_d.cpu().numpy()
        rgbs.append(rgb)
        depths.append(f['depth'].cpu().numpy() if f['depth'] is not None else None)
        bgmaps.append(f['alphainv_last'].cpu().numpy())
        if gt_imgs is not None and render_factor == 0:
            psnrs.append(-10. * np.log10(np.mean(np.square(rgb - gt_imgs[i]))))
            _score(rgb_d, gt_imgs[i], eval_ssim, eval_lpips_alex, eval_lpips_vgg, ssims, lpips_alex, lpips_vgg)
    _report(psnrs, ssims, lpips_vgg, lpips_alex)
    _post(rgbs, depths, bgmaps, render_video_flipy, render_video_rot90)
    _dump(rgbs, savedir, dump_images, global_step)
    return np.array(rgbs), np.array(depths), np.array(bgmaps), psnrs, ssims, lpips_vgg


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
    rgbs, rgb_features, depths, bgmaps, psnrs, ssims, viewdirs_all = [], [], [], [], [], [], []
    lpips_alex, lpips_vgg = [], []
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
            # run_sr.py:146-151: printed, not returned
            _score(rgb_d, gt_imgs[i], eval_ssim, eval_lpips_alex, eval_lpips_vgg, ssims, lpips_alex, lpips_vgg)
    _report(psnrs, ssims, lpips_vgg, lpips_alex)
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
    sr, lr, _ = _render_frame_4k(model, net_sr, H, W, K, c2w, ndc, render_kwargs, test_tile, out_u8, flip_x, flip_y)
    return sr, lr


def _render_frame_4k(model, net_sr, H, W, K, c2w, ndc, render_kwargs, test_tile, out_u8, flip_x, flip_y):
    """:func:`render_frame_4k` and the frame's ``viewdirs`` ``[H*W, 3]``."""
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
    return sr, lr, viewdirs.view(-1, 3)


@torch.no_grad()
def render_test_4k(model, net_sr, render_poses, HW, Ks, ndc, render_kwargs, gt_imgs=None, savedir=None, ckpt_name='',
                   dump_images=False, eval_ssim=False, eval_lpips_alex=False, eval_lpips_vgg=False, global_step=0,
                   test_tile=510, flip_x=None, flip_y=None):
    """run_sr.py --render_test (run_sr.py:1340-1396) with every frame rendered and written from the device.

    Each view is one :func:`render_frame_4k` pass (march, decode, quantise), with no numpy round trip between the
    marcher and the decoder.  The LR results are what :func:`render_viewpoints_sr` returns on the same inputs, bit for
    bit: ``(rgbs, depths, bgmaps, psnrs, viewdirs_all, rgb_features)``; with ``gt_imgs`` the PSNR is computed and
    SSIM / LPIPS scored and printed as there.  With ``savedir``: ``dump_images`` writes the LR frames as
    ``e<global_step>_<i>.png`` (the pixels of ``render_viewpoints_sr``'s dumps), and every SR frame is written as
    ``<ckpt_name>_<i>.png``, ``to8b`` of the clamped decoder output; both are encoded on the GPU
    (:func:`k4nerf.utils.png_encode`).  ``ckpt_name`` is the reference's ``ckpt_path.split('/')[-1][:-4]``."""
    import os
    from .utils import frame_u8_cuda, write_png
    assert len(render_poses) == len(HW) and len(HW) == len(Ks)
    flip_x = render_kwargs.get('flip_x', False) if flip_x is None else flip_x
    flip_y = render_kwargs.get('flip_y', False) if flip_y is None else flip_y
    rgbs, rgb_features, depths, bgmaps, psnrs, ssims, viewdirs_all = [], [], [], [], [], [], []
    lpips_alex, lpips_vgg = [], []
    for i, c2w in enumerate(render_poses):
        H, W = int(HW[i][0]), int(HW[i][1])
        sr, lr, viewdirs = _render_frame_4k(model, net_sr, H, W, Ks[i], c2w, ndc, render_kwargs, test_tile, True,
                                            flip_x, flip_y)
        rgb_f = lr['rgb_marched'].view(H, W, 3)
        rgb_d = rgb_f.clamp(0, 1)
        rgb = rgb_d.cpu().numpy()
        rgbs.append(rgb)
        rgb_features.append(rgb_f.cpu().numpy())
        depths.append(lr['depth'].view(H, W, 1).cpu().numpy())
        bgmaps.append(lr['alphainv_last'].view(H, W, 1).cpu().numpy())
        viewdirs_all.append(viewdirs)
        if gt_imgs is not None:
            psnrs.append(-10. * np.log10(np.mean(np.square(rgb - gt_imgs[i]))))
            _score(rgb_d, gt_imgs[i], eval_ssim, eval_lpips_alex, eval_lpips_vgg, ssims, lpips_alex, lpips_vgg)
        if savedir is not None:
            if dump_images:
                write_png(os.path.join(savedir, 'e{}_{:03d}.png'.format(global_step, i)), frame_u8_cuda(rgb_f))
            write_png(os.path.join(savedir, '{}_{:03d}.png'.format(ckpt_name, i)), sr)
    _report(psnrs, ssims, lpips_vgg, lpips_alex)
    return np.array(rgbs), np.array(depths), np.array(bgmaps), psnrs, viewdirs_all, np.array(rgb_features)


@torch.no_grad()
def render_val_4k(model, net_sr, poses, HW, Ks, ndc, render_kwargs, gt_imgs, srgt, load_sr, savedir=None, global_step=0,
                  sel_b=0, test_tile=510, dump_images=False, eval_ssim=False, eval_lpips_alex=False, eval_lpips_vgg=False,
                  lpips_weights=None, flip_x=None, flip_y=None):
    """The joint stage's validation block of run_sr.py (run_sr.py:1088-1146) with every SR frame scored and written on
    the device.  Each view is one :func:`render_frame_4k` pass; its LR results are :func:`render_viewpoints_sr`'s on the
    same inputs, bit for bit, scored against ``gt_imgs`` and dumped (``dump_images``) as there.  The clamped SR frame
    stays on the device and is scored against ``srgt[i]`` (the block's ``rgb_srgt_val``: numpy arrays or CUDA tensors,
    uploaded once in their own layout):

    * ``sr_psnr = -10. * np.log10(utils.rgb_mse(sr, gt))``: numpy's float32 value bit for bit;
    * ``sr_ssim = utils.rgb_ssim(sr, gt, max_val=1)``;
    * ``sr_lpips = utils.rgb_lpips`` (VGG, ``lpips_weights`` as its ``weights``) of ``utils.resize_quarter`` of both
      frames when ``load_sr == 1`` (cv2's ``fx = fy = 1/4``), of the frames themselves otherwise.

    With ``savedir``, ``test_<global_step>.png`` (``to8b`` of the LR frame) and ``testsr_<global_step>_<sel_b>.png`` (of
    the SR frame) are written from the device for every view, as the reference overwrites them.  The reference's three
    ``Testing ... (sr)`` lines are printed per view after the LR report.  Returns ``render_viewpoints_sr``'s
    ``(rgbs, depths, bgmaps, psnrs, viewdirs_all, rgb_features)`` followed by the per-view lists ``sr_psnrs``,
    ``sr_ssims`` and ``sr_lpips``; choosing and saving the checkpoint stays with the caller."""
    import os
    from .utils import frame_u8_cuda, resize_quarter, rgb_mse, write_png
    assert len(poses) == len(HW) and len(HW) == len(Ks) and len(srgt) >= len(poses)
    flip_x = render_kwargs.get('flip_x', False) if flip_x is None else flip_x
    flip_y = render_kwargs.get('flip_y', False) if flip_y is None else flip_y
    dev = next(model.parameters()).device
    srgt = torch.as_tensor(srgt).to(dev)
    rgbs, rgb_features, depths, bgmaps, psnrs, ssims, viewdirs_all = [], [], [], [], [], [], []
    lpips_alex, lpips_vgg, sr_psnrs, sr_ssims, sr_lpips = [], [], [], [], []
    for i, c2w in enumerate(poses):
        H, W = int(HW[i][0]), int(HW[i][1])
        sr, lr, viewdirs = _render_frame_4k(model, net_sr, H, W, Ks[i], c2w, ndc, render_kwargs, test_tile, False,
                                            flip_x, flip_y)
        rgb_f = lr['rgb_marched'].view(H, W, 3)
        rgb_d = rgb_f.clamp(0, 1)
        rgb = rgb_d.cpu().numpy()
        rgbs.append(rgb)
        rgb_features.append(rgb_f.cpu().numpy())
        depths.append(lr['depth'].view(H, W, 1).cpu().numpy())
        bgmaps.append(lr['alphainv_last'].view(H, W, 1).cpu().numpy())
        viewdirs_all.append(viewdirs)
        if gt_imgs is not None:
            psnrs.append(-10. * np.log10(np.mean(np.square(rgb - gt_imgs[i]))))
            _score(rgb_d, gt_imgs[i], eval_ssim, eval_lpips_alex, eval_lpips_vgg, ssims, lpips_alex, lpips_vgg)
        if savedir is not None and dump_images:
            write_png(os.path.join(savedir, 'e{}_{:03d}.png'.format(global_step, i)), frame_u8_cuda(rgb_f))
        sr_hwc, gt = sr.permute(1, 2, 0), srgt[i]
        sr_psnrs.append(-10. * np.log10(rgb_mse(sr_hwc, gt)))
        sr_ssims.append(rgb_ssim(sr_hwc, gt, max_val=1))
        if load_sr == 1:
            sr_lpips.append(rgb_lpips(resize_quarter(sr_hwc), resize_quarter(gt), 'vgg', weights=lpips_weights))
        else:
            sr_lpips.append(rgb_lpips(sr_hwc, gt, 'vgg', weights=lpips_weights))
        if savedir is not None:
            write_png(os.path.join(savedir, f'test_{global_step}.png'), frame_u8_cuda(rgb_f))
            write_png(os.path.join(savedir, f'testsr_{global_step}_{sel_b}.png'), frame_u8_cuda(sr_hwc))
    _report(psnrs, ssims, lpips_vgg, lpips_alex)
    for p, s, l in zip(sr_psnrs, sr_ssims, sr_lpips):
        print('Testing psnr', p, '(sr)')
        print('Testing ssim', s, '(sr)')
        print('Testing lpips', l, '(sr)')
    return (np.array(rgbs), np.array(depths), np.array(bgmaps), psnrs, viewdirs_all, np.array(rgb_features),
            sr_psnrs, sr_ssims, sr_lpips)


@torch.no_grad()
def render_video_4k(model, net_sr, render_poses, HW, Ks, ndc, render_kwargs, render_factor=0, render_video_flipy=False,
                    render_video_rot90=0, test_tile=510, flip_x=None, flip_y=None, on_frame=None):
    """The three videos of run_sr.py --render_video (run_sr.py:1399-1463) as the uint8 arrays it hands to
    ``imageio.mimwrite``: ``(sr [n, s*H', s*W', 3], lr [n, H', W', 3], depth [n, H', W', 3])``, ``s = net_sr.scale``,
    the primes meaning after ``render_video_rot90``.  Every frame is :func:`render_frame_4k` (``render_factor``
    scales ``HW`` and ``Ks`` as ``render_viewpoints`` does); its SR and LR frames are quantised on the device
    (``utils.frame_u8_cuda``), the SR one copied to the host as uint8, and its depth and bgmap stay on the device until
    the depth video is made from all of them (``utils.depth_video_frames``).

    ``on_frame(i, sr_u8, lr_u8)`` (optional) receives each frame's uint8 CUDA tensors as soon as they exist, e.g. for a
    streaming encoder; the SR frames are then not kept and ``sr`` is returned as ``None``.  ``lr_u8`` is a view of the
    LR video's device buffer: copy it to keep it beyond the call.

    With ``render_video_flipy`` / ``render_video_rot90`` all three streams are flipped and rotated, and the decoder
    reads the unflipped frame and condition, exactly as without them.  (The reference flips the depths it conditions
    the decoder on but not the decoder's input image, and leaves its SR video unflipped.)"""
    from .utils import depth_video_frames, frame_u8_cuda
    assert len(render_poses) == len(HW) and len(HW) == len(Ks)
    flip_x = render_kwargs.get('flip_x', False) if flip_x is None else flip_x
    flip_y = render_kwargs.get('flip_y', False) if flip_y is None else flip_y
    if render_factor != 0:
        HW = (np.copy(HW) / render_factor).astype(int)
        Ks = np.copy(Ks)
        Ks[:, :2, :3] /= render_factor
    n = len(render_poses)
    H, W = int(HW[0][0]), int(HW[0][1])
    if any((int(h), int(w)) != (H, W) for h, w in HW):
        raise ValueError('render_video_4k: every frame of a video must have the same size')
    dev = next(model.parameters()).device
    k = int(render_video_rot90) % 4
    rot = lambda h, w: (w, h) if k & 1 else (h, w)
    s = net_sr.scale
    depths = torch.empty((n, H, W), dtype=torch.float32, device=dev)
    bgmaps = torch.empty((n, H, W), dtype=torch.float32, device=dev)
    lr_u8 = torch.empty((n, *rot(H, W), 3), dtype=torch.uint8, device=dev)
    sr_host = None if on_frame is not None else np.empty((n, *rot(s * H, s * W), 3), dtype=np.uint8)
    for i, c2w in enumerate(render_poses):
        sr, lr = render_frame_4k(model, net_sr, H, W, Ks[i], c2w, ndc, render_kwargs, test_tile=test_tile, flip_x=flip_x,
                                 flip_y=flip_y)
        depths[i].copy_(lr['depth'].reshape(H, W))
        bgmaps[i].copy_(lr['alphainv_last'].reshape(H, W))
        frame_u8_cuda(lr['rgb_marched'].reshape(H, W, 3), render_video_flipy, k, out=lr_u8[i])
        sr_u8 = frame_u8_cuda(sr.permute(1, 2, 0), render_video_flipy, k)
        if on_frame is not None:
            on_frame(i, sr_u8, lr_u8[i])
        else:
            torch.from_numpy(sr_host[i]).copy_(sr_u8)
    depth_u8 = depth_video_frames(depths, bgmaps, q=(5, 95), render_video_flipy=render_video_flipy, render_video_rot90=k)
    return sr_host, lr_u8.cpu().numpy(), depth_u8.cpu().numpy()


@torch.no_grad()
def render_video_4k_sharded(model, net_sr, render_poses, HW, Ks, ndc, render_kwargs, render_factor=0,
                            render_video_flipy=False, render_video_rot90=0, test_tile=510, flip_x=None, flip_y=None,
                            on_frame=None, group=None, dst=0):
    """:func:`render_video_4k` on every rank of ``group`` (one process per GPU of one node, scene and decoder
    replicated, as for :func:`render_frame_4k_sharded`): frame ``i`` is :func:`render_frame_4k` on rank ``i % world``,
    whole, so ranks exchange no part of a frame (:func:`k4nerf.dist.render_video_frames`).  Rank ``dst`` returns
    ``(sr, lr, depth)``, bit for bit :func:`render_video_4k`'s on the same inputs, and calls ``on_frame(i, sr_u8, lr_u8)``
    in increasing ``i``; every other rank returns ``(None, None, None)``.  The u8 frames of each round (one frame per
    rank) are gathered to ``dst``; the depth video's 5th / 95th percentiles are exact over all frames
    (:func:`k4nerf.utils.depth_video_frames_sharded`: three histogram all-reduces).  A ``gloo`` group takes the CUDA
    tensors through the host.  Collective: every rank calls it with the same arguments."""
    from . import dist as kdist
    from .utils import frame_u8_cuda
    assert len(render_poses) == len(HW) and len(HW) == len(Ks)
    flip_x = render_kwargs.get('flip_x', False) if flip_x is None else flip_x
    flip_y = render_kwargs.get('flip_y', False) if flip_y is None else flip_y
    if render_factor != 0:
        HW = (np.copy(HW) / render_factor).astype(int)
        Ks = np.copy(Ks)
        Ks[:, :2, :3] /= render_factor
    H, W = int(HW[0][0]), int(HW[0][1])
    if any((int(h), int(w)) != (H, W) for h, w in HW):
        raise ValueError('render_video_4k_sharded: every frame of a video must have the same size')
    k = int(render_video_rot90) % 4
    rot = lambda h, w: (w, h) if k & 1 else (h, w)
    s = net_sr.scale

    def render_into(i, sr_u8, lr_u8, depth, bgmap):
        sr, lr = render_frame_4k(model, net_sr, H, W, Ks[i], render_poses[i], ndc, render_kwargs, test_tile=test_tile,
                                 flip_x=flip_x, flip_y=flip_y)
        depth.copy_(lr['depth'].reshape(H, W))
        bgmap.copy_(lr['alphainv_last'].reshape(H, W))
        frame_u8_cuda(lr['rgb_marched'].reshape(H, W, 3), render_video_flipy, k, out=lr_u8)
        frame_u8_cuda(sr.permute(1, 2, 0), render_video_flipy, k, out=sr_u8)
    return kdist.render_video_frames(render_into, len(render_poses), H, W, (*rot(s * H, s * W), 3), (*rot(H, W), 3),
                                     next(model.parameters()).device, render_video_flipy, k, on_frame, group, dst)


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
