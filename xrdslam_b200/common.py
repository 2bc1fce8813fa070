"""Pixel sampling and ray generation (mirror of slam/common/common.py:39-122,
188-227,288-310 and slam/utils/utils.py:28-65).  Frames stay resident on the
device once uploaded (the reference re-uploads the full image every call,
common.py:67-68 -- SURVEY row f1)."""
import numpy as np
import torch


def _as_dev(x, device, dtype=torch.float32):
    if isinstance(x, np.ndarray):
        x = torch.from_numpy(x)
    return x.to(device=device, dtype=dtype)


class _PosedRays(torch.autograd.Function):
    """csrc/rays.cu: rays from camera-frame directions + per-ray pose row, and the pose
    gradient reduction (one launch each; replaces torch's gather / index_put backward)."""
    @staticmethod
    def forward(ctx, dirs, ids, poses):
        import ctypes as C
        from . import _cabi
        dirs = dirs.detach().to(torch.float32).contiguous()
        P = poses.detach().to(torch.float32).contiguous()
        R = dirs.shape[0]
        rays_o = torch.empty(R, 3, device=dirs.device)
        rays_d = torch.empty(R, 3, device=dirs.device)
        _cabi.launch_on(dirs.device, 'xrd_rays_from_poses', R, _cabi.ptr(dirs), _cabi.ptr(ids),
                        _cabi.ptr(P), P.shape[0], _cabi.ptr(rays_o), _cabi.ptr(rays_d))
        ctx.save_for_backward(dirs, ids)
        ctx.n_poses = P.shape[0]
        return rays_o, rays_d

    @staticmethod
    def backward(ctx, g_o, g_d):
        from . import _cabi
        dirs, ids = ctx.saved_tensors
        d_poses = torch.empty(ctx.n_poses, 4, 4, device=dirs.device)
        g_o, g_d = g_o.contiguous(), g_d.contiguous()
        _cabi.launch_on(dirs.device, 'xrd_rays_pose_grads', dirs.shape[0], _cabi.ptr(dirs),
                        _cabi.ptr(ids), ctx.n_poses, _cabi.ptr(g_o), _cabi.ptr(g_d),
                        _cabi.ptr(d_poses))
        return None, None, d_poses


def rays_from_poses(dirs_cam, pose_ids, poses):
    """rays_o, rays_d [R,3] from camera-frame directions [R,3], per-ray pose rows `pose_ids`
    ([R] int64, negative = from the end, or None: pose 0) and c2w `poses` [n,4,4];
    differentiable w.r.t. poses (coslam.py:208-216 / common.py:39-53)."""
    if dirs_cam.is_cuda:
        if pose_ids is not None:
            pose_ids = pose_ids.to(dirs_cam.device, torch.int64).contiguous()
        return _PosedRays.apply(dirs_cam, pose_ids, poses.to(dirs_cam.device))
    # host tensors (dataset preparation, CPU tests of the host logic): plain torch
    ids = pose_ids if pose_ids is not None else torch.zeros(dirs_cam.shape[0], dtype=torch.int64)
    rays_d = torch.sum(dirs_cam[:, None, :] * poses[ids, :3, :3], -1)
    return poses[ids, :3, -1], rays_d


def sample_window(camera, depth_imgs, rgb_imgs, poses, n, Hedge=0, Wedge=0, indices=None,
                  return_index=False):
    """get_samples for every frame of a window in THREE launches (draw, gather, rays):
    depth_imgs / rgb_imgs: lists of device-resident [H,W] / [H,W,3] fp32 frames, poses:
    [F,4,4] c2w on the device (differentiable).  Frame-major outputs
    rays_o, rays_d [F*n,3], depth [F*n,1], colour [F*n,3] (+ i, j int64 column / row).
    Mirrors common.py:188-227 applied per frame and concatenated (nice_slam.py:141-171)."""
    import ctypes as C
    from . import _cabi
    dev = poses.device
    _cabi.require_cuda(dev, 'poses')
    F = len(depth_imgs)
    H, W = camera.height, camera.width
    H0, H1, W0, W1 = Hedge, H - Hedge, Wedge, W - Wedge
    if indices is None:
        indices = torch.randint((H1 - H0) * (W1 - W0), (F * n, ), device=dev)
    indices = indices.to(dev, torch.int64).contiguous()
    tot = F * n
    dirs = torch.empty(tot, 3, device=dev)
    depth = torch.empty(tot, 1, device=dev)
    rgb = torch.empty(tot, 3, device=dev)
    ids = torch.empty(tot, dtype=torch.int64, device=dev)
    ij = torch.empty(tot, 2, dtype=torch.int64, device=dev) if return_index else None
    cfg = _cabi.XrdPixelSampleCfg(F, n, H, W, H0, H1, W0, W1, camera.fx, camera.fy, camera.cx,
                                  camera.cy)
    dp = (C.c_void_p * F)(*[_cabi.ptr(t) for t in depth_imgs])
    cp = (C.c_void_p * F)(*[_cabi.ptr(t) for t in rgb_imgs])
    _cabi.launch_on(dev, 'xrd_sample_pixels', C.byref(cfg), dp, cp, _cabi.ptr(indices),
                    _cabi.ptr(dirs), _cabi.ptr(depth), _cabi.ptr(rgb), _cabi.ptr(ids), _cabi.ptr(ij))
    rays_o, rays_d = _PosedRays.apply(dirs, ids, poses)
    if return_index:
        return rays_o, rays_d, depth, rgb, ij[:, 0], ij[:, 1]
    return rays_o, rays_d, depth, rgb


def get_rays_from_uv(i, j, c2w, fx, fy, cx, cy, device):
    """rays for pixel coords (i: column, j: row); differentiable w.r.t. c2w."""
    c2w = _as_dev(c2w, device)
    dirs = torch.stack([(i - cx) / fx, -(j - cy) / fy, -torch.ones_like(i)],
                       -1).to(device).reshape(-1, 3)
    return rays_from_poses(dirs, None, c2w.reshape(1, 4, 4))


def get_sample_uv(H0, H1, W0, W1, n, depth, color, device='cuda:0',
                  indices=None):
    """n pixels (with replacement, Q7) from rows H0..H1, cols W0..W1.
    ``indices`` (optional, [n] int64 into the cropped region, row-major) makes
    the draw an explicit input for parity runs."""
    depth = _as_dev(depth, device)[H0:H1, W0:W1]
    color = _as_dev(color, device)[H0:H1, W0:W1]
    w = W1 - W0
    if indices is None:
        indices = torch.randint((H1 - H0) * w, (n, ), device=device)
    indices = indices.to(device)
    i = (indices % w + W0).to(torch.float32)
    j = (torch.div(indices, w, rounding_mode='floor') + H0).to(torch.float32)
    d = depth.reshape(-1, 1)[indices]
    c = color.reshape(-1, 3)[indices]
    return i, j, d, c


# ---- colour-gradient pixel selection (Point-SLAM, common.py:74-106, :230-285) ---------------
# skimage.color.rgb2gray / skimage.filters.sobel_h, sobel_v are restated on scipy.ndimage (what
# skimage itself calls): Y = 0.2125 R + 0.7154 G + 0.0721 B; sobel = 3x3 correlation-free
# convolution with [1,2,1]^T x [1,0,-1] / 4, boundary mode 'reflect'.  skimage is not in this
# image: "parity unpinned" at that boundary (float64 here); everything after the gradient image
# (argpartition, region mask, np.random.choice) is the reference's own arithmetic.
_HSOBEL = np.array([[1, 2, 1], [0, 0, 0], [-1, -2, -1]], dtype=np.float64) / 4.0


def rgb2gray_np(image):
    img = np.asarray(image, dtype=np.float64)
    return img[..., 0] * 0.2125 + img[..., 1] * 0.7154 + img[..., 2] * 0.0721


def sobel_magnitude_np(image):
    from scipy import ndimage
    gray = rgb2gray_np(image)
    grad_y = ndimage.convolve(gray, _HSOBEL, mode='reflect')       # sobel_h
    grad_x = ndimage.convolve(gray, _HSOBEL.T, mode='reflect')     # sobel_v
    return np.sqrt(grad_x**2 + grad_y**2)


def get_sample_uv_with_grad(H0, H1, W0, W1, n, image, ratio=15):
    """n flat pixel indices drawn (np.random.choice, no replacement) from the ratio*n pixels
    with the largest colour-gradient magnitude that fall inside rows H0..H1, cols W0..W1."""
    image = np.asarray(image)
    grad_mag = sobel_magnitude_np(image)
    img_size = (image.shape[0], image.shape[1])
    selected_index = np.argpartition(grad_mag, -ratio * n, axis=None)[-ratio * n:]
    indices_h, indices_w = np.unravel_index(selected_index, img_size)
    mask = (indices_h >= H0) & (indices_h < H1) & (indices_w >= W0) & (indices_w < W1)
    indices_h, indices_w = indices_h[mask], indices_w[mask]
    selected_index = np.ravel_multi_index(np.array((indices_h, indices_w)), img_size)
    samples = np.random.choice(range(0, indices_h.shape[0]), size=n, replace=False)
    return selected_index[samples]


def get_samples_with_pixel_grad(camera, n_color, c2w, depth, color, device, Hedge=0, Wedge=0,
                                depth_filter=True, return_index=True, depth_limit=None):
    """Rays through n_color pixels chosen by colour gradient (common.py:230-285); depth /
    colour are the frame's HOST arrays like in the reference."""
    H, W = camera.height, camera.width
    assert n_color > 0, 'invalid number of rays to sample.'
    color_np = np.asarray(color)
    index_color_grad = get_sample_uv_with_grad(Hedge, H - Hedge, Wedge, W - Wedge, n_color,
                                               color_np)
    merged = np.union1d(index_color_grad, [])
    jj, ii = np.unravel_index(merged.astype(int), (H, W))  # row, column
    i = torch.from_numpy(ii).to(device).float()
    j = torch.from_numpy(jj).to(device).float()
    rays_o, rays_d = get_rays_from_uv(i, j, c2w, camera.fx, camera.fy, camera.cx, camera.cy,
                                      device)
    i, j = i.long(), j.long()
    depth_t = _as_dev(depth, device)
    color_t = _as_dev(color, device)
    sample_depth = depth_t[j, i].reshape(-1)
    sample_color = color_t[j, i].reshape(-1, 3)
    if depth_filter:
        mask = sample_depth > 0
        if depth_limit is not None:
            mask = mask & (sample_depth < depth_limit)
        rays_o, rays_d = rays_o[mask], rays_d[mask]
        sample_depth, sample_color = sample_depth[mask], sample_color[mask]
        i, j = i[mask], j[mask]
    if return_index:
        return rays_o, rays_d, sample_depth, sample_color, i.to(torch.int64), j.to(torch.int64)
    return rays_o, rays_d, sample_depth, sample_color


def get_samples(camera, n, c2w, depth, color, device, Hedge=0, Wedge=0,
                depth_filter=False, return_index=False, depth_limit=None,
                indices=None):
    i, j, sample_depth, sample_color = get_sample_uv(
        Hedge, camera.height - Hedge, Wedge, camera.width - Wedge, n, depth,
        color, device=device, indices=indices)
    rays_o, rays_d = get_rays_from_uv(i, j, c2w, camera.fx, camera.fy,
                                      camera.cx, camera.cy, device)
    if depth_filter:
        sample_depth = sample_depth.reshape(-1)
        mask = sample_depth > 0
        if depth_limit is not None:
            mask = mask & (sample_depth < depth_limit)
        rays_o, rays_d = rays_o[mask], rays_d[mask]
        sample_depth, sample_color = sample_depth[mask], sample_color[mask]
        i, j = i[mask], j[mask]
    if return_index:
        return (rays_o, rays_d, sample_depth, sample_color, i.to(torch.int64),
                j.to(torch.int64))
    return rays_o, rays_d, sample_depth, sample_color


def get_rays(camera, c2w, device):
    """All H*W rays of a frame (render_img)."""
    c2w = _as_dev(c2w, device)
    i, j = torch.meshgrid(
        torch.linspace(0, camera.width - 1, camera.width, device=device),
        torch.linspace(0, camera.height - 1, camera.height, device=device),
        indexing='xy')
    dirs = torch.stack([(i - camera.cx) / camera.fx,
                        -(j - camera.cy) / camera.fy, -torch.ones_like(i)], -1)
    dirs = dirs.reshape(camera.height, camera.width, 1, 3)
    rays_d = torch.sum(dirs * c2w[:3, :3], -1)
    rays_o = c2w[:3, -1].expand(rays_d.shape)
    return rays_o, rays_d


def get_camera_rays(H, W, fx, fy=None, cx=None, cy=None, type='OpenGL'):
    """Camera-frame ray directions [H,W,3] (slam/utils/utils.py:28-65)."""
    i, j = torch.meshgrid(torch.arange(W, dtype=torch.float32),
                          torch.arange(H, dtype=torch.float32), indexing='xy')
    if cx is None:
        cx, cy = 0.5 * W, 0.5 * H
    if fy is None:
        fy = fx
    if type == 'OpenGL':
        return torch.stack([(i - cx) / fx, -(j - cy) / fy, -torch.ones_like(i)], -1)
    if type == 'OpenCV':
        return torch.stack([(i - cx) / fx, (j - cy) / fy, torch.ones_like(i)], -1)
    raise NotImplementedError(type)


# ---- Point-SLAM mesh (common.py:622-711): TSDF fusion of the keyframes on the device ----------
def get_mesh_from_RGBD(camera, keyframe_graph, scale=1, frame_tensor=None, device='cuda:0'):
    """get_mesh_from_RGBD (common.py:622-663) on csrc/tsdf.cu: every keyframe, with its current
    pose, is fused into a block-sparse TSDF volume (voxel_length 4/512 * scale, sdf_trunc 0.04 *
    scale, colours (rgb * 255) as uint8); the coloured mesh is translated by compensate_vector.
    -> TriMesh of DEVICE arrays (verts f32 [V,3], faces i32 [F,3], colours f32 [V,3] in [0,1]).
    ``frame_tensor(frame, 'depth' | 'rgb')`` supplies the device images (Algorithm._frame_tensor
    keeps them resident); by default they are uploaded here."""
    from .mesher import TriMesh
    from .tsdf import TSDFVolume, o3d_poses
    if frame_tensor is None:
        frame_tensor = lambda f, w: torch.as_tensor(np.asarray(getattr(f, w), dtype=np.float32)
                                                    ).to(device)
    c2w, w2c = o3d_poses([kf.get_pose().detach().cpu().numpy() for kf in keyframe_graph])
    depth = torch.stack([frame_tensor(kf, 'depth') for kf in keyframe_graph])
    color = torch.stack([(frame_tensor(kf, 'rgb') * 255).to(torch.uint8) for kf in keyframe_graph])
    volume = TSDFVolume(voxel_length=4.0 * scale / 512.0, sdf_trunc=0.04 * scale,
                        device=depth.device)
    volume.integrate(depth, color, c2w, (camera.fx, camera.fy, camera.cx, camera.cy), w2c=w2c)
    verts, faces, colors = volume.extract_triangle_mesh()
    # address the misalignment in open3d marching cubes (common.py:637-639, fp32 here)
    compensate = torch.tensor([-0.0 * scale / 512.0, 2.5 * scale / 512.0, -2.5 * scale / 512.0],
                              dtype=torch.float32, device=verts.device)
    return TriMesh(verts + compensate, faces, vertex_colors=colors)


def clean_mesh(mesh, min_len=100):
    """clean_mesh (common.py:666-711) on the device arrays of get_mesh_from_RGBD: weld
    bit-identical vertices, keep the connected components with >= min_len vertices, drop
    faces that repeat a vertex and duplicate faces (semantics in include/xrdslam_b200.h;
    trimesh's tolerance-based merge is not reproduced).  -> TriMesh of HOST arrays with uint8
    colours (mesher.colors_to_u8)."""
    from .mesher import TriMesh, colors_to_u8
    from .tsdf import clean_mesh_arrays
    v, f, c = clean_mesh_arrays(mesh.vertices, mesh.faces, mesh.vertex_colors, min_len)
    return TriMesh(v.cpu().numpy(), f.cpu().numpy(), vertex_colors=colors_to_u8(c).cpu().numpy())


# ---- save_render_imgs (common.py:429-479): the render metrics on the device -------------------
def save_render_imgs(idx, gt_color_np, gt_depth_np, color_np, depth_np, img_save_dir):
    """The metrics of save_render_imgs on the device (eval_image.render_metrics): -> (psnr,
    ssim, lpips, depth_l1_render) as floats, or None without a rendered colour.  LPIPS is NaN
    (its network weights are not shipped) and no figure is written, so img_save_dir is unused."""
    from .eval_image import render_metrics
    r = render_metrics(gt_color_np, gt_depth_np, color_np, depth_np)
    if r is None:
        return None
    return r['psnr'], r['ssim'], r['lpips'], r['depth_l1']


# ---- cull_mesh (common.py:714-789): the frames' visibility test on the device -----------------
CULL_CHUNK = 16  # frames per depth upload and visibility launch


def cull_w2c(c2w):
    """Rows 0..2 of torch.inverse(c2w) for one f32 [4,4] DEVICE pose, as cull_mesh computes it
    (common.py:745).  linalg.inv_ex is the same inverse without the host-synchronising error
    check."""
    return torch.linalg.inv_ex(c2w)[0][:3]


def _cull_inputs(dataset, estimate_c2w_list, i):
    _, _, depth, c2w = dataset[i]
    if estimate_c2w_list is not None:
        c2w = estimate_c2w_list[i]
    return torch.as_tensor(depth), torch.as_tensor(c2w)


def cull_visibility(dataset, vertices, estimate_c2w_list=None, eval_rec=False, truncation=0.06,
                    device='cuda:0', chunk=CULL_CHUNK):
    """seen u8 [V] on the device: 1 where some frame i < n_imgs sees the vertex (cull_mesh's
    ~whole_mask, semantics in include/xrdslam_b200.h, csrc/cull.cu).  Frames go to the device
    `chunk` at a time through two pinned host buffers and two device buffers, the upload of a
    chunk on a side stream overlapping the visibility launch of the previous one; depth already
    on the device is copied device to device.  Device memory beyond the vertices and `seen` is
    2 * chunk * (H * W + 16) floats, whatever n_imgs is.  No host synchronisation per frame:
    the host waits only before refilling a pinned buffer, for that buffer's previous upload."""
    import ctypes as C
    from . import _cabi
    from ._cabi import XRD_CULL_MAX_FRAMES, XrdCullParams
    dev = torch.device(device)
    _cabi.require_cuda(dev, 'cull_mesh')
    n_imgs = len(estimate_c2w_list) if estimate_c2w_list is not None else len(dataset)
    cam = dataset.get_camera()
    H, W = int(cam.height), int(cam.width)
    P = XrdCullParams(H, W, float(cam.fx), float(cam.fy), float(cam.cx), float(cam.cy),
                      float(truncation), int(bool(eval_rec)))
    verts = _as_dev(vertices, dev).reshape(-1, 3).contiguous()
    V = verts.shape[0]
    seen = torch.zeros(V, dtype=torch.uint8, device=dev)
    if V == 0 or n_imgs == 0:
        return seen
    chunk = max(1, min(int(chunk), XRD_CULL_MAX_FRAMES, n_imgs))
    with torch.cuda.device(dev):
        main = torch.cuda.current_stream(dev)
        side = torch.cuda.Stream(dev)
        depth_d = [torch.empty(chunk, H, W, device=dev) for _ in range(2)]
        pose_d = [torch.empty(chunk, 4, 4, device=dev) for _ in range(2)]
        depth_h = [None, None]
        pose_h = [torch.empty(chunk, 4, 4).pin_memory() for _ in range(2)]
        w2c = torch.empty(chunk, 3, 4, device=dev)
        # the buffers come from the caller's stream: work still queued there may use their
        # memory (a freed block's previous owner), so the side stream starts after it
        side.wait_stream(main)
        uploaded = [None, None]   # side stream: the buffers' last upload is done
        consumed = [None, None]   # main stream: the buffers' last launch is done
        for k, s in enumerate(range(0, n_imgs, chunk)):
            b, n = k % 2, min(chunk, n_imgs - s)
            if uploaded[b] is not None:
                uploaded[b].synchronize()
            on_dev = []
            for j in range(n):
                depth, c2w = _cull_inputs(dataset, estimate_c2w_list, s + j)
                if tuple(depth.shape) != (H, W) or c2w.numel() != 16:
                    raise ValueError(f'frame {s + j}: depth must be [{H},{W}] and c2w [4,4], got '
                                     f'{tuple(depth.shape)} and {tuple(c2w.shape)}')
                if depth.is_cuda:
                    on_dev.append((depth_d[b][j], depth))
                else:
                    if depth_h[b] is None:
                        depth_h[b] = torch.empty(chunk, H, W).pin_memory()
                    depth_h[b][j].copy_(depth)
                if c2w.is_cuda:
                    on_dev.append((pose_d[b][j], c2w.reshape(4, 4)))
                else:
                    pose_h[b][j].copy_(c2w.reshape(4, 4))
            ev = torch.cuda.Event()
            with torch.cuda.stream(side):
                if consumed[b] is not None:
                    side.wait_event(consumed[b])
                if depth_h[b] is not None:
                    depth_d[b][:n].copy_(depth_h[b][:n], non_blocking=True)
                pose_d[b][:n].copy_(pose_h[b][:n], non_blocking=True)
                ev.record(side)
            uploaded[b] = ev
            main.wait_event(ev)
            for dst, t in on_dev:   # device-resident inputs: on the main stream, after the upload
                dst.copy_(t)
            for j in range(n):
                w2c[j].copy_(cull_w2c(pose_d[b][j]))
            _cabi.launch('xrd_cull_visible', _cabi.ptr(verts), V, _cabi.ptr(w2c),
                         _cabi.ptr(depth_d[b]), n, C.byref(P), _cabi.ptr(seen),
                         stream=main.cuda_stream)
            consumed[b] = torch.cuda.Event()
            consumed[b].record(main)
    return seen


def cull_compact(seen, vertices, faces, colors=None):
    """update_faces(~whole_mask[faces].all(1)) + remove_unreferenced_vertices on DEVICE arrays
    (csrc/cull.cu, order-preserving): -> (verts f32 [V',3], faces i32 [F',3], colours [V',...] of
    the input's dtype or None).  One host read: the counts."""
    from . import _cabi
    dev = seen.device
    V = seen.shape[0]
    verts = vertices.to(dev, torch.float32).reshape(-1, 3).contiguous()
    faces = faces.to(dev, torch.int32).reshape(-1, 3).contiguous()
    nF = faces.shape[0]
    if verts.shape[0] != V:
        raise ValueError(f'{verts.shape[0]} vertices but a mask of {V}')
    cb, cbytes = 0, None
    if colors is not None:
        colors = colors.to(dev).contiguous()
        if colors.shape[0] != V:
            raise ValueError('vertex_colors must have one row per vertex')
        row = int(np.prod(colors.shape[1:], dtype=np.int64))
        cb = row * colors.element_size()
        cbytes = colors.reshape(V, row).view(torch.uint8)   # [V, cb]: any element type
    ws, nb = _cabi.workspace(dev, 'cull', V, nF,
                             error=f'cull_mesh: unsupported mesh size V={V}, F={nF}')
    counts = torch.empty(3, dtype=torch.int32, device=dev)
    with torch.cuda.device(dev):
        _cabi.launch_on(dev, 'xrd_cull_count', _cabi.ptr(seen), V, _cabi.ptr(faces), nF,
                        _cabi.ptr(counts), _cabi.ptr(ws), nb)
        V2, F2, bad = counts.tolist()
        if bad:
            raise ValueError(f'cull_mesh: {bad} faces index outside [0, {V})')
        out_v = torch.empty(V2, 3, dtype=torch.float32, device=dev)
        out_f = torch.empty(F2, 3, dtype=torch.int32, device=dev)
        out_c = torch.empty(V2, cb, dtype=torch.uint8, device=dev) if colors is not None else None
        _cabi.launch_on(dev, 'xrd_cull_emit', _cabi.ptr(verts), _cabi.ptr(cbytes), cb, V,
                        _cabi.ptr(faces), nF, _cabi.ptr(out_v), _cabi.ptr(out_c), _cabi.ptr(out_f),
                        _cabi.ptr(ws), nb)
    if colors is not None:
        out_c = out_c.view(colors.dtype).reshape((V2, ) + tuple(colors.shape[1:]))
    return out_v, out_f, out_c


def cull_mesh(dataset, mesh, estimate_c2w_list=None, eval_rec=False, truncation=0.06,
              device='cuda:0', chunk=CULL_CHUNK):
    """cull_mesh (common.py:714-789) on the device: the faces of `mesh` (TriMesh of host numpy
    or device tensor arrays, colours optional) that some frame i < n_imgs sees, n_imgs =
    len(estimate_c2w_list) if given else len(dataset); frame i's depth is dataset[i][2] and its
    pose estimate_c2w_list[i] if given else dataset[i][3].  With eval_rec a vertex hidden more
    than `truncation` behind the frame's depth is not seen.  -> TriMesh of HOST arrays (f32
    vertices); the input mesh is not modified.  trimesh's tolerance merge (process) is not
    reproduced.  Host reads: the mesh counts, once."""
    from .mesher import TriMesh
    dev = torch.device(device)
    tensor = lambda a: (torch.from_numpy(np.ascontiguousarray(a)) if isinstance(a, np.ndarray)
                        else torch.as_tensor(a))
    verts = tensor(mesh.vertices).to(dev, torch.float32).reshape(-1, 3)
    faces = tensor(mesh.faces).to(dev, torch.int32).reshape(-1, 3)
    colors = None if mesh.vertex_colors is None else tensor(mesh.vertex_colors)
    seen = cull_visibility(dataset, verts, estimate_c2w_list, eval_rec, truncation, dev, chunk)
    v, f, c = cull_compact(seen, verts, faces, colors)
    return TriMesh(v.cpu().numpy(), f.cpu().numpy(),
                   vertex_colors=None if c is None else c.cpu().numpy())
