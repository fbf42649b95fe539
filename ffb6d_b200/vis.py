"""Pose and label drawing on the GPU: what the reference's demo and debug views draw.

Mirrors of the reference's helpers that have callers there, same names and argument meaning:

* :func:`get_label_color` -- ``Basic_Utils.get_label_color`` (utils/basic_utils.py:362-423), all three modes, on
  the host; :func:`label_color_list` -- the trainers' ``color_lst`` (train_ycb.py:50-54, train_lm.py:118-122);
* :func:`project_p3d` -- ``Basic_Utils.project_p3d`` (utils/basic_utils.py:268-277), bitwise numpy's float64 result;
* :func:`draw_p2ds` -- ``Basic_Utils.draw_p2ds`` (utils/basic_utils.py:283-295): ``cv2.circle(img, p, r, c, -1)``
  at every point, pixel for pixel;
* :func:`cal_view_pred_pose` -- demo.py's ``cal_view_pred_pose`` (demo.py:85-151) for a whole batch, returning the
  BGR images the demo writes (the network and the vote are :func:`ffb6d_b200.estimate.forward_and_vote`, the steps
  :func:`ffb6d_b200.estimate.estimate_poses` runs); :func:`draw_poses` is its drawing step, sync-free and capturable in a CUDA graph;
* :func:`view_labels` -- the trainers' ``view_labels`` (train_ycb.py:189-204, train_lm.py:198-213), batched.

Everything drawn runs in :func:`ffb6d_b200.ops.project_p3d` and :func:`ffb6d_b200.ops.draw_p2ds`: one launch
projects every point of every object of a batch, and one call draws them, instead of one ``cv2.circle`` per point.
Writing files and ``imshow`` stay with the caller.
"""
import numpy as np
import torch

from . import ops, pose as _pose
from .schedule import check_dataset

# get_label_color's two fixed tables (modes 0 and 1), one colour per class id 0 .. 21, in the order the reference
# hands them to OpenCV (BGR)
_LABEL_COLORS = {
    0: ((255, 255, 255), (180, 105, 255), (0, 255, 0), (0, 0, 255), (0, 255, 255), (255, 0, 255), (180, 105, 255),
        (128, 0, 0), (0, 128, 0), (0, 165, 255), (128, 128, 0), (0, 0, 255), (255, 0, 0), (0, 194, 0), (0, 194, 0),
        (255, 255, 0), (64, 64, 0), (64, 0, 64), (185, 218, 255), (0, 0, 255), (0, 64, 0), (0, 0, 192)),
    1: ((255, 255, 255), (0, 127, 255), (0, 255, 0), (255, 0, 0), (180, 105, 255), (255, 0, 255), (180, 105, 255),
        (128, 0, 0), (0, 128, 0), (185, 218, 255), (128, 128, 0), (0, 0, 255), (255, 0, 0), (0, 194, 0), (0, 194, 0),
        (255, 255, 0), (0, 0, 255), (64, 0, 64), (185, 218, 255), (0, 0, 255), (0, 0, 255), (0, 255, 255)),
}


def get_label_color(cls_id, n_obj=22, mode=0):
    """The colour tuple of class ``cls_id``: mode 0 and 1 look it up in a fixed table of 22 entries (an id outside
    it raises IndexError, negative ids count from the end, as numpy indexing does in the reference); any other mode
    spreads ``n_obj`` colours over the 24-bit range, ``255^3 // n_obj * cls_id`` split into base-255 digits."""
    if mode in (0, 1):
        return _LABEL_COLORS[mode][int(cls_id)]
    m = 255 * 255 * 255 // n_obj * cls_id
    return (int(m // 255 // 255), int((m // 255) % 255), int(m % 255))


def label_color_list(n_objects):
    """The trainers' ``color_lst``: black for label 0, then ``255^3 // (i + 1)`` in base-255 digits for label
    ``i + 1``, ``n_objects`` of them."""
    out = [(0, 0, 0)]
    for i in range(n_objects):
        m = (255 * 255 * 255) // (i + 1)
        out.append((m // (255 * 255), (m // 255) % 255, m % 255))
    return out


def _device():
    return torch.device("cuda", torch.cuda.current_device())


def _points(p3d, cam_scale, dev):
    """``p3d`` as the float tensor the kernel projects, with numpy's dtype for ``p3d * cam_scale``: float32 stays
    float32 when scaled by a Python float, and anything else is promoted the way numpy promotes it."""
    t = p3d if torch.is_tensor(p3d) else torch.as_tensor(np.asarray(p3d))
    np_dtype = np.dtype(str(t.dtype).replace("torch.", "")) if t.dtype != torch.bool else np.dtype(np.bool_)
    scaled = (np.zeros(0, np_dtype) * cam_scale).dtype
    want = torch.float32 if scaled == np.float32 else torch.float64
    if scaled not in (np.float32, np.float64):
        raise ValueError("p3d * cam_scale must be float32 or float64, numpy makes it %s" % scaled)
    return t.to(dev, want).reshape(-1, 3).contiguous()


def _K(K, dev):
    return torch.as_tensor(np.asarray(K, np.float64) if not torch.is_tensor(K) else K).to(dev, torch.float64)


def project_p3d(p3d, cam_scale, K):
    """``p3d [N,3]`` (numpy, or a CUDA tensor) -> int32 ``[N,2]`` CUDA: the pixel ``rint(K p / z)`` of each point
    ``p = p3d * cam_scale``, depths below 1e-8 taken as 1, NaN and coordinates beyond int32 as ``INT32_MIN``, bitwise
    what the reference's numpy code returns.  ``K [3,3]`` is used in float64."""
    dev = p3d.device if torch.is_tensor(p3d) and p3d.is_cuda else _device()
    p = _points(p3d, cam_scale, dev)
    n = p.shape[0]
    if n == 0:
        return torch.empty((0, 2), dtype=torch.int32, device=dev)
    zero = torch.zeros(1, dtype=torch.int32, device=dev)
    count = torch.full((1,), n, dtype=torch.int32, device=dev)
    return ops.project_p3d(p, zero, count, n, _K(K, dev), float(cam_scale))[0]


def draw_p2ds(img, p2ds, r=1, color=((255, 0, 0),)):
    """Draw a filled circle of radius ``r`` at every point of ``p2ds [N,2]`` into ``img [H,W,3]`` uint8, as the
    reference's ``cv2.circle`` loop: points clipped to ``[0,W] x [0,H]``, later points over earlier ones.  ``color``:
    a tuple, or a list of them; a list whose length is not N means ``color[0]`` for every point (the reference's
    rule).  A CUDA ``img`` is drawn in place and returned; a numpy one is copied to the GPU and the drawn copy
    returned.

    One difference: the reference clips the caller's ``p2ds`` in place; here they are left as they were (no
    reference caller reads them again)."""
    dev = img.device if torch.is_tensor(img) and img.is_cuda else _device()
    im = img if torch.is_tensor(img) and img.is_cuda else torch.as_tensor(np.ascontiguousarray(img)).to(dev)
    if im.dim() != 3 or im.shape[2] != 3 or im.dtype != torch.uint8:
        raise ValueError("img must be uint8 [H,W,3], got %s %s" % (im.dtype, tuple(im.shape)))
    p = torch.as_tensor(np.asarray(p2ds) if not torch.is_tensor(p2ds) else p2ds).to(dev, torch.int32).reshape(-1, 2)
    n = p.shape[0]
    if n == 0:
        return im
    if isinstance(color, tuple):
        color = [color]
    col = np.asarray(color[0] if len(color) != n else color, np.int64).reshape(-1, 3).astype(np.uint8)
    colors = torch.as_tensor(col).to(dev).reshape(1, -1, 3) if len(col) == n else torch.as_tensor(col).to(dev)
    zero = torch.zeros(1, dtype=torch.int32, device=dev)
    ops.draw_p2ds(im[None], p[None].contiguous(), zero, zero, torch.full((1,), n, dtype=torch.int32, device=dev), n,
                  torch.full((1,), int(r), dtype=torch.int32, device=dev), colors)
    return im


def _colour_table(colors, dev):
    return torch.as_tensor(np.asarray(colors, np.int64).astype(np.uint8) if not torch.is_tensor(colors)
                           else colors).to(dev, torch.uint8).reshape(-1, 3)


def draw_poses(images, table, frame_cls_ids, present, poses, K, colors, radius=1, mesh_ids=None, ws=None):
    """Draw every predicted object's posed mesh into ``images [B,H,W,3]`` uint8 CUDA, in place, without a host
    synchronisation (capturable in a CUDA graph): the loop of demo.py:120-135 for a whole batch.

    One set per (frame ``b``, slot ``j``) of ``frame_cls_ids [B,n_obj(,1)]`` (the ground-truth ``cls_ids``), drawn in
    slot order: class ``c = frame_cls_ids[b, j]``, enabled where ``present[b, c]`` (``[B,n_cls]``, what
    :func:`ffb6d_b200.pose.cal_batch_poses` returns), mesh ``mesh_ids[c]`` of ``table`` (a
    :class:`ffb6d_b200.pose.MeshTable`, float64 for the demo's rounding; ``mesh_ids`` None: mesh ``c``) posed by
    ``poses[b, c]`` (``[B,n_cls,3,4]`` float64), projected with ``K [3,3]`` and drawn at ``radius`` in colour
    ``colors[c]`` (``[n_cls,3]`` uint8).  Ids out of range draw nothing.  Start and count of every set come from
    indexing ``table.off`` on the device.  ``ws``: a :func:`ffb6d_b200.ops.draw_p2ds_workspace` of ``images``.
    Returns ``images``."""
    dev = images.device
    ids = torch.as_tensor(frame_cls_ids).to(dev)
    B = images.shape[0]
    ids = ids.reshape(B, ids.shape[1], -1)[:, :, 0].long()
    n_obj = ids.shape[1]
    n_cls = present.shape[1]
    ok = (ids >= 0) & (ids < n_cls)
    c = torch.where(ok, ids, 0)
    rows = torch.arange(B, device=dev)[:, None]
    mid = c if mesh_ids is None else torch.as_tensor(mesh_ids).to(dev).long()[c]
    n_mesh = table.off.shape[0] - 1
    ok = ok & (mid >= 0) & (mid < n_mesh) & present[rows, c].bool()
    mid = torch.where(ok, mid, 0)
    start = table.off[mid]
    count = table.off[mid + 1] - start
    S = B * n_obj
    pose = poses[rows, c].reshape(S, 3, 4).contiguous()
    col = _colour_table(colors, dev)[c].reshape(S, 3).contiguous()
    enable = ok.reshape(S).contiguous()
    start, count = start.reshape(S).contiguous(), count.reshape(S).contiguous()
    frame = rows.expand(B, n_obj).reshape(S).to(torch.int32)
    p2ds = ops.project_p3d(table.pts, start, count, table.max_points, _K(K, dev), 1.0, pose, enable)
    rad = torch.full((S,), int(radius), dtype=torch.int32, device=dev)
    return ops.draw_p2ds(images, p2ds, frame, start, count, table.pts.shape[0], rad, col, enable, ws)


def _rgb_hwc(rgb):
    """The network's ``rgb [B,3,H,W]`` as the demo reads it back: ``astype("uint8")`` of each value, HWC."""
    t = rgb if rgb.dtype == torch.uint8 else rgb.to(torch.uint8)
    return t.permute(0, 2, 3, 1).contiguous()


def cal_view_pred_pose(model, item, *, dataset, mesh_pts, mesh_kps, cls_radius=None, K, obj_id=-1):
    """demo.py's ``cal_view_pred_pose`` (demo.py:85-151) for a whole batch: run ``model`` on ``item`` (a dict of
    CUDA tensors with ``rgb [B,3,H,W]``, ``cld_rgb_nrm [B,C,N]`` and ``cls_ids [B,n_obj,1]``; the model returns the
    reference's ``end_points``), vote every frame with :func:`ffb6d_b200.pose.cal_batch_poses` and draw each
    ground-truth object the voting found, with its posed mesh at radius 1 in ``get_label_color(id, mode=2)``.

    ``mesh_pts``: a :class:`~ffb6d_b200.pose.MeshTable` (float64 for bitwise agreement) or the mapping ``id ->
    [P,3]`` one is built from; ``mesh_kps``: a :class:`~ffb6d_b200.pose.VoteTable` or mapping (YCB), the ``[n_kps+1,
    3]`` keypoints of ``obj_id`` (LineMOD); ``cls_radius``: ``config.ycb_r_lst``; ``K [3,3]``; ``dataset``
    ``"ycb"`` or ``"linemod"``; ``obj_id``: the LineMOD object.

    Returns the BGR ``uint8 [B,H,W,3]`` CUDA tensor the demo hands to ``cv2.imwrite``; frame 0 is the demo's image
    (it draws only frame 0).  YCB flips the image to BGR before drawing; LineMOD draws on RGB and flips after, so its
    colour lands reversed, and always draws class 1, with the identity pose where it was not predicted.  Raises
    ValueError, as :func:`~ffb6d_b200.pose.cal_frame_poses`, for a mask id out of range or a predicted class
    without keypoints (YCB; its one host synchronisation)."""
    check_dataset(dataset, "cal_view_pred_pose")
    if dataset == "linemod" and obj_id < 0:
        raise ValueError("LineMOD needs the object's obj_id")
    from .estimate import forward_and_vote
    model.eval()
    end_points, vt, (present, _, _, poses) = forward_and_vote(model, item, dataset, mesh_kps, cls_radius)
    with torch.no_grad():
        segs = end_points["pred_rgbd_segs"]
        dev = segs.device
        table = mesh_pts if isinstance(mesh_pts, _pose.MeshTable) else _pose.MeshTable(mesh_pts, dev, torch.float64)
        images = _rgb_hwc(item["rgb"])
        ids = item["cls_ids"]
        if dataset == "ycb":
            n_cls = segs.shape[1]
            bad = torch.stack((torch.isnan(poses[:, 0]).any(), (present & ~vt.has_mesh.bool()[None]).any()))
            bad_id, no_kps = bad.cpu().tolist()
            if bad_id:
                raise ValueError("the mask holds a class id outside [0, %d)" % n_cls)
            if no_kps:
                raise ValueError("no mesh keypoints for a predicted class")
            colors = [get_label_color(c, n_obj=22, mode=2) for c in range(n_cls)]
            images = images.flip(-1).contiguous()
            return draw_poses(images, table, ids, present, poses, K, colors)
        eye = torch.eye(3, 4, dtype=torch.float64, device=dev)
        B = segs.shape[0]
        pose1 = torch.where(present[:, 1, None, None], poses[:, 1], eye)
        lm_poses = torch.stack((eye.expand(B, 3, 4), pose1), 1).contiguous()
        lm_present = torch.zeros((B, 2), dtype=torch.bool, device=dev)
        lm_present[:, 1] = True
        colors = [(0, 0, 0), get_label_color(obj_id, n_obj=22, mode=2)]
        mesh_ids = torch.tensor([-1, int(obj_id)], device=dev)
        draw_poses(images, table, ids, lm_present, lm_poses, K, colors, mesh_ids=mesh_ids)
        return images.flip(-1).contiguous()


def view_labels(rgb, cld, labels, K, n_objects=22):
    """The trainers' ``view_labels`` for a batch: black ``uint8 [B,H,W,3]`` CUDA images (``H, W`` from ``rgb
    [B,3,H,W]``) with every point of ``cld [B,3,N]`` (float32, channel-major as ``cld_rgb_nrm[:, :3]``) projected
    with ``K`` and drawn at radius 3 in ``label_color_list(n_objects)[labels[b, i]]`` (label 0 black, drawn like the
    others, so it covers earlier points).  A label outside ``[0, n_objects]`` raises ValueError (the reference would
    index past its list, or from its end for a negative label); that check is one host synchronisation."""
    dev = cld.device
    B, H, W = rgb.shape[0], rgb.shape[2], rgb.shape[3]
    N = cld.shape[2]
    lab = torch.as_tensor(labels).to(dev).reshape(B, N).long()
    lo_hi = torch.stack((lab.min(), lab.max())).cpu().tolist() if lab.numel() else [0, 0]
    if lo_hi[0] < 0 or lo_hi[1] > n_objects:
        raise ValueError("labels must lie in [0, %d], got [%d, %d]" % (n_objects, lo_hi[0], lo_hi[1]))
    images = torch.zeros((B, H, W, 3), dtype=torch.uint8, device=dev)
    if N == 0:
        return images
    pts = cld.permute(0, 2, 1).reshape(B * N, 3).to(torch.float32).contiguous()
    start = torch.arange(B, dtype=torch.int32, device=dev) * N
    count = torch.full((B,), N, dtype=torch.int32, device=dev)
    p2ds = ops.project_p3d(pts, start, count, N, _K(K, dev), 1.0)
    col = _colour_table(label_color_list(n_objects), dev)[lab].contiguous()
    frame = torch.arange(B, dtype=torch.int32, device=dev)
    rad = torch.full((B,), 3, dtype=torch.int32, device=dev)
    return ops.draw_p2ds(images, p2ds, frame, start, count, B * N, rad, col)
