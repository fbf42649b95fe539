"""LineMOD's `fuse` training frames on the GPU (DESIGN.md §4.34).

The reference draws a `fuse` pickle for 40 % of its synthetic LineMOD frames (datasets/linemod/linemod_dataset.py:
85-106): several objects cut out of real frames and pasted into one, made offline by raster_triangle, with the target
object's mask value kept as its label and a camera matrix of its own.  Here the frame is composed where the training
step runs, from a table of object crops kept on the device:

    table = FuseCropTable(frames)                             # once: (rgb, dpt_mm, mask, cls_id) per decoded frame
    keys, K_f, target = draw_fuse_frame(rng, table, cls_id, K, 480, 640)    # the worker, numpy only
    dpt_mm, rgb, labels = fuse_rgbd(table, crop, offset, label, 480, 640)   # the trainer, [B,M] slots

The compositor is specified (the header's ``ffb6d_fuse_rgbd``, restated by oracle/fuse_oracle.py): crops are pasted
whole at integer offsets in slot order, nothing is scaled or rotated, and the target's offset goes into the frame's
principal point, so back-projecting a pasted target pixel with the drawn ``K`` gives the camera-frame point of its
source pixel and the source frame's ``RT`` stays the frame's pose.  Whether raster_triangle's pickles hold the same
pixels is not claimed.  The draws are host code that needs neither CUDA nor torch tensors on the device.
"""
import numpy as np
import torch

from ._lib import lib, launch, FUSE_MAX_CROPS, FUSE_MAX_FRAME_PIXELS, FUSE_MAX_FRAMES, FUSE_MAX_SLOTS

# the training batch's fuse keys (build_ffb6d_train_item(..., crops=)): which frames are fused, and each fused frame's
# slots in paste order: crop index into the table (-1 empty), the crop's top-left corner (row, col) in the frame and
# its label value
FUSE_KEYS = ("fused", "fuse_crop", "fuse_offset", "fuse_label")


class FuseCropTable:
    """Object crops of decoded real frames, packed into device planes for :func:`fuse_rgbd`.

    :param frames: an iterable of ``(rgb [H,W,3] uint8, dpt [H,W] uint16 mm, mask [H,W], cls_id)``.  The silhouette is
      ``mask != 0`` (LineMOD's ``mask/*.png`` is 255 on the object: the reference's ``labels > 0``).  Each frame is
      cropped to the inclusive bounding box of its silhouette as it is read; only the crops are kept.
    :param device: where the planes live (default: the current CUDA device)

    Device planes, crop ``k`` owning pixels ``[off[k], off[k] + h w)`` row-major: ``rgb`` (3 bytes per pixel),
    ``dpt`` (uint16 mm), ``sil`` (uint8 0/1); ``off [n]`` int64 and ``hw [n,2]`` int32.  Host metadata: ``cls [n]``,
    ``origin [n,2]`` (row0, col0 of the crop in its frame) and ``size [n,2]`` (h, w), int64 numpy arrays.
    ``len(table)`` is the crop count, ``table.nbytes`` the device bytes, ``table.classes`` the sorted class ids."""

    def __init__(self, frames, device=None):
        rgb_l, dpt_l, sil_l, cls, origin, size = [], [], [], [], [], []
        for k, frame in enumerate(frames):
            if not isinstance(frame, (tuple, list)) or len(frame) != 4:
                raise ValueError("FuseCropTable: frame %d must be (rgb, dpt, mask, cls_id)" % k)
            rgb, dpt, mask = (t.detach().cpu().numpy() if isinstance(t, torch.Tensor) else np.asarray(t)
                              for t in frame[:3])
            if rgb.dtype != np.uint8 or rgb.ndim != 3 or rgb.shape[2] != 3:
                raise ValueError("FuseCropTable: frame %d: rgb must be uint8 [H,W,3], got %s %s"
                                 % (k, rgb.dtype, rgb.shape))
            if dpt.dtype != np.uint16 or dpt.shape != rgb.shape[:2]:
                raise ValueError("FuseCropTable: frame %d: dpt must be uint16 %s (millimetres), got %s %s"
                                 % (k, rgb.shape[:2], dpt.dtype, dpt.shape))
            if mask.shape != rgb.shape[:2] or not (mask.dtype == np.bool_ or np.issubdtype(mask.dtype, np.number)):
                raise ValueError("FuseCropTable: frame %d: mask must be a numeric [H,W] = %s, got %s %s"
                                 % (k, rgb.shape[:2], mask.dtype, mask.shape))
            sil = mask != 0
            rows, cols = np.flatnonzero(sil.any(1)), np.flatnonzero(sil.any(0))
            if rows.size == 0:
                raise ValueError("FuseCropTable: frame %d: empty silhouette (mask != 0 nowhere)" % k)
            r0, r1, c0, c1 = int(rows[0]), int(rows[-1]), int(cols[0]), int(cols[-1])
            win = (slice(r0, r1 + 1), slice(c0, c1 + 1))
            rgb_l.append(np.ascontiguousarray(rgb[win]).reshape(-1))
            dpt_l.append(np.ascontiguousarray(dpt[win]).reshape(-1))
            sil_l.append(sil[win].astype(np.uint8).reshape(-1))
            cls.append(int(frame[3]))
            origin.append((r0, c0))
            size.append((r1 - r0 + 1, c1 - c0 + 1))
        if not size:
            raise ValueError("FuseCropTable: no frames")
        if len(size) > FUSE_MAX_CROPS:
            raise ValueError("FuseCropTable: %d crops exceed %d" % (len(size), FUSE_MAX_CROPS))
        self.meta = FuseCropMeta(cls, origin, size)
        self.cls, self.origin, self.size, self.classes = (self.meta.cls, self.meta.origin, self.meta.size,
                                                          self.meta.classes)
        npx = self.size[:, 0] * self.size[:, 1]
        dev = torch.device("cuda", torch.cuda.current_device()) if device is None else torch.device(device)
        self.device = dev
        self.rgb = torch.from_numpy(np.concatenate(rgb_l)).to(dev)
        self.dpt = torch.from_numpy(np.concatenate(dpt_l)).to(dev)
        self.sil = torch.from_numpy(np.concatenate(sil_l)).to(dev)
        self.off = torch.from_numpy(np.concatenate([[0], np.cumsum(npx)[:-1]]).astype(np.int64)).to(dev)
        self.hw = torch.from_numpy(self.size.astype(np.int32)).to(dev)
        self.nbytes = sum(t.numel() * t.element_size() for t in (self.rgb, self.dpt, self.sil, self.off, self.hw))

    def __len__(self):
        return len(self.cls)

    def crops_of(self, cls_id):
        """The indices of the crops of class ``cls_id``."""
        return self.meta.crops_of(cls_id)


class FuseCropMeta:
    """A crop table's host metadata alone (``table.meta``): ``cls``, ``origin``, ``size``, ``classes``, all numpy.
    It is what :func:`draw_fuse_frame` reads, and what a DataLoader worker holds: it pickles without CUDA."""

    def __init__(self, cls, origin, size):
        self.cls = np.array(cls, np.int64).reshape(-1)
        self.origin = np.array(origin, np.int64).reshape(-1, 2)
        self.size = np.array(size, np.int64).reshape(-1, 2)
        self.classes = tuple(int(c) for c in np.unique(self.cls))
        self._by_class = {c: np.flatnonzero(self.cls == c) for c in self.classes}

    def __len__(self):
        return len(self.cls)

    def crops_of(self, cls_id):
        """The indices of the crops of class ``cls_id``."""
        return self._by_class.get(int(cls_id), np.zeros(0, np.int64))


def check_crop_indices(table, crop, name="fuse_rgbd"):
    """``ValueError`` unless host crop indices lie in ``[-1, len(table))``.  CUDA indices are not read (that would
    synchronise); the kernel pastes nothing for a slot whose index lies outside the table."""
    if isinstance(crop, torch.Tensor) and crop.is_cuda:
        return
    c = crop.numpy() if isinstance(crop, torch.Tensor) else np.asarray(crop)
    if c.size and (c.min() < -1 or c.max() >= len(table)):
        raise ValueError("%s: crop indices must lie in [-1, %d) (-1: empty slot), got [%d, %d]"
                         % (name, len(table), c.min(), c.max()))


def _device_arg(t, name, dtype, shape, dev):
    """A host array or a CUDA tensor as the kernel reads it: a contiguous CUDA tensor of ``dtype`` and ``shape``."""
    if isinstance(t, torch.Tensor) and t.is_cuda:
        if t.dtype != dtype or tuple(t.shape) != tuple(shape):
            raise ValueError("fuse_rgbd: %s must be %s %s, got %s %s" % (name, dtype, tuple(shape), t.dtype,
                                                                          tuple(t.shape)))
        if t.device != dev:
            raise ValueError("fuse_rgbd: %s is on %s, expected %s" % (name, t.device, dev))
        return t.contiguous()
    a = t.numpy() if isinstance(t, torch.Tensor) else np.asarray(t)
    if tuple(a.shape) != tuple(shape):
        raise ValueError("fuse_rgbd: %s must be %s, got %s" % (name, tuple(shape), tuple(a.shape)))
    return torch.from_numpy(np.ascontiguousarray(a.astype(torch.empty((), dtype=dtype).numpy().dtype))).to(dev)


def fuse_rgbd(table, crop, offset, label, H, W, *, active=None, out=None):
    """Paste crops of ``table`` into ``B`` frames of ``M`` slots each (``ffb6d_fuse_rgbd``, DESIGN.md §4.34).

    :param table: a :class:`FuseCropTable`
    :param crop: ``[B,M]`` int32 crop indices, -1 for an empty slot (host values are checked against the table; a
      CUDA tensor is read on the device, where an index outside the table pastes nothing)
    :param offset: ``[B,M,2]`` int32 (row, col) of each crop's top-left corner in the frame, any values
    :param label: ``[B,M]`` uint8 label values
    :param H, W: the frame size
    :param active: ``[B]`` bools, host or CUDA (None: every frame); an inactive frame is not written
    :param out: None, or ``(dpt_mm [B,H,W] uint16, rgb [B,H,W,3] uint8, labels [B,H,W] uint8)`` contiguous CUDA
      tensors pasted over in place: their pixels that no slot covers are the background
    :return: ``(dpt_mm, rgb, labels)``: new tensors starting from zeros, or the ``out`` tensors.  Pixel ``(r, c)``
      takes the highest slot whose crop holds ``(r - row, c - col)`` with its silhouette set: the crop's depth and
      colour and the slot's label.
    """
    if not isinstance(table, FuseCropTable):
        raise ValueError("fuse_rgbd: table must be a FuseCropTable, got %s" % type(table).__name__)
    H, W = int(H), int(W)
    if not (H >= 1 and W >= 1 and H * W <= FUSE_MAX_FRAME_PIXELS):
        raise ValueError("fuse_rgbd: H=%d W=%d outside 1 <= H, W, H W <= %d" % (H, W, FUSE_MAX_FRAME_PIXELS))
    dev = table.device
    shape_c = tuple(crop.shape) if hasattr(crop, "shape") else np.asarray(crop).shape
    if len(shape_c) != 2:
        raise ValueError("fuse_rgbd: crop must be [B,M], got %s" % (shape_c,))
    B, M = (int(n) for n in shape_c)
    if B > FUSE_MAX_FRAMES:
        raise ValueError("fuse_rgbd: B=%d frames exceed %d" % (B, FUSE_MAX_FRAMES))
    if not 1 <= M <= FUSE_MAX_SLOTS:
        raise ValueError("fuse_rgbd: M=%d slots outside [1, %d]" % (M, FUSE_MAX_SLOTS))
    check_crop_indices(table, crop)
    c = _device_arg(crop, "crop", torch.int32, (B, M), dev)
    o = _device_arg(offset, "offset", torch.int32, (B, M, 2), dev)
    lab = _device_arg(label, "label", torch.uint8, (B, M), dev)
    act = None if active is None else _device_arg(active, "active", torch.bool, (B,), dev).view(torch.uint8)
    if out is None:
        dmm = torch.zeros((B, H, W), dtype=torch.uint16, device=dev)
        rgb = torch.zeros((B, H, W, 3), dtype=torch.uint8, device=dev)
        labels = torch.zeros((B, H, W), dtype=torch.uint8, device=dev)
    else:
        if not isinstance(out, (tuple, list)) or len(out) != 3:
            raise ValueError("fuse_rgbd: out must be (dpt_mm, rgb, labels)")
        dmm, rgb, labels = out
        for t, name, dtype, shape in ((dmm, "out dpt_mm", torch.uint16, (B, H, W)),
                                      (rgb, "out rgb", torch.uint8, (B, H, W, 3)),
                                      (labels, "out labels", torch.uint8, (B, H, W))):
            if (not isinstance(t, torch.Tensor) or t.dtype != dtype or tuple(t.shape) != shape or t.device != dev
                    or not t.is_contiguous()):
                raise ValueError("fuse_rgbd: %s must be a contiguous %s %s tensor on %s, got %s"
                                 % (name, dtype, shape, dev, (t.dtype, tuple(t.shape), t.device)
                                    if isinstance(t, torch.Tensor) else type(t).__name__))
    launch(lib.ffb6d_fuse_rgbd, dev, table.rgb.data_ptr(), table.dpt.data_ptr(), table.sil.data_ptr(),
           table.off.data_ptr(), table.hw.data_ptr(), len(table), c.data_ptr(), o.data_ptr(), lab.data_ptr(), B, M,
           H, W, None if act is None else act.data_ptr(), dmm.data_ptr(), rgb.data_ptr(), labels.data_ptr())
    return dmm, rgb, labels


# ------------------------------------------------------------------------------------------------------ host draws
def draw_fuse_frame(rng, table, target_cls, K, H, W):
    """One `fuse` frame's draws on the host: one crop of each class of ``table`` (uniform among that class's crops), a
    random paste order, and each crop's offset, uniform in rows ``[0, max(H - h, 1))`` and cols ``[0, max(W - w, 1))``.
    The distribution of such a frame, not any stream: the reference's pickles were drawn offline.

    :param rng: a ``numpy.random.RandomState`` (or the ``numpy.random`` module), as the datasets' ``self.rng``
    :param table: a :class:`FuseCropTable` or its ``meta`` (:class:`FuseCropMeta`, what a worker holds)
    :param target_cls: the class the frame trains; it must have crops in the table
    :param K: the ``[3,3]`` camera matrix of the crops' frames
    :return: ``(keys, K_f, target)``: ``keys`` the batch's :data:`FUSE_KEYS` for this frame (``fused`` True,
      ``fuse_crop [M]`` int32, ``fuse_offset [M,2]`` int32, ``fuse_label [M]`` uint8: 1 on the target's slot, 0
      elsewhere, the reference's ``labels == cls_id``), with ``M`` the table's class count; ``K_f`` the frame's
      float64 camera, ``K`` with ``cx += col - col0`` and ``cy += row - row0`` of the target; ``target`` the target's
      crop index (its source frame's ``RT`` is the frame's pose)
    """
    if int(target_cls) not in table.classes:
        raise ValueError("draw_fuse_frame: class %r has no crops in the table (classes %s)"
                         % (target_cls, list(table.classes)))
    picks = []
    for c in table.classes:
        ks = table.crops_of(c)
        picks.append(ks[rng.randint(0, len(ks))])
    picks = np.array(picks, np.int64)
    order = rng.permutation(len(picks))
    crop = picks[order]
    offset = np.zeros((len(crop), 2), np.int32)
    for s, k in enumerate(crop):
        h, w = table.size[k]
        offset[s] = rng.randint(0, max(H - h, 1)), rng.randint(0, max(W - w, 1))
    label = (table.cls[crop] == int(target_cls)).astype(np.uint8)
    t = int(np.flatnonzero(label)[0])
    target = int(crop[t])
    K_f = np.array(K, dtype=np.float64, copy=True)
    K_f[0, 2] += offset[t, 1] - table.origin[target, 1]
    K_f[1, 2] += offset[t, 0] - table.origin[target, 0]
    keys = dict(fused=True, fuse_crop=crop.astype(np.int32), fuse_offset=offset, fuse_label=label)
    return keys, K_f, target


def unfused_keys(table):
    """The :data:`FUSE_KEYS` of a frame that is not fused (a real or a render frame of a batch with ``crops=``);
    ``table`` a :class:`FuseCropTable` or its ``meta``."""
    M = len(table.classes)
    return dict(fused=False, fuse_crop=np.full(M, -1, np.int32), fuse_offset=np.zeros((M, 2), np.int32),
                fuse_label=np.zeros(M, np.uint8))


def draw_linemod_frame_kind(rng, real_ratio=0.3, fuse_ratio=0.4):
    """``real_syn_gen``'s choice of frame kind when both synthetic kinds exist (linemod_dataset.py:85-106): its two
    ``rng.rand()`` draws in its order, ``"real"`` below ``real_ratio``, else ``"fuse"`` below ``fuse_ratio``, else
    ``"render"``.  (The second draw is made only for a synthetic frame, as there.)"""
    if rng.rand() < real_ratio:
        return "real"
    return "fuse" if rng.rand() < fuse_ratio else "render"
