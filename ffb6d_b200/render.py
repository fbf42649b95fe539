"""Synthetic RGB-D frames of vertex-coloured meshes on the GPU (DESIGN.md §4.31).

The reference trains LineMOD mostly on synthetic frames: ``real_syn_gen`` draws a `render` pickle, made offline by
raster_triangle, for at least 60 % of its synthetic draws (datasets/linemod/linemod_dataset.py:85-106).  Here the
frame is rendered where the training step runs:

    table = RenderMeshTable([(xyz_m, faces, rgb)])               # once: the meshes on the device
    depth, rgb, labels = render_rgbd(table, mesh_idx, RTs, label, K, 480, 640)

The rasteriser is specified (the header's ``ffb6d_render_rgbd``, restated by oracle/render_oracle.py) and its frames
are that oracle's bit for bit; whether raster_triangle draws the same pixels is not claimed.  Mesh parsing stays with
the caller, as it does for :mod:`ffb6d_b200.objinfo`.

Textured meshes -- YCB's, or any scanned object: positions, per-vertex UVs and an RGB texture -- render through the
same call from a :class:`TexturedMeshTable` (DESIGN.md §4.35): same depth and labels, the colour sampled from the
texture's mip chain (``ffb6d_render_rgbd_textured``, restated by oracle/textured_render_oracle.py).
"""
import numpy as np
import torch

from ._lib import (lib, launch, workspace, RND_MAX_SLOTS, RND_MAX_MESH_VERTS, RND_MAX_FRAME_FACES, RND_MAX_TEX_SIDE,
                   RND_MAX_TEX_LEVELS, RND_MAX_UV)
from .ops import _intrinsics_arg, _need_cuda, _tensor

# the training batch's render keys (build_ffb6d_train_item(..., meshes=)): which frames are renders, and each render's
# slots: mesh index into the table (-1 empty), pose (object to camera, metres) and label value
RENDER_KEYS = ("rendered", "render_mesh", "render_RTs", "render_label")
# raster_triangle's renders and the datasets' near plane are not stated; 1 cm is the default here
Z_NEAR = 0.01


class RenderMeshTable:
    """Vertex-coloured meshes packed into device buffers for :func:`render_rgbd`.

    :param meshes: a list of ``(xyz [V,3] metres, faces [F,3] vertex indices, rgb [V,3] uint8)`` (numpy arrays or
      tensors).  The face indices are checked on the host, once: each must lie in ``[0, V)``.
    :param device: where the buffers live (default: the current CUDA device)

    ``len(table)`` is the number of meshes; ``max_verts`` / ``max_faces`` the largest mesh's counts."""

    def __init__(self, meshes, device=None):
        if isinstance(meshes, tuple) and len(meshes) == 3 and not isinstance(meshes[0], tuple):
            raise ValueError("RenderMeshTable: meshes must be a list of (xyz, faces, rgb) tuples")
        meshes = list(meshes)
        if not meshes:
            raise ValueError("RenderMeshTable: no meshes")
        xyz_l, face_l, rgb_l, nv, nf = [], [], [], [], []
        for k, mesh in enumerate(meshes):
            if len(mesh) != 3:
                raise ValueError("RenderMeshTable: mesh %d must be (xyz, faces, rgb)" % k)
            xyz, faces, rgb = (t.detach().cpu().numpy() if isinstance(t, torch.Tensor) else np.asarray(t) for t in mesh)
            if xyz.ndim != 2 or xyz.shape[1] != 3 or not 1 <= len(xyz) <= RND_MAX_MESH_VERTS:
                raise ValueError("RenderMeshTable: mesh %d: xyz must be [V,3] with V >= 1, got %s" % (k, xyz.shape))
            if rgb.shape != xyz.shape or rgb.dtype != np.uint8:
                raise ValueError("RenderMeshTable: mesh %d: rgb must be uint8 [V,3] = %s, got %s %s"
                                 % (k, xyz.shape, rgb.dtype, rgb.shape))
            if faces.ndim != 2 or faces.shape[1] != 3 or len(faces) < 1 or not np.issubdtype(faces.dtype, np.integer):
                raise ValueError("RenderMeshTable: mesh %d: faces must be integer [F,3] with F >= 1, got %s %s"
                                 % (k, faces.dtype, faces.shape))
            if faces.min() < 0 or faces.max() >= len(xyz):
                raise ValueError("RenderMeshTable: mesh %d: face indices must lie in [0, %d), got [%d, %d]"
                                 % (k, len(xyz), faces.min(), faces.max()))
            xyz_l.append(xyz.astype(np.float32))
            face_l.append(faces.astype(np.int32))
            rgb_l.append(rgb)
            nv.append(len(xyz))
            nf.append(len(faces))
        dev = torch.device("cuda", torch.cuda.current_device()) if device is None else torch.device(device)
        self.device = dev
        self.max_verts, self.max_faces = max(nv), max(nf)
        self.n_verts, self.n_faces = tuple(nv), tuple(nf)
        # row-major whatever the callers' layouts (a column-major array would keep its strides through from_numpy)
        self.xyz = torch.from_numpy(np.ascontiguousarray(np.concatenate(xyz_l))).to(dev)
        self.rgb = torch.from_numpy(np.ascontiguousarray(np.concatenate(rgb_l))).to(dev)
        self.faces = torch.from_numpy(np.ascontiguousarray(np.concatenate(face_l))).to(dev)
        self.vert_off = torch.from_numpy(np.concatenate([[0], np.cumsum(nv)]).astype(np.int64)).to(dev)
        self.face_off = torch.from_numpy(np.concatenate([[0], np.cumsum(nf)]).astype(np.int64)).to(dev)

    def __len__(self):
        return len(self.n_verts)


def _mesh_arrays(name, k, mesh, n_parts, parts):
    if len(mesh) != n_parts:
        raise ValueError("%s: mesh %d must be (%s)" % (name, k, parts))
    return [t.detach().cpu().numpy() if isinstance(t, torch.Tensor) else np.asarray(t) for t in mesh]


def _check_geometry(name, k, xyz, faces):
    if xyz.ndim != 2 or xyz.shape[1] != 3 or not 1 <= len(xyz) <= RND_MAX_MESH_VERTS:
        raise ValueError("%s: mesh %d: xyz must be [V,3] with V >= 1, got %s" % (name, k, xyz.shape))
    if faces.ndim != 2 or faces.shape[1] != 3 or len(faces) < 1 or not np.issubdtype(faces.dtype, np.integer):
        raise ValueError("%s: mesh %d: faces must be integer [F,3] with F >= 1, got %s %s"
                         % (name, k, faces.dtype, faces.shape))
    if faces.min() < 0 or faces.max() >= len(xyz):
        raise ValueError("%s: mesh %d: face indices must lie in [0, %d), got [%d, %d]"
                         % (name, k, len(xyz), faces.min(), faces.max()))


def tex_levels(th, tw):
    """The sizes ``[(h, w), ...]`` of a ``th x tw`` texture's mip chain, level 0 first, down to 1 x 1."""
    n = max(int(th), int(tw)).bit_length()
    return [(max(1, int(th) >> l), max(1, int(tw) >> l)) for l in range(n)]


class TexturedMeshTable:
    """Textured meshes packed into device buffers for :func:`render_rgbd` (DESIGN.md §4.35), each texture with its
    mip chain built on the device (``ffb6d_render_texture_mips``), once.

    :param meshes: a list of ``(xyz [V,3] metres, faces [F,3] vertex indices, uv [V,2], texture [Th,Tw,3] uint8)``
      (numpy arrays or tensors): per-vertex UVs in the .obj / trimesh convention (``v = 0`` the bottom row of the
      decoded image; seams split into separate vertices, as ``trimesh.load(path).visual.uv`` has them) and the RGB
      texture as decoded.  Checked on the host, once: face indices in ``[0, V)``, UVs finite with ``|uv| <= 2^16``
      after rounding to float32, texture sides in ``[1, 16384]``, three channels (RGBA is refused).
    :param device: where the buffers live (default: the current CUDA device).  A table on the CPU holds level 0 only
      and cannot be rendered; it serves host-side checks.

    Not a :class:`RenderMeshTable`: the training paths (``meshes=``) take vertex-coloured meshes only.
    ``len(table)`` is the number of meshes; ``max_verts`` / ``max_faces`` the largest mesh's counts, ``max_tex_side``
    the largest texture side, ``tex_hw`` the ``(Th, Tw)`` of each texture."""

    def __init__(self, meshes, device=None):
        name = "TexturedMeshTable"
        if isinstance(meshes, tuple) and len(meshes) == 4 and not isinstance(meshes[0], tuple):
            raise ValueError("%s: meshes must be a list of (xyz, faces, uv, texture) tuples" % name)
        meshes = list(meshes)
        if not meshes:
            raise ValueError("%s: no meshes" % name)
        xyz_l, face_l, uv_l, tex_l, nv, nf = [], [], [], [], [], []
        for k, mesh in enumerate(meshes):
            xyz, faces, uv, tex = _mesh_arrays(name, k, mesh, 4, "xyz, faces, uv, texture")
            _check_geometry(name, k, xyz, faces)
            if uv.shape != (len(xyz), 2) or not np.issubdtype(uv.dtype, np.floating):
                raise ValueError("%s: mesh %d: uv must be floating [V,2] = (%d, 2), got %s %s"
                                 % (name, k, len(xyz), uv.dtype, uv.shape))
            uv = uv.astype(np.float32)
            if not np.all(np.abs(uv) <= RND_MAX_UV):              # NaN fails too
                raise ValueError("%s: mesh %d: uv must be finite with |uv| <= %d" % (name, k, RND_MAX_UV))
            if tex.ndim == 3 and tex.shape[2] == 4:
                raise ValueError("%s: mesh %d: RGBA texture %s: pass the RGB channels (alpha is not rendered)"
                                 % (name, k, tex.shape))
            if tex.ndim != 3 or tex.shape[2] != 3 or tex.dtype != np.uint8:
                raise ValueError("%s: mesh %d: texture must be uint8 [Th,Tw,3], got %s %s" % (name, k, tex.dtype,
                                                                                            tex.shape))
            if not (1 <= tex.shape[0] <= RND_MAX_TEX_SIDE and 1 <= tex.shape[1] <= RND_MAX_TEX_SIDE):
                raise ValueError("%s: mesh %d: texture sides must lie in [1, %d], got %dx%d"
                                 % (name, k, RND_MAX_TEX_SIDE, tex.shape[0], tex.shape[1]))
            xyz_l.append(xyz.astype(np.float32))
            face_l.append(faces.astype(np.int32))
            uv_l.append(uv)
            tex_l.append(tex)
            nv.append(len(xyz))
            nf.append(len(faces))
        dev = torch.device("cuda", torch.cuda.current_device()) if device is None else torch.device(device)
        self.device = dev
        self.max_verts, self.max_faces = max(nv), max(nf)
        self.n_verts, self.n_faces = tuple(nv), tuple(nf)
        self.xyz = torch.from_numpy(np.ascontiguousarray(np.concatenate(xyz_l))).to(dev)
        self.uv = torch.from_numpy(np.ascontiguousarray(np.concatenate(uv_l))).to(dev)
        self.faces = torch.from_numpy(np.ascontiguousarray(np.concatenate(face_l))).to(dev)
        self.vert_off = torch.from_numpy(np.concatenate([[0], np.cumsum(nv)]).astype(np.int64)).to(dev)
        self.face_off = torch.from_numpy(np.concatenate([[0], np.cumsum(nf)]).astype(np.int64)).to(dev)
        # every mesh's chain, level after level, mesh after mesh; unused level slots repeat the last offset
        hw = [t.shape[:2] for t in tex_l]
        off = np.zeros((len(tex_l), RND_MAX_TEX_LEVELS), np.int64)
        total = 0
        for m, (th, tw) in enumerate(hw):
            for l, (h, w) in enumerate(tex_levels(th, tw)):
                off[m, l:] = total
                total += h * w
        self.tex_hw = torch.from_numpy(np.asarray(hw, np.int32).reshape(-1, 2)).to(dev)
        self.tex_off = torch.from_numpy(off).to(dev)
        self.max_tex_side = int(max(max(h, w) for h, w in hw))
        self.tex = torch.zeros(total * 3, dtype=torch.uint8, device=dev)
        for m, t in enumerate(tex_l):
            n = t.shape[0] * t.shape[1] * 3
            self.tex[off[m, 0] * 3:off[m, 0] * 3 + n].copy_(torch.from_numpy(np.ascontiguousarray(t).reshape(-1)))
        if dev.type == "cuda":
            launch(lib.ffb6d_render_texture_mips, dev, self.tex.data_ptr(), self.tex_hw.data_ptr(),
                   self.tex_off.data_ptr(), len(tex_l), self.max_tex_side)

    def __len__(self):
        return len(self.n_verts)

    def level(self, m, l):
        """Level ``l`` of mesh ``m``'s mip chain as a ``[h, w, 3]`` uint8 view of the table's buffer."""
        th, tw = (int(n) for n in self.tex_hw[m].tolist())
        h, w = tex_levels(th, tw)[l]
        o = int(self.tex_off[m, l]) * 3
        return self.tex[o:o + h * w * 3].view(h, w, 3)


def check_mesh_indices(table, mesh_idx, name="render_rgbd"):
    """``ValueError`` unless host mesh indices lie in ``[-1, len(table))``.  CUDA indices are not read (that would
    synchronise); the kernel draws nothing for a slot whose index lies outside the table."""
    if isinstance(mesh_idx, torch.Tensor) and mesh_idx.is_cuda:
        return
    m = mesh_idx.numpy() if isinstance(mesh_idx, torch.Tensor) else np.asarray(mesh_idx)
    if m.size and (m.min() < -1 or m.max() >= len(table)):
        raise ValueError("%s: mesh indices must lie in [-1, %d) (-1: empty slot), got [%d, %d]"
                         % (name, len(table), m.min(), m.max()))


def _device_arg(t, name, dtype, shape, dev):
    """A host array or a CUDA tensor as the kernel reads it: a contiguous CUDA tensor of ``dtype`` and ``shape``."""
    if isinstance(t, torch.Tensor) and t.is_cuda:
        return _tensor(t, name, dtype, shape, dev)
    a = t.numpy() if isinstance(t, torch.Tensor) else np.asarray(t)
    if tuple(a.shape) != tuple(shape):
        raise ValueError("%s must be %s, got %s" % (name, tuple(shape), tuple(a.shape)))
    return torch.from_numpy(np.ascontiguousarray(a.astype(torch.empty((), dtype=dtype).numpy().dtype))).to(dev)


def render_rgbd(table, mesh_idx, RTs, label, K, H, W, *, z_near=Z_NEAR, active=None, out=None):
    """Render ``B`` frames of ``M`` mesh instances each (``ffb6d_render_rgbd``, DESIGN.md §4.31).

    :param table: a :class:`RenderMeshTable`, or a :class:`TexturedMeshTable` (on a CUDA device): then each drawn
      pixel's colour is its texture's, filtered through the mip chain (``ffb6d_render_rgbd_textured``, §4.35), and
      depth and labels are what a :class:`RenderMeshTable` of the same geometry gives
    :param mesh_idx: ``[B,M]`` int32 indices into the table, -1 for an empty slot (host values are checked against the
      table; a CUDA tensor is read on the device, where an index outside the table draws nothing)
    :param RTs: ``[B,M,3,4]`` float32 poses, object to camera, metres; :param label: ``[B,M]`` uint8 label values
    :param K: the camera as :func:`ffb6d_b200.ops.backproject` takes it (host ``[3,3]`` / ``[B,3,3]``, or device
      float64 ``(fx, fy, cx, cy)`` ``[4]`` / ``[B,4]``)
    :param H, W: the frame size; :param z_near: the near plane in metres (>= 0.001); a face with a vertex nearer is
      not drawn
    :param active: ``[B]`` bools, host or CUDA (None: every frame); an inactive frame's outputs are not written
    :param out: None, or ``(dpt_mm [B,H,W] uint16, rgb [B,H,W,3] uint8, labels [B,H,W] uint8)`` CUDA tensors written
      in place, the depth as LineMOD's ``dpt_mm`` (``trunc(fl32(depth * 1000.0f))``)
    :return: ``(depth [B,H,W] float32 metres, rgb [B,H,W,3] uint8, labels [B,H,W] uint8)``, 0 where no face is drawn;
      with ``out``, those tensors.  Inactive frames of a new output are zeros.
    """
    textured = isinstance(table, TexturedMeshTable)
    if not (textured or isinstance(table, RenderMeshTable)):
        raise ValueError("render_rgbd: table must be a RenderMeshTable or a TexturedMeshTable, got %s"
                         % type(table).__name__)
    if textured and table.device.type != "cuda":
        raise ValueError("render_rgbd: a TexturedMeshTable must live on a CUDA device, got %s" % table.device)
    H, W = int(H), int(W)
    dev = table.device
    check_mesh_indices(table, mesh_idx)
    shape_m = tuple(mesh_idx.shape) if hasattr(mesh_idx, "shape") else np.asarray(mesh_idx).shape
    if len(shape_m) != 2:
        raise ValueError("render_rgbd: mesh_idx must be [B,M], got %s" % (shape_m,))
    B, M = (int(n) for n in shape_m)
    if not 1 <= M <= RND_MAX_SLOTS:
        raise ValueError("render_rgbd: M=%d slots outside [1, %d]" % (M, RND_MAX_SLOTS))
    if M * table.max_faces > RND_MAX_FRAME_FACES:
        raise ValueError("render_rgbd: M * max_faces = %d exceeds %d" % (M * table.max_faces, RND_MAX_FRAME_FACES))
    z = float(z_near)
    if not (z >= 0.001 and np.isfinite(z)):
        raise ValueError("render_rgbd: z_near must be finite and >= 0.001 m, got %r" % (z_near,))
    midx = _device_arg(mesh_idx, "mesh_idx", torch.int32, (B, M), dev)
    rts = _device_arg(RTs, "RTs", torch.float32, (B, M, 3, 4), dev)
    lab = _device_arg(label, "label", torch.uint8, (B, M), dev)
    act = None if active is None else _device_arg(active, "active", torch.bool, (B,), dev).to(torch.uint8)
    if out is None:
        depth = torch.zeros((B, H, W), dtype=torch.float32, device=dev)
        rgb = torch.zeros((B, H, W, 3), dtype=torch.uint8, device=dev)
        labels = torch.zeros((B, H, W), dtype=torch.uint8, device=dev)
        dmm = None
    else:
        if not isinstance(out, (tuple, list)) or len(out) != 3:
            raise ValueError("render_rgbd: out must be (dpt_mm, rgb, labels)")
        dmm, rgb, labels = out
        for t, name, dtype, shape in ((dmm, "out dpt_mm", torch.uint16, (B, H, W)),
                                      (rgb, "out rgb", torch.uint8, (B, H, W, 3)),
                                      (labels, "out labels", torch.uint8, (B, H, W))):
            _need_cuda(t, name)
            if t.dtype != dtype or tuple(t.shape) != shape or t.device != dev or not t.is_contiguous():
                raise ValueError("render_rgbd: %s must be contiguous %s %s on %s, got %s %s on %s"
                                 % (name, dtype, shape, dev, t.dtype, tuple(t.shape), t.device))
        depth = None
    intr, per_frame = _intrinsics_arg(K, B, dev)
    nbytes = int(lib.ffb6d_render_workspace_bytes(B, M, H, W, table.max_verts, table.max_faces))
    if B and not nbytes:
        raise ValueError("render_rgbd: sizes outside the kernel's limits (B=%d M=%d H=%d W=%d)" % (B, M, H, W))
    ws = workspace(nbytes, dev)
    frame = (midx.data_ptr(), rts.data_ptr(), lab.data_ptr(), B, M, intr.data_ptr(), per_frame, H, W, z,
             None if act is None else act.data_ptr(), None if depth is None else depth.data_ptr(),
             None if dmm is None else dmm.data_ptr(), rgb.data_ptr(), labels.data_ptr(), ws.data_ptr(), nbytes)
    if textured:
        launch(lib.ffb6d_render_rgbd_textured, dev, table.xyz.data_ptr(), table.uv.data_ptr(), table.faces.data_ptr(),
               table.vert_off.data_ptr(), table.face_off.data_ptr(), table.tex.data_ptr(), table.tex_hw.data_ptr(),
               table.tex_off.data_ptr(), table.max_tex_side, len(table), table.max_verts, table.max_faces, *frame)
    else:
        launch(lib.ffb6d_render_rgbd, dev, table.xyz.data_ptr(), table.rgb.data_ptr(), table.faces.data_ptr(),
               table.vert_off.data_ptr(), table.face_off.data_ptr(), len(table), table.max_verts, table.max_faces,
               *frame)
    return (depth if out is None else dmm), rgb, labels
