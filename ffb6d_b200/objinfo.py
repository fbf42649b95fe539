"""The object tables of the reference's mesh tool, utils/dataset_tools/gen_obj_info.py.

For each object, ``gen_one_mesh_info`` (gen_obj_info.py:92-117) writes the 3D bounding box corners, the radius, the
centre and the farthest-point keypoints of the mesh's vertices; the datasets and ``cal_frame_poses`` read them back
(``Basic_Utils.get_kps`` / ``get_ctr``, utils/basic_utils.py:572-640).  The box arithmetic is restated here with the
expressions of ``MeshUtils`` (utils/dataset_tools/utils.py:88-115); the keypoints come from
:func:`ffb6d_b200.ops.farthest_point_sampling` on the GPU.

Mesh files are not read here: the caller passes the vertex array ``[N,3]`` (what ``MeshUtils.get_p3ds_from_mesh``
returns, already divided by ``scale2m``).  The tool's textured keypoints -- ORB corners of renders from a sphere of
views, lifted onto the mesh and reduced by farthest point sampling (rgbd_rnder_sift_kp3ds.py:138-166,
gen_obj_info.py:119-126), the table the datasets read with ``use_orbfps`` -- run on the GPU through
:func:`textured_kp3ds` (DESIGN.md §4.32); the tool's ``--extractor SIFT`` (the paper's SIFT-FPS keypoints) through
``textured_kp3ds(..., extractor="SIFT")`` (§4.33); a textured object (the tool's ``--use_pyrender`` branch,
pyrender_sift_kp3ds.py:104-132, YCB's meshes) through ``textured_kp3ds`` of a
:class:`~ffb6d_b200.render.TexturedMeshTable` (§4.35), centred as that branch centres it.  Plain numpy; only :func:`gen_obj_info` and :func:`textured_kp3ds` load
the CUDA library.
"""
import math
import os

import numpy as np

# the tool's camera (rgbd_rnder_sift_kp3ds.py test(): --K, --h, --w) and its short-view rule (:80)
TOOL_K = np.array([[700, 0, 320], [0, 700, 240], [0, 0, 1]], np.int64)
TOOL_H, TOOL_W = 480, 640
MIN_RENDER_PIXELS = 500


def get_3D_bbox(pcld, small=False):
    """The eight corners ``[8,3]`` of the axis-aligned box of ``pcld [N,3]`` (``MeshUtils.get_3D_bbox``)."""
    min_x, max_x = pcld[:, 0].min(), pcld[:, 0].max()
    min_y, max_y = pcld[:, 1].min(), pcld[:, 1].max()
    min_z, max_z = pcld[:, 2].min(), pcld[:, 2].max()
    bbox = np.array([
        [min_x, min_y, min_z],
        [min_x, min_y, max_z],
        [min_x, max_y, min_z],
        [min_x, max_y, max_z],
        [max_x, min_y, min_z],
        [max_x, min_y, max_z],
        [max_x, max_y, min_z],
        [max_x, max_y, max_z],
    ])
    if small:
        center = np.mean(bbox, 0)
        bbox = (bbox - center[None, :]) * 2.0 / 3.0 + center[None, :]
    return bbox


def get_r(bbox):
    """Half the diagonal of the box (``MeshUtils.get_r``)."""
    return np.linalg.norm(bbox[7, :] - bbox[0, :]) / 2.0


def get_centers_3d(corners_3d):
    """The centre of the box (``MeshUtils.get_centers_3d``)."""
    centers_3d = (np.max(corners_3d, 0) + np.min(corners_3d, 0)) / 2
    return centers_3d


def camera_positions(n1, n2, r):
    """``PoseUtils.CameraPositions``: ``n1 x n2`` camera positions on a sphere of radius ``r`` (numpy's types follow
    ``r``'s, as in the tool, where ``r`` is a float32 scalar)."""
    theta_list = np.linspace(0.1, np.pi, n1 + 1)[:-1]
    phi_list = np.linspace(0, 2 * np.pi, n2 + 1)[:-1]
    return [(r * math.sin(theta) * math.cos(phi), r * math.sin(theta) * math.sin(phi), r * math.cos(theta))
            for theta in theta_list for phi in phi_list]


def camera_pose(T):
    """``PoseUtils.getCameraPose``: the OpenGL camera at ``T`` looking at the origin, ``[4,4]`` float64."""
    z_direct = np.array(T)
    z_direct = z_direct / np.linalg.norm(z_direct)
    x_direct = -np.cross(z_direct, np.array([0, 0, 1]))
    x_direct = x_direct / np.linalg.norm(x_direct)
    y_direct = np.cross(z_direct, x_direct)
    y_direct = y_direct / np.linalg.norm(y_direct)
    camera = np.eye(4)
    camera[:3, :3] = np.transpose(np.array([x_direct, y_direct, z_direct]))
    camera[:3, 3] = T
    return camera


def o2c_pose(cam_pose, obj_pose=np.eye(4)):
    """``PoseUtils.get_o2c_pose_cv(cam_pose, obj_pose)``: object to OpenCV camera, ``[4,4]`` float64; ``obj_pose`` the
    object's pose in the world (the raster_triangle branch's identity, or the pyrender branch's ``T(-mean)``)."""
    R_bcam2cv = np.array([(1, 0, 0), (0, -1, 0), (0, 0, -1)])
    R_world2bcam = cam_pose[:3, :3].T
    T_world2bcam = -1 * R_world2bcam @ cam_pose[:3, 3]
    RT = np.eye(4)
    RT[:3, :3] = R_bcam2cv @ R_world2bcam
    RT[:3, 3] = R_bcam2cv @ T_world2bcam
    return np.matmul(RT, obj_pose)


def sphere_poses(radius, n_longitude=3, n_latitude=3, centre=None):
    """The tool's views of an object whose box has radius ``radius`` (``get_r``; a float32 scalar for float32
    vertices, as in the tool): ``[n_longitude * n_latitude, 4, 4]`` float64 object-to-camera poses on a sphere of
    radius ``radius / 0.035 * 0.18`` (rgbd_rnder_sift_kp3ds.py:147-158).  With ``centre`` (``[3]``) the object is
    first moved by ``-centre``, as the pyrender branch moves it by its vertices' mean (pyrender_sift_kp3ds.py:105-120)."""
    sph_r = radius / 0.035 * 0.18
    if centre is None:
        return np.stack([o2c_pose(camera_pose(p)) for p in camera_positions(n_longitude, n_latitude, sph_r)])
    obj_pose = np.eye(4)
    obj_pose[:3, 3] = -1.0 * np.asarray(centre, np.float64)
    return np.stack([o2c_pose(camera_pose(p), obj_pose)
                     for p in camera_positions(n_longitude, n_latitude, sph_r)])


def textured_kp3ds(table, mesh, K=TOOL_K, H=TOOL_H, W=TOOL_W, n_longitude=3, n_latitude=3, radius=None,
                   extractor="ORB", centre=None):
    """The tool's ``extract_textured_kp3ds`` on the GPU for one or more meshes of a
    :class:`~ffb6d_b200.render.RenderMeshTable`: each object rendered from its sphere of views (``render_rgbd``),
    ORB keypoints of every render (``orb_detect``) and their lift into the object frame (``orb_lift``); with
    ``extractor="SIFT"`` the tool's SIFT branch, ``sift_detect`` and ``sift_lift``.  With a
    :class:`~ffb6d_b200.render.TexturedMeshTable` the tool's pyrender branch: the same stages on textured renders,
    each object centred first.

    :param mesh: an index into ``table``, or a list of them (one object each)
    :param K, H, W: the camera and frame size (the tool's defaults); :param n_longitude, n_latitude: the views
    :param radius: each object's box radius (:func:`get_r`), or None to compute it from the table's vertices
    :param extractor: ``"ORB"`` or ``"SIFT"``, the tool's ``--extractor``
    :param centre: each object's centre ``[3]`` (a list of them for several objects), moved to the origin before the
      views are taken (:func:`sphere_poses`); None: no move for a :class:`RenderMeshTable` (the raster_triangle
      branch), the mean of the table's vertices for a :class:`TexturedMeshTable`.  The lift takes the float64
      centred poses and the render their float32 rounding.
    :return: ``(cloud [n_obj, V cap, 3] float32, n_points [n_obj] int32, short [n_obj, V] bool)`` on the device, V =
      n_longitude n_latitude: each object's pooled points, views in order.  A view with fewer than 500 drawn pixels
      contributes no points and is flagged in ``short`` (the tool stops with an error there).
    """
    import torch
    from . import _lib
    from .ops import orb_detect, orb_lift, sift_detect, sift_lift
    from .render import RenderMeshTable, TexturedMeshTable, render_rgbd
    if extractor not in ("ORB", "SIFT"):
        raise ValueError("textured_kp3ds: extractor must be 'ORB' or 'SIFT', got %r" % (extractor,))
    textured = isinstance(table, TexturedMeshTable)
    if not (textured or isinstance(table, RenderMeshTable)):
        raise ValueError("textured_kp3ds: table must be a RenderMeshTable or a TexturedMeshTable, got %s"
                         % type(table).__name__)
    objs = [int(m) for m in (mesh if isinstance(mesh, (list, tuple, np.ndarray)) else [mesh])]
    if not objs or min(objs) < 0 or max(objs) >= len(table):
        raise ValueError("textured_kp3ds: mesh indices must lie in [0, %d), got %s" % (len(table), objs))
    V = int(n_longitude) * int(n_latitude)
    B = V * len(objs)
    if V < 1 or B > min(_lib.RND_MAX_FRAMES, _lib.ORB_MAX_FRAMES) or len(objs) > _lib.ORB_MAX_OBJECTS:
        raise ValueError("textured_kp3ds: %d objects of %d views exceed the render limit of %d frames"
                         % (len(objs), V, min(_lib.RND_MAX_FRAMES, _lib.ORB_MAX_FRAMES)))
    H, W = int(H), int(W)
    lo, hi = (_lib.ORB_MIN_SIDE, _lib.ORB_MAX_SIDE) if extractor == "ORB" else (_lib.SIFT_MIN_SIDE, _lib.SIFT_MAX_SIDE)
    if not (lo <= H <= hi and lo <= W <= hi):
        raise ValueError("textured_kp3ds: H and W must lie in [%d, %d], got %dx%d" % (lo, hi, H, W))
    if radius is None or (centre is None and textured):
        off = np.concatenate([[0], np.cumsum(table.n_verts)])
        xyz = table.xyz.cpu().numpy()
        verts = [xyz[off[m]:off[m + 1]] for m in objs]
        if radius is None:
            radius = [get_r(get_3D_bbox(v)) for v in verts]
        if centre is None and textured:
            centre = [np.mean(v.astype(np.float64), axis=0) for v in verts]
    radius = list(radius) if isinstance(radius, (list, tuple, np.ndarray)) else [radius]
    if len(radius) != len(objs):
        raise ValueError("textured_kp3ds: %d radii for %d objects" % (len(radius), len(objs)))
    if centre is None:
        centre = [None] * len(objs)
    else:
        centre = np.asarray(centre, np.float64)
        if centre.shape not in ((3,), (len(objs), 3)):
            raise ValueError("textured_kp3ds: centre must be [3] or [%d,3], got %s" % (len(objs), centre.shape))
        centre = list(centre.reshape(-1, 3)) if centre.ndim == 2 else [centre]
        if len(centre) != len(objs):
            raise ValueError("textured_kp3ds: %d centres for %d objects" % (len(centre), len(objs)))
    RT = np.concatenate([sphere_poses(r, n_longitude, n_latitude, c) for r, c in zip(radius, centre)])
    dev = table.device
    mesh_idx = np.repeat(np.asarray(objs, np.int32), V)[:, None]
    depth, rgb, _ = render_rgbd(table, mesh_idx, RT[:, None, :3, :].astype(np.float32), np.ones((B, 1), np.uint8),
                                K, H, W)
    detect, lift = (orb_detect, orb_lift) if extractor == "ORB" else (sift_detect, sift_lift)
    count, pt = detect(rgb)[:2]
    short = torch.count_nonzero(depth > 1e-8, dim=(1, 2)) < MIN_RENDER_PIXELS
    count = torch.where(short, torch.zeros_like(count), count)
    cloud, n_points = lift(count, pt, depth, K, RT, V)
    return cloud, n_points, short.view(len(objs), V)


def gen_obj_info(points, n_keypoint=8, init_center=False, start=None, *, mesh=None, K=TOOL_K, H=TOOL_H, W=TOOL_W,
                 n_longitude=3, n_latitude=3, textured_start=None, extractor="ORB"):
    """The tables ``gen_one_mesh_info`` computes for one object's vertices ``points [N,3]``.

    :param n_keypoint: number of farthest-point keypoints (the tool's ``--n_keypoint``, 8 in the reference's configs)
    :param init_center, start: as :func:`ffb6d_b200.ops.farthest_point_sampling`; the tool calls it with neither,
      so its first keypoint is a random vertex
    :param mesh: None, or a :class:`~ffb6d_b200.render.RenderMeshTable` whose mesh 0 is this object (vertices
      ``points``): then the tool's textured keypoints are computed too (:func:`textured_kp3ds` with ``K``, ``H``,
      ``W``, ``n_longitude``, ``n_latitude``), and their farthest point sampling starts at ``textured_start`` (None:
      random, as the tool's).  A :class:`~ffb6d_b200.render.TexturedMeshTable` runs the tool's ``--use_pyrender``
      branch: the views are centred on ``np.mean(points, axis=0)`` (taken in float64), the tool's mean of the
      ``.obj``'s vertices -- pass those as ``points``, not the table's seam-split copy
    :param extractor: the textured keypoints' detector, ``"ORB"`` or ``"SIFT"`` (the tool's ``--extractor``)
    :return: dict ``corners [8,3]``, ``radius``, ``center [3]`` and ``fps [n_keypoint,3]`` (float32 vertices).
      ``fps`` is what ``pose_gt_objects(kps=...)`` and ``cal_frame_poses(mesh_kps=...)`` take as an object's keypoints.
      With ``mesh`` also ``textured_fps [n_keypoint,3]`` (float32; what ``use_orbfps`` reads) and ``short_views``
      (indices of views with fewer than 500 drawn pixels, which contributed no points).  With
      ``extractor="SIFT"`` also ``extractor`` (``"SIFT"``), which :func:`write_obj_info` names the file by.
    """
    from ._lib import FPS_MAX_POINTS
    from .ops import farthest_point_sampling
    points = np.asarray(points)
    if points.ndim != 2 or points.shape[1] != 3 or points.shape[0] < 1:
        raise ValueError("points must be [N,3] with N >= 1, got shape %s" % (points.shape,))
    if extractor not in ("ORB", "SIFT"):
        raise ValueError("gen_obj_info: extractor must be 'ORB' or 'SIFT', got %r" % (extractor,))
    c3ds = get_3D_bbox(points)
    info = dict(corners=c3ds, radius=get_r(c3ds), center=get_centers_3d(c3ds),
                fps=farthest_point_sampling(points, n_keypoint, init_center=init_center, start=start))
    if mesh is None:
        return info
    from .render import TexturedMeshTable
    centre = np.mean(points.astype(np.float64), axis=0) if isinstance(mesh, TexturedMeshTable) else None
    cloud, n_points, short = textured_kp3ds(mesh, 0, K, H, W, n_longitude, n_latitude, radius=info["radius"],
                                            extractor=extractor, centre=centre)
    n = int(n_points[0])
    if not 1 <= n <= FPS_MAX_POINTS:
        raise ValueError("gen_obj_info: %d textured keypoints; farthest point sampling takes 1 to %d" % (n, FPS_MAX_POINTS))
    info["textured_fps"] = farthest_point_sampling(cloud[0, :n].contiguous(), n_keypoint,
                                                   start=textured_start).cpu().numpy()
    info["short_views"] = np.nonzero(short[0].cpu().numpy())[0]
    if extractor != "ORB":
        info["extractor"] = extractor
    return info


def write_obj_info(info, sv_fd, obj_name):
    """Write the tables of :func:`gen_obj_info` as the tool does (gen_obj_info.py:97-117): ``<obj>_corners.txt``,
    ``<obj>_radius.txt``, ``<obj>_center.txt`` and ``<obj>_fps.txt`` under ``sv_fd``, one point per line.  They load
    back with ``np.loadtxt(path, dtype=np.float32)``, as ``Basic_Utils.get_kps`` / ``get_ctr`` read them.  When
    ``info`` has ``textured_fps``, ``<obj>_ORB_fps.txt`` too (gen_obj_info.py:122-126), which the datasets read as
    ``<obj>_8_kps.txt`` with ``use_orbfps`` -- ``<obj>_SIFT_fps.txt`` when ``info["extractor"]`` is ``"SIFT"``, the
    tool's name for its SIFT branch.
    :return: dict of the paths written."""
    os.makedirs(sv_fd, exist_ok=True)
    paths = {k: os.path.join(sv_fd, "%s_%s.txt" % (obj_name, k)) for k in ("corners", "radius", "center", "fps")}
    with open(paths["corners"], 'w') as of:
        for p3d in info["corners"]:
            print(p3d[0], p3d[1], p3d[2], file=of)
    with open(paths["radius"], 'w') as of:
        print(info["radius"], file=of)
    with open(paths["center"], 'w') as of:
        ctr = info["center"]
        print(ctr[0], ctr[1], ctr[2], file=of)
    with open(paths["fps"], 'w') as of:
        for p3d in info["fps"]:
            print(p3d[0], p3d[1], p3d[2], file=of)
    if "textured_fps" in info:
        key = "%s_fps" % info.get("extractor", "ORB")
        paths[key] = os.path.join(sv_fd, "%s_%s.txt" % (obj_name, key))
        with open(paths[key], 'w') as of:
            for p3d in info["textured_fps"]:
                print(p3d[0], p3d[1], p3d[2], file=of)
    return paths
