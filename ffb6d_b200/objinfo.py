"""The object tables of the reference's mesh tool, utils/dataset_tools/gen_obj_info.py.

For each object, ``gen_one_mesh_info`` (gen_obj_info.py:92-117) writes the 3D bounding box corners, the radius, the
centre and the farthest-point keypoints of the mesh's vertices; the datasets and ``cal_frame_poses`` read them back
(``Basic_Utils.get_kps`` / ``get_ctr``, utils/basic_utils.py:572-640).  The box arithmetic is restated here with the
expressions of ``MeshUtils`` (utils/dataset_tools/utils.py:88-115); the keypoints come from
:func:`ffb6d_b200.ops.farthest_point_sampling` on the GPU.

Mesh files are not read here: the caller passes the vertex array ``[N,3]`` (what ``MeshUtils.get_p3ds_from_mesh``
returns, already divided by ``scale2m``).  The textured ORB keypoints of the tool (rendering and 2D feature
extraction) are out of scope.  Plain numpy; only :func:`gen_obj_info` loads the CUDA library.
"""
import os

import numpy as np


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


def gen_obj_info(points, n_keypoint=8, init_center=False, start=None):
    """The tables ``gen_one_mesh_info`` computes for one object's vertices ``points [N,3]``.

    :param n_keypoint: number of farthest-point keypoints (the tool's ``--n_keypoint``, 8 in the reference's configs)
    :param init_center, start: as :func:`ffb6d_b200.ops.farthest_point_sampling`; the tool calls it with neither,
      so its first keypoint is a random vertex
    :return: dict ``corners [8,3]``, ``radius``, ``center [3]`` and ``fps [n_keypoint,3]`` (float32 vertices).
      ``fps`` is what ``pose_gt_objects(kps=...)`` and ``cal_frame_poses(mesh_kps=...)`` take as an object's keypoints.
    """
    from .ops import farthest_point_sampling
    points = np.asarray(points)
    if points.ndim != 2 or points.shape[1] != 3 or points.shape[0] < 1:
        raise ValueError("points must be [N,3] with N >= 1, got shape %s" % (points.shape,))
    c3ds = get_3D_bbox(points)
    return dict(corners=c3ds, radius=get_r(c3ds), center=get_centers_3d(c3ds),
                fps=farthest_point_sampling(points, n_keypoint, init_center=init_center, start=start))


def write_obj_info(info, sv_fd, obj_name):
    """Write the tables of :func:`gen_obj_info` as the tool does (gen_obj_info.py:97-117): ``<obj>_corners.txt``,
    ``<obj>_radius.txt``, ``<obj>_center.txt`` and ``<obj>_fps.txt`` under ``sv_fd``, one point per line.  They load
    back with ``np.loadtxt(path, dtype=np.float32)``, as ``Basic_Utils.get_kps`` / ``get_ctr`` read them.
    :return: dict of the four paths."""
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
    return paths
