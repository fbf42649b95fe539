"""The per-object half of the datasets' ``get_pose_gt_info``, on the host.

``get_pose_gt_info`` (datasets/ycb/ycb_dataset.py:348-386, datasets/linemod/linemod_dataset.py:398-436) returns two
kinds of arrays.  The per-object ones -- ``RTs``, ``kp_3ds``, ``ctr_3ds``, ``cls_ids`` -- depend only on the frame's
poses and the meshes' keypoints, not on the sampled points, so a DataLoader worker keeps computing them.  The
per-point ones -- ``kp_targ_ofst``, ``ctr_targ_ofst`` -- need ``choose``, which exists only on the device once the
input path runs there; :func:`ffb6d_b200.ops.point_item` builds them from the float64 tables returned here.

Plain numpy: importable without the CUDA library, as a worker process wants.
"""
import numpy as np


def pose_gt_objects(poses, cls_ids, kps, ctrs, n_objects, n_kps, dataset="ycb"):
    """The per-object arrays of ``get_pose_gt_info`` for one frame, with the reference's expressions.

    :param poses: YCB: ``meta['poses']`` ``[3,4,n]``; LineMOD: the frame's ``RT`` ``[3,4]``
    :param cls_ids: YCB: the class ids (``meta['cls_indexes'].flatten().astype(np.uint32)``); LineMOD: ``[1]``
    :param kps: per object, the mesh keypoints ``[n_kps,3]`` (what ``bs_utils.get_kps`` returns for its class)
    :param ctrs: per object, the mesh centre ``[3]`` (``bs_utils.get_ctr``)
    :param n_objects, n_kps: ``config.n_objects``, ``config.n_keypoints``
    :param dataset: ``"ycb"`` or ``"linemod"``
    :return: dict of the item keys ``RTs [n_objects,3,4]``, ``kp_3ds [n_objects,n_kps,3]``, ``ctr_3ds
      [n_objects,3]`` (float32) and ``cls_ids [n_objects,1]`` (int32, zero padding, as the reference), plus the
      tables :func:`ffb6d_b200.ops.point_item` takes: ``obj_cls [n_objects]`` int32 (-1 on padding slots, so that
      the background label 0 never matches one), ``obj_kps [n_objects,n_kps,3]`` and ``obj_ctr [n_objects,3]``
      float64.
    :raises ValueError: more objects than ``n_objects`` (the reference raises ``IndexError`` there), or keypoint
      arrays that are not ``[n_kps,3]``
    """
    if dataset not in ("ycb", "linemod"):
        raise ValueError("dataset must be 'ycb' or 'linemod', got %r" % (dataset,))
    cls_ids = list(cls_ids)
    if dataset == "linemod" and cls_ids != [1]:
        raise ValueError("LineMOD frames hold one object of class 1, got cls_ids=%r" % (cls_ids,))
    if len(cls_ids) > n_objects:
        raise ValueError("%d objects in the frame, more than n_objects=%d" % (len(cls_ids), n_objects))
    if len(kps) != len(cls_ids) or len(ctrs) != len(cls_ids):
        raise ValueError("need one keypoint set and one centre per object")
    for kp in kps:
        if np.shape(kp) != (n_kps, 3):
            raise ValueError("mesh keypoints must be [n_kps=%d, 3], got %s" % (n_kps, np.shape(kp)))
    RTs = np.zeros((n_objects, 3, 4))
    kp3ds = np.zeros((n_objects, n_kps, 3))
    ctr3ds = np.zeros((n_objects, 3))
    cls_ids_out = np.zeros((n_objects, 1))
    obj_cls = np.full((n_objects,), -1, np.int32)
    for i, cls_id in enumerate(cls_ids):
        # the reference's expressions shape for shape: numpy's dot may pick another BLAS kernel for another shape
        if dataset == "ycb":                                          # ycb_dataset.py:356-378
            r = poses[:, :, i][:, 0:3]
            t = np.array(poses[:, :, i][:, 3:4].flatten()[:, None])
            RTs[i] = np.concatenate((r, t), axis=1)
            ctr = np.asarray(ctrs[i]).copy()[:, None]
            ctr = np.dot(ctr.T, r.T) + t[:, 0]
            kp = np.dot(np.asarray(kps[i]).copy(), r.T) + t[:, 0]
        else:                                                         # linemod_dataset.py:406-427
            RTs[i] = poses
            r = poses[:, :3]
            t = poses[:, 3]
            ctr = np.dot(np.asarray(ctrs[i])[:, None].T, r.T) + t
            kp = np.dot(np.asarray(kps[i]), r.T) + t
        ctr3ds[i, :] = ctr[0]
        cls_ids_out[i, :] = np.array([cls_id])
        kp3ds[i] = kp
        obj_cls[i] = int(cls_id)
    return dict(RTs=RTs.astype(np.float32), kp_3ds=kp3ds.astype(np.float32), ctr_3ds=ctr3ds.astype(np.float32),
                cls_ids=cls_ids_out.astype(np.int32), obj_cls=obj_cls, obj_kps=kp3ds, obj_ctr=ctr3ds)
