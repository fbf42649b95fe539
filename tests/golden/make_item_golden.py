#!/usr/bin/env python
"""Generate tests/golden/item_cases.npz by running THE REFERENCE'S OWN per-point item code in this container.

Source of truth: ``dpt_2_pcld`` and ``get_pose_gt_info`` of both datasets (datasets/ycb/ycb_dataset.py:165-176,
348-386; datasets/linemod/linemod_dataset.py:188-199, 398-436), executed from the reference's source text (the dataset
modules import normalSpeed and read dataset files, so the methods are taken out of the files with ``ast``).  Their
``config``, ``bs_utils`` and ``self`` are stubs that hand out the synthetic meshes' keypoints and centres.  The lines
of ``get_item`` around them (ycb_dataset.py:215-242, linemod_dataset.py:259-289: ``dpt_m``, ``msk_dp``, the draw of
``choose`` with numpy's global random stream and the five indexing lines) are restated here, because ``get_item``
reads files and calls normalSpeed.  The depth completion is left out: its golden data is fill_cases.npz, and a
completed depth map is an input like any other here.  The inputs are the frames of
``ffb6d_b200.synthetic.item_test_frames``; the tests regenerate them from their seeds.

Stored per frame: sha256s of the inputs; the reference's ``choose``; its per-object arrays (the float64 ``kp3ds`` /
``ctr3ds`` of ``get_pose_gt_info`` and the item's float32 / int32 casts); and its per-point arrays after the item's
casts -- in full for the small frames, as a sha256 each for the 480x640 frames, to keep the file small.

Run:  python tests/golden/make_item_golden.py      (needs /root/reference; rewrites item_cases.npz)
"""
import hashlib
import os
import sys
import types

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
from oracle import ref_loader as R                                  # noqa: E402
from ffb6d_b200.synthetic import item_test_frames                   # noqa: E402

OUT = os.path.join(os.path.dirname(os.path.abspath(__file__)), "item_cases.npz")
POINT_KEYS = ("cld_rgb_nrm", "labels", "kp_targ_ofst", "ctr_targ_ofst")
CHOOSE_SEED = 1234


def sha(a):
    return hashlib.sha256(np.ascontiguousarray(a).tobytes()).hexdigest()


def reference_methods(dataset):
    """(dpt_2_pcld, get_pose_gt_info) of the dataset's ``Dataset`` class, as plain functions of (self, ...)."""
    path = os.path.join(R.REF_ROOT, "ffb6d", "datasets", dataset, "%s_dataset.py" % ("ycb" if dataset == "ycb" else
                                                                                      "linemod"))
    fns = R._extract(path, "Dataset", ["dpt_2_pcld", "get_pose_gt_info"])
    for f in fns.values():
        f.__globals__["np"] = np
    return fns["dpt_2_pcld"], fns["get_pose_gt_info"]


def stubs(frame, dataset, n_points, n_objects, h, w):
    """``self`` (and, for YCB, the module globals ``config`` / ``bs_utils``) of the reference's methods."""
    n_kps = frame["kps"][0].shape[0]
    names = {int(c): "cls%02d" % int(c) for c in frame["cls_ids"]}
    mesh = {names[int(c)]: (k, t) for c, k, t in zip(frame["cls_ids"], frame["kps"], frame["ctrs"])}
    kp_type_want = "farthest" if n_kps == 8 else "farthest{}".format(n_kps)

    class BsUtils:
        @staticmethod
        def get_kps(cls, kp_type=None, ds_type=None):
            assert kp_type == kp_type_want and ds_type == dataset
            return mesh[cls][0].copy()

        @staticmethod
        def get_ctr(cls, ds_type="ycb", ctr_pth=None):
            assert ds_type == dataset
            return mesh[cls][1].copy()

    config = types.SimpleNamespace(n_objects=n_objects, n_keypoints=n_kps, n_sample_points=n_points,
                                   mini_batch_size=1)
    self = types.SimpleNamespace(
        xmap=np.array([[j for i in range(w)] for j in range(h)]),       # ycb_dataset.py:31-32
        ymap=np.array([[i for i in range(w)] for j in range(h)]),
        cls_lst=["cls%02d" % c for c in range(1, 22)], config=config, bs_utils=BsUtils(), cls_type="cls01",
        all_lst=[])
    return self, config, BsUtils()


def reference_item(frame, dataset, n_points, n_objects):
    h, w = frame["labels"].shape
    dpt_2_pcld, get_pose_gt_info = reference_methods(dataset)
    self, config, bs_utils = stubs(frame, dataset, n_points, n_objects, h, w)
    get_pose_gt_info.__globals__.update(config=config, bs_utils=bs_utils)
    K, rgb, labels, nrm_map = frame["K"], frame["rgb"], frame["labels"], frame["nrm"]
    if dataset == "ycb":                                                 # ycb_dataset.py:195-216
        cam_scale = np.float32(frame["cam_scale"])
        dpt_um = frame["raw"]
        msk_dp = dpt_um > 1e-6
        dpt_m = dpt_um.astype(np.float32) / cam_scale
        dpt_xyz = dpt_2_pcld(self, dpt_m, 1.0, K)
    else:                                                                # linemod_dataset.py:237-264
        cam_scale = 1000.0
        dpt_mm = frame["raw"].copy().astype(np.uint16)
        dpt_m = dpt_mm.astype(np.float32) / cam_scale
        dpt_xyz = dpt_2_pcld(self, dpt_m, 1.0, K)
        dpt_xyz[np.isnan(dpt_xyz)] = 0.0
        dpt_xyz[np.isinf(dpt_xyz)] = 0.0
        msk_dp = dpt_mm > 1e-6
    # the draw of choose (ycb_dataset.py:218-235), on numpy's global stream
    choose = msk_dp.flatten().nonzero()[0].astype(np.uint32)
    assert len(choose) >= 400
    choose_2 = np.array([i for i in range(len(choose))])
    if len(choose_2) > n_points:
        c_mask = np.zeros(len(choose_2), dtype=int)
        c_mask[:n_points] = 1
        np.random.shuffle(c_mask)
        choose_2 = choose_2[c_mask.nonzero()]
    else:
        choose_2 = np.pad(choose_2, (0, n_points - len(choose_2)), 'wrap')
    choose = np.array(choose)[choose_2]
    sf_idx = np.arange(choose.shape[0])
    np.random.shuffle(sf_idx)
    choose = choose[sf_idx]
    # the five indexing lines (ycb_dataset.py:237-242)
    cld = dpt_xyz.reshape(-1, 3)[choose, :]
    rgb_pt = rgb.reshape(-1, 3)[choose, :].astype(np.float32)
    nrm_pt = nrm_map[:, :, :3].reshape(-1, 3)[choose, :]
    labels_pt = labels.flatten()[choose]
    cld_rgb_nrm = np.concatenate((cld, rgb_pt, nrm_pt), axis=1).transpose(1, 0)
    if dataset == "ycb":
        out = get_pose_gt_info(self, cld, labels_pt, frame["cls_ids"], {"poses": frame["poses"]})
    else:
        out = get_pose_gt_info(self, cld, labels_pt, frame["poses"])
    RTs, kp3ds, ctr3ds, cls_ids, kp_targ_ofst, ctr_targ_ofst = out
    return dict(choose=choose.astype(np.int32), cld_rgb_nrm=cld_rgb_nrm.astype(np.float32),
                labels=labels_pt.astype(np.int32), RTs=RTs.astype(np.float32),
                kp_targ_ofst=kp_targ_ofst.astype(np.float32), ctr_targ_ofst=ctr_targ_ofst.astype(np.float32),
                cls_ids=cls_ids.astype(np.int32), ctr_3ds=ctr3ds.astype(np.float32), kp_3ds=kp3ds.astype(np.float32),
                kp3ds64=kp3ds, ctr3ds64=ctr3ds, dpt_map_m=dpt_m.astype(np.float32))


def input_digests(frame):
    return {"sha256_in_" + k: np.array(sha(frame[k])) for k in ("raw", "rgb", "nrm", "labels", "poses")}


def item_cases():
    out = {}
    for j, (name, (frame, dataset, n_points, n_objects)) in enumerate(sorted(item_test_frames().items())):
        np.random.seed(CHOOSE_SEED + j)
        ref = reference_item(frame, dataset, n_points, n_objects)
        full = frame["labels"].size >= 480 * 640
        for k, v in input_digests(frame).items():
            out[name + "/" + k] = v
        for k, v in ref.items():
            if k == "dpt_map_m":
                out[name + "/sha256_dpt_map_m"] = np.array(sha(v))
            elif full and k in POINT_KEYS:
                out[name + "/sha256_" + k] = np.array(sha(v))
            else:
                out[name + "/" + k] = v
    return out


def main():
    if not R.reference_sources_present():
        raise SystemExit("needs /root/reference")
    np.savez_compressed(OUT, **item_cases())
    print("wrote", OUT, os.path.getsize(OUT), "bytes")


if __name__ == "__main__":
    main()
