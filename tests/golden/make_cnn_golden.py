#!/usr/bin/env python
"""Generate tests/golden/cnn_cases.npz and tests/golden/ffb6d_state_keys.json from the reference's own code.

Source of truth: the reference's models/ffb6d.py, models/cnn/pspnet.py and models/cnn/extractors.py, imported from
its tree on the CPU.  Its imports are satisfied without running anything of the reference's environment: ``common``
(which writes into its tree on import) is a stub holding only the ``config`` the extractors read, ``helper_tool`` /
``sklearn`` / ``tqdm`` (needed by the RandLA and training utilities, never called here) are stubs where they are not
installed, ``torch.utils.model_zoo.load_url`` raises, and the ResNet is built with ``pretrained=False``.  Nothing of
the reference is copied: only a seeded input, the reference's outputs and its state-dict keys are stored.

* ``ffb6d_state_keys.json``: every key and shape of ``FFB6D(n_classes=22, n_pts=12288, rndla_cfg, n_kps=8)``.
* ``cnn_cases.npz``: the reference's ``cnn_pre_stages``, every ``cnn_ds_stages[j]`` and every ``cnn_up_stages[j]``
  in eval mode, float64, with the seeded weights of ``oracle/cnn_oracle.py``, chained without fusion on one
  1x3x56x72 image (PSP at 7x9: overlapping bins at the sizes 2, 3 and 6 along the rows, 2 and 6 along the
  columns).  ``rgb`` is the input (float32, used as is); for stage k (0 pre, 1-4 ds, 5-8 up) ``shape{k}`` is the
  output's shape, ``idx{k}`` int32 flat positions (up to 3072 per stage, drawn without replacement from a seeded
  RandomState, sorted) and ``out{k}`` the float64 outputs there.  A sample keeps the fixture small (about 0.4 MB
  instead of 19 MB for every value); a wrong bin bound, tap, stride or shared module changes most values of a
  stage, so it shows in any few thousand of them.

Run:  python tests/golden/make_cnn_golden.py      (needs the reference's sources; rewrites both files)
"""
import json
import os
import sys
import types

import numpy as np
import torch
import torch.nn as nn

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
from oracle import cnn_oracle, ref_loader as R                      # noqa: E402

HERE = os.path.dirname(os.path.abspath(__file__))
H, W = 56, 72
SAMPLES = 3072


def reference_ffb6d():
    sys.dont_write_bytecode = True
    import torch.utils.model_zoo as mz

    def no_download(*a, **k):
        raise RuntimeError("no downloads")
    mz.load_url = no_download
    sys.path.insert(0, os.path.join(R.REF_ROOT, "ffb6d"))
    stubs = {"common": {"config": types.SimpleNamespace(resnet_ptr_mdl_p=None)},
             "helper_tool": {"DataProcessing": object}, "sklearn": {}, "sklearn.metrics": {"confusion_matrix": None},
             "tqdm": {}}
    for name, attrs in stubs.items():
        if name != "common":
            try:
                __import__(name)
                continue
            except ImportError:
                pass
        m = types.ModuleType(name)
        m.__dict__.update(attrs)
        sys.modules[name] = m
    import models.ffb6d as ref
    from models.cnn.pspnet import PSPNet
    ref.psp_models["resnet34"] = lambda: PSPNet(sizes=(1, 2, 3, 6), psp_size=512, deep_features_size=256,
                                                backend="resnet34", pretrained=False)
    cfg = types.SimpleNamespace(k_n=16, num_layers=4, d_out=[32, 64, 128, 256], in_c=9, num_classes=22)
    return ref.FFB6D(n_classes=22, n_pts=12288, rndla_cfg=cfg, n_kps=8)


def main():
    torch.manual_seed(0)
    net = reference_ffb6d()
    keys = [[k, list(v.shape)] for k, v in net.state_dict().items()]
    with open(os.path.join(HERE, "ffb6d_state_keys.json"), "w") as fh:
        json.dump(keys, fh, indent=0)
        fh.write("\n")

    branch = nn.Module()
    branch.cnn_pre_stages, branch.cnn_ds_stages, branch.cnn_up_stages = \
        net.cnn_pre_stages, net.cnn_ds_stages, net.cnn_up_stages
    branch = cnn_oracle.load_seeded(branch.double(), seed=0).eval()
    rs = np.random.RandomState(1)
    rgb = rs.uniform(-2.0, 2.0, (1, 3, H, W)).astype(np.float32)
    data = {"rgb": rgb}
    x = torch.from_numpy(rgb).double()
    stages = [branch.cnn_pre_stages] + list(branch.cnn_ds_stages) + list(branch.cnn_up_stages)
    import warnings
    with torch.no_grad(), warnings.catch_warnings():
        warnings.simplefilter("ignore")                # F.upsample and the implicit LogSoftmax dim
        for k, st in enumerate(stages):
            x = st(x)
            flat = x.numpy().reshape(-1)
            idx = np.sort(np.random.RandomState(100 + k).choice(flat.size, min(flat.size, SAMPLES), replace=False))
            data["shape%d" % k] = np.asarray(x.shape, np.int64)
            data["idx%d" % k] = idx.astype(np.int32)
            data["out%d" % k] = flat[idx].astype(np.float64)
            print("stage %d: %s, %d of %d values" % (k, tuple(x.shape), idx.size, flat.size))
    np.savez(os.path.join(HERE, "cnn_cases.npz"), **data)


if __name__ == "__main__":
    main()
