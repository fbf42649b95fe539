"""Seeded weights for FFB6D's image branch (``cnn_*`` keys of the reference's FFB6D state dict), so that the golden
fixture of the image branch stores outputs only: tests/golden/make_cnn_golden.py loads these weights into the
reference's own modules, tests/test_cnn_golden.py into :mod:`ffb6d_b200.cnn`.

Every tensor is drawn from its own ``RandomState(seed ^ crc32(key))``, so a value depends on its key alone.  Scales
keep activations O(1) through the 40 layers: convs ``N(0, sqrt(2 / fan_in))`` (the trunk's convs are followed by
BatchNorm anyway), BatchNorm weight U(0.5, 1.5), bias and running mean N(0, 0.1), running variance U(0.5, 1.5), conv
biases N(0, 0.1), PReLU slopes U(0.1, 0.4).  ``final`` is one module at two stages: its second key
(``cnn_up_stages.3.1.*``) gets the values of its first (``cnn_up_stages.2.0.*``)."""
import zlib

import numpy as np

FINAL_ALIAS = ("cnn_up_stages.3.1.", "cnn_up_stages.2.0.")


def _draw(key, shape, seed):
    rs = np.random.RandomState((seed ^ zlib.crc32(key.encode())) & 0x7FFFFFFF)
    leaf = key.rsplit(".", 1)[1]
    if leaf == "num_batches_tracked":
        return np.zeros(shape, np.int64)
    if leaf == "running_var":
        return rs.uniform(0.5, 1.5, shape)
    if leaf == "running_mean":
        return rs.normal(0.0, 0.1, shape)
    if len(shape) == 4:                                    # conv weight
        fan_in = int(np.prod(shape[1:]))
        return rs.normal(0.0, np.sqrt(2.0 / fan_in), shape)
    if len(shape) == 1 and shape[0] == 1:                  # PReLU slope
        return rs.uniform(0.1, 0.4, shape)
    if leaf == "weight":                                   # BatchNorm weight
        return rs.uniform(0.5, 1.5, shape)
    return rs.normal(0.0, 0.1, shape)                      # BatchNorm / conv bias


def seeded_state(shapes, seed=0):
    """``{key: float64 / int64 ndarray}`` for ``shapes = {key: shape}`` (the ``cnn_*`` part of a state dict)."""
    out = {}
    for key, shape in shapes.items():
        src = key
        if key.startswith(FINAL_ALIAS[0]):
            src = FINAL_ALIAS[1] + key[len(FINAL_ALIAS[0]):]
        out[key] = _draw(src, tuple(shapes[src]) if src in shapes else tuple(shape), seed)
    return out


def load_seeded(module, seed=0, dtype=None):
    """Fill ``module`` (whose state-dict keys are ``cnn_*`` keys) with :func:`seeded_state`; returns the module."""
    import torch
    sd = module.state_dict()
    vals = seeded_state({k: tuple(v.shape) for k, v in sd.items()}, seed)
    new = {k: torch.from_numpy(vals[k]).to(dtype=(dtype or v.dtype) if v.dtype.is_floating_point else v.dtype)
           for k, v in sd.items()}
    module.load_state_dict(new, strict=True)
    return module
