"""numpy restatement of the 3xTF32 operand split of ``fusion_mlp.cu`` (``to_tf32``, ``split1``; DESIGN.md §4.4).

Every fp32 operand of the tensor-core GEMMs is split into ``hi = tf32(x)`` and ``lo = tf32(x - hi)``, on bit patterns:

1. ``to_tf32(u)``: ``(u + 0x1000) & 0xFFFFE000`` (mod 2^32: round half away from zero at mantissa bit 13).
   ``to_tf32_finite(u)``: the same with ``u + 0x1000`` clamped to ``0x7F7FFFFF`` as a signed int32 and to
   ``0xFF7FFFFF`` as a uint32.  The clamps change nothing for a finite x below ``(2 - 2^-11) * 2^127`` in magnitude;
   in the top band ``0x7F7FF000`` .. ``0x7F7FFFFF`` (either sign), where rounding would carry into the exponent and
   give an infinity, they make the rounding a truncation, so ``hi`` stays finite.
2. ``split1(x)``: ``h = to_tf32_finite(x)``, ``d = x - h`` (fp32, round to nearest, subnormals kept),
   ``lo = to_tf32(d)`` (``|d| <= 2^-10 |x|`` never reaches the band), ``hi = fma(d, 0, h)``: ``h`` for a finite x
   (an exact -0 becomes +0), NaN for a NaN or infinite x.  Float arithmetic on the GPU returns the NaN ``0x7FFFFFFF``
   whatever NaN goes in; so does this restatement.

For every finite x, ``|x - (hi + lo)| <= 2^-22 |x| + 2^-137``: the relative term is the rounding of ``d`` to TF32's
11 significant bits, the absolute one that of a subnormal ``d`` to a multiple of 2^-136.
"""
import numpy as np

GPU_NAN = 0x7FFFFFFF
TOP_BAND = (0x7F7FF000, 0x7F7FFFFF)     # |x| bit patterns whose round-to-nearest TF32 is an infinity
SPLIT_REL = 2.0 ** -22
SPLIT_ABS = 2.0 ** -137


def to_tf32_bits(u):
    """``to_tf32`` on uint32 bit patterns (array in, uint32 array out)."""
    return (np.asarray(u, np.uint32) + np.uint32(0x1000)) & np.uint32(0xFFFFE000)


def to_tf32_finite_bits(u):
    """``to_tf32_finite`` on uint32 bit patterns (array in, uint32 array out)."""
    r = np.asarray(u, np.uint32) + np.uint32(0x1000)
    r = np.where(r.view(np.int32) > 0x7F7FFFFF, np.uint32(0x7F7FFFFF), r)      # min as int32
    r = np.minimum(r, np.uint32(0xFF7FFFFF))                                   # min as uint32
    return (r & np.uint32(0xFFFFE000)).astype(np.uint32)


def _gpu_nan(v):
    v = np.array(v, np.float32)
    v.view(np.uint32)[np.isnan(v)] = GPU_NAN
    return v


def split(x, rounding=to_tf32_finite_bits):
    """``split1`` of float32 ``x`` (any shape): ``(hi, lo)`` float32, bit for bit what the kernels stage.
    ``rounding``: the bit-pattern rounding of ``hi`` (tests pass variants of :func:`to_tf32_finite_bits`)."""
    x = np.asarray(x, np.float32)
    with np.errstate(invalid="ignore", over="ignore"):
        h = np.asarray(rounding(x.view(np.uint32)), np.uint32).view(np.float32)
        d = _gpu_nan(x - h)
        lo = to_tf32_bits(d.view(np.uint32)).view(np.float32)
        hi = _gpu_nan(d * np.float32(0) + h)    # fma(d, 0, h): d * 0 is exact, so one rounding either way
    return hi, lo
