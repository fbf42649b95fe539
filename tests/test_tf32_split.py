"""CPU: the 3xTF32 operand split of the tensor-core GEMMs (``to_tf32`` / ``split1`` of ``fusion_mlp.cu``, restated in
``oracle/tf32_oracle.py``) over the whole float32 range: every exponent, both signs, the mantissas at the rounding
edges, the top band where round-to-nearest would carry into the exponent, subnormals, infinities and NaNs.
``tests/test_gpu_gemm_range.py`` ties the restatement to the device code bit for bit."""
import numpy as np
import pytest

from oracle import tf32_oracle as T

# mantissas at the rounding edges: the 13 bits below TF32's 10-bit mantissa just under, at and above the half, all
# ones (with and without the top TF32 bits set, where the rounding carries through the whole mantissa), zero
EDGE_MANTISSAS = [0x000000, 0x000001, 0x000FFF, 0x001000, 0x001001, 0x001FFF, 0x002000, 0x003000, 0x7FEFFF, 0x7FF000,
                  0x7FE000, 0x7FFFFF, 0x400000, 0x555555]


def _patterns(mantissas):
    sign = np.array([0, 1], np.uint32)[:, None, None] << np.uint32(31)
    expo = np.arange(256, dtype=np.uint32)[None, :, None] << np.uint32(23)
    mant = np.asarray(mantissas, np.uint32)[None, None, :]
    return (sign | expo | mant).ravel()


def _dense_patterns():
    """Every sign and exponent with every value of the 13 rounded-off bits, under three settings of the 10 kept
    mantissa bits (none, alternating, all set): every carry the rounding can make."""
    low = np.arange(1 << 13, dtype=np.uint32)
    mant = (np.array([0x000, 0x2AA, 0x3FF], np.uint32)[:, None] << np.uint32(13) | low[None, :]).ravel()
    return _patterns(mant)


EDGES = _patterns(EDGE_MANTISSAS)


def _f32(bits):
    return np.asarray(bits, np.uint32).view(np.float32)


def _split_error(x, hi, lo):
    """|x - (hi + lo)| in float64 (exact: hi + lo has at most 35 significant bits) and the bound 2^-22 |x| + 2^-137."""
    x64 = x.astype(np.float64)
    err = np.abs(x64 - (hi.astype(np.float64) + lo.astype(np.float64)))
    return err, T.SPLIT_REL * np.abs(x64) + T.SPLIT_ABS


@pytest.mark.parametrize("which", ["edges", "dense"])
def test_split_of_every_finite_float_is_finite_and_exact_to_2e22(which):
    """hi and lo are finite for every finite x, top band included, and ``|x - (hi + lo)| <= 2^-22 |x| + 2^-137``;
    where lo is normal (|x| >= 2^-103) the relative term alone bounds it."""
    u = EDGES if which == "edges" else _dense_patterns()
    x = _f32(u)
    fin = np.isfinite(x)
    x = x[fin]
    hi, lo = T.split(x)
    bad = ~(np.isfinite(hi) & np.isfinite(lo))
    assert not bad.any(), "non-finite split of finite x: %s" % [hex(int(v)) for v in x[bad][:8].view(np.uint32)]
    err, bound = _split_error(x, hi, lo)
    over = err > bound
    assert not over.any(), "split error over the bound at %s" % [hex(int(v)) for v in x[over][:8].view(np.uint32)]
    big = np.abs(x) >= 2.0 ** -103
    assert (err[big] <= T.SPLIT_REL * np.abs(x[big].astype(np.float64))).all()
    # hi is a TF32 value: its 13 low mantissa bits are clear, and so are lo's
    assert not (hi.view(np.uint32) & 0x1FFF).any() and not (lo.view(np.uint32) & 0x1FFF).any()


def test_top_band_truncates_and_everything_below_rounds():
    """Below the top band hi's rounding is the plain ``(u + 0x1000) & 0xFFFFE000`` (round half away from zero), bit
    for bit; in the band (0x7F7FF000 .. 0x7F7FFFFF, either sign) it is the truncation ``u & 0xFFFFE000``, the largest
    TF32 value below x, so hi = +-0x7F7FE000."""
    u = _dense_patterns()
    mag = u & np.uint32(0x7FFFFFFF)
    got = T.to_tf32_finite_bits(u)
    assert np.array_equal(T.to_tf32_bits(u), (u + np.uint32(0x1000)) & np.uint32(0xFFFFE000))
    below = mag < T.TOP_BAND[0]
    band = (mag >= T.TOP_BAND[0]) & (mag <= T.TOP_BAND[1])
    assert band.sum() == 2 * (T.TOP_BAND[1] - T.TOP_BAND[0] + 1)   # the whole band, both signs
    assert np.array_equal(got[below], (u[below] + np.uint32(0x1000)) & np.uint32(0xFFFFE000))
    assert np.array_equal(got[band], u[band] & np.uint32(0xFFFFE000))
    hi, _ = T.split(_f32(u[band]))
    assert np.array_equal(hi.view(np.uint32) & np.uint32(0x7FFFFFFF), np.full(band.sum(), 0x7F7FE000, np.uint32))


def test_round_to_nearest_at_the_edges():
    """Ties round away from zero, everything else to the nearest TF32 value: 1 + k 2^-23 for the 13 bits below."""
    one = 0x3F800000
    cases = {0x0FFF: one, 0x1000: one + 0x2000, 0x1001: one + 0x2000, 0x1FFF: one + 0x2000, 0x2FFF: one + 0x2000,
             0x3000: one + 0x4000}
    for low, want in cases.items():
        for s in (0, 0x80000000):
            for f in (T.to_tf32_bits, T.to_tf32_finite_bits):
                assert int(f(np.uint32(s | one | low))) == s | want, hex(s | one | low)
    # the carry through a full mantissa moves to the next binade, and a subnormal rounds onto the 2^-136 grid
    assert int(T.to_tf32_bits(np.uint32(0x3FFFF000))) == 0x40000000
    assert int(T.to_tf32_bits(np.uint32(0x00000FFF))) == 0 and int(T.to_tf32_bits(np.uint32(0x00001000))) == 0x2000


NONFINITE = {"nan": 0x7FC00000, "nan_7fffffff": 0x7FFFFFFF, "nan_ffffffff": 0xFFFFFFFF, "snan": 0x7F800001,
             "nan_7ffff000": 0x7FFFF000, "-nan": 0xFFC00000, "inf": 0x7F800000, "-inf": 0xFF800000}


@pytest.mark.parametrize("bad", list(NONFINITE))
def test_nonfinite_input_gives_nan_hi(bad):
    """A NaN or an infinity gives hi = NaN, so every product with it, and every output it enters, is NaN (what
    ``test_fusion_mlp_nonfinite_input`` requires of the layers).  This holds for every NaN payload, including those
    the integer rounding wraps to +-0."""
    hi, lo = T.split(_f32([NONFINITE[bad]]))
    assert np.isnan(hi).all()


def test_every_nonfinite_pattern_of_the_sweep_gives_nan_hi():
    x = _f32(_dense_patterns())
    x = x[~np.isfinite(x)]
    assert x.size == 2 * 3 * (1 << 13)
    hi, _ = T.split(x)
    assert np.isnan(hi).all()


def test_signed_zero():
    """+0 splits into (+0, +0); -0 into (+0, +0) too (``fma(d, 0, h)`` with d = +0), which no product can tell apart."""
    for bits in (0, 0x80000000):
        hi, lo = T.split(_f32([bits]))
        assert hi.view(np.uint32)[0] == 0 and lo.view(np.uint32)[0] == 0


def _unguarded(u):
    """hi's rounding without the clamps of the top band."""
    return (np.asarray(u, np.uint32) + np.uint32(0x1000)) & np.uint32(0xFFFFE000)


def test_unguarded_rounding_fails_on_the_top_band():
    """The checks above see the defect the clamps remove: plain round-to-nearest carries every finite x of the top
    band into +-inf, and the split then gives hi = NaN (inf - inf, through fma), while 0x7F7FEFFF just below splits
    cleanly either way."""
    for s in (0, 0x80000000):
        band = _f32(np.arange(T.TOP_BAND[0], T.TOP_BAND[1] + 1, dtype=np.uint32) | np.uint32(s))
        hi, _ = T.split(band, rounding=_unguarded)
        assert np.isnan(hi).all()
        hi, lo = T.split(band)
        assert np.isfinite(hi).all() and np.isfinite(lo).all()
        below = _f32([0x7F7FEFFF | s])
        assert np.array_equal(T.split(below, rounding=_unguarded)[0].view(np.uint32), T.split(below)[0].view(np.uint32))
        assert np.isfinite(T.split(below)[0]).all()
