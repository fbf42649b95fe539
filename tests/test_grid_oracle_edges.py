"""CPU: the grid-subsampling oracle (oracle/grid_oracle.c, the yardstick of tests/test_gpu_grid.py) against the
reference's own compiled ``grid_subsampling`` (oracle/_ref/libgrid_ref.so) on the edge cases of
tests/grid_edges.py: negative voxel indices, clouds far from the origin, wrapping keys, NaN and ±inf, a voxel of
more than 2^24 points, wide features and extreme labels.  The oracle's own voxel keys are checked against the
numpy restatement of the reference's x86-64 key arithmetic, which the device test relies on."""
import numpy as np
import pytest

import grid_edges as E
from oracle import cpu_oracle as O


@pytest.fixture(scope="module")
def reference():
    from oracle import ref_loader as R
    if not R.grid_available():
        if R.reference_sources_present():
            pytest.fail("%s is missing although the reference's sources are present: build() compiles it "
                        "(make -C oracle ref)" % R.GRID_SO)
        pytest.skip("%s is not built and the reference's sources are not on this machine: nothing to compare "
                    "the oracle with" % R.GRID_SO)

    def fn(pts, feats, labels, dl):
        out = R.grid_subsampling(pts, feats, labels, dl)
        return out[0], (out[1] if feats is not None else None), (out[-1] if labels is not None else None)
    return fn


class Oracle:
    """oracle.grid_sub_sampling in the form grid_edges.run takes; keeps the keys the oracle reports."""

    def __call__(self, pts, feats, labels, dl):
        out = O.grid_sub_sampling(pts, feats, labels, dl)
        self.keys = out[-1]
        return out[0], (out[1] if feats is not None else None), (out[-2] if labels is not None else None)


def check(reference, case):
    oracle = Oracle()
    got = E.run(oracle, case)
    E.assert_matches_reference(got, E.run(reference, case), case)
    assert np.array_equal(oracle.keys, got[3]), "the oracle's keys are not the restatement's"
    return got


def test_size_t_of_is_the_x86_conversion():
    f = np.array([-1, -0.5, -0.0, 5, np.nan, np.inf, -np.inf, 2.0 ** 63, 1.5e19, 2.0 ** 64, 1e30, -1e30],
                 np.float32)
    want = [2 ** 64 - 1, 2 ** 64 - 1, 0, 5, 2 ** 63, 0, 2 ** 63, 2 ** 63, 15000000520515485696, 0, 0, 2 ** 63]
    assert E.size_t_of(np.floor(f)).tolist() == want


def test_negative_index_four_points(reference):
    """min x = -3.7, dl = 0.02: the float32 origin is -3.6999998, the first point's x index is -1 and wraps into
    the voxel at the end of the row below, which is empty: four voxels.  A saturating cast merges the first
    two points into three."""
    case = E.Case(E.FOUR_POINTS, 0.02, np.arange(12, dtype=np.float32).reshape(4, 3), np.arange(4))
    org, _, _ = E.grid_frame(case.pts, case.dl)
    assert org[0] == np.float32(-3.6999998) and org[0] > case.pts[0, 0]
    assert E.voxel_indices(case.pts, case.dl)[0, 0] == 2 ** 64 - 1
    assert len(check(reference, case)[0]) == 4


@pytest.mark.parametrize("dl", E.NEG_DLS + (0.01, 0.05))
def test_negative_index_search(reference, dl):
    """Every (min, dl) pair the search finds, on each axis: the oracle wraps the -1 index as the reference does."""
    n = 0
    for m, a, case in E.negative_index_pair_clouds(dl):
        assert E.voxel_indices(case.pts, dl)[0, a] == 2 ** 64 - 1, (m, a)
        sp = check(reference, case)[0]
        assert len(sp) == (2 if a < 2 else 3), (m, a)            # A merges into B's voxel unless a is z
        n += 1
    assert n >= 3 * 5, "the search found only %d clouds at dl=%g" % (n, dl)


@pytest.mark.parametrize("seed", [0, 1])
@pytest.mark.parametrize("axes", E.NEG_AXES)
@pytest.mark.parametrize("dl", E.NEG_DLS)
def test_negative_index_clouds(reference, dl, axes, seed):
    check(reference, E.negative_index_case(dl, axes, seed))


@pytest.mark.parametrize("lattice", [False, True])
@pytest.mark.parametrize("seed", [0, 1])
@pytest.mark.parametrize("dl", E.FAR_DLS)
@pytest.mark.parametrize("offset", E.FAR_OFFSETS)
def test_far_from_origin(reference, offset, dl, seed, lattice):
    check(reference, E.far_case(offset, dl, seed, lattice))


@pytest.mark.parametrize("seed", [0, 1])
@pytest.mark.parametrize("e", [0, 10, 20])
def test_key_collision(reference, e, seed):
    case = E.key_collision_case(e, seed)
    sp = check(reference, case)[0]
    assert len(sp) < len(np.unique(E.voxel_indices(case.pts, case.dl), axis=0))


@pytest.mark.parametrize("seed", [0, 1])
@pytest.mark.parametrize("dl,extent", E.WIDE)
def test_key_overflow_wide(reference, dl, extent, seed):
    check(reference, E.wide_case(dl, extent, seed))


@pytest.mark.parametrize("seed", [0, 1])
@pytest.mark.parametrize("kind", E.NON_FINITE)
def test_non_finite(reference, kind, seed):
    check(reference, E.non_finite_case(kind, seed))


@pytest.mark.parametrize("n", [1, 100003])
def test_one_voxel(reference, n):
    case = E.one_voxel_case(n, 0)
    assert len(check(reference, case)[0]) == 1


def test_voxel_of_2_24_plus_3_points(reference):
    """One voxel of 2^24 + 3 points: the sum of ones stops at 2^24 and (float)count rounds to 2^24 + 4."""
    case = E.one_voxel_case(2 ** 24 + 3, 1)
    got = E.run(Oracle(), case, with_keys=False)
    want = E.run(reference, case, with_keys=False)
    assert len(got[0]) == len(want[0]) == 1
    E.same_bits(got[0], want[0], "barycentre")
    E.same_bits(got[1], want[1], "mean feature")
    assert got[1][0, 0] == np.float32(2 ** 24) / np.float32(2 ** 24 + 3) != 1
    assert got[2][0, 0] == want[2][0, 0] == 0


@pytest.mark.parametrize("seed", [0, 1])
@pytest.mark.parametrize("dl", [0.03, 0.1])
@pytest.mark.parametrize("fdim", E.FDIMS)
def test_features(reference, fdim, dl, seed):
    check(reference, E.features_case(fdim, dl, seed))


@pytest.mark.parametrize("seed", [0, 1])
@pytest.mark.parametrize("dl", [0.03, 0.1])
@pytest.mark.parametrize("ldim", E.LDIMS)
def test_labels(reference, ldim, dl, seed):
    case = E.labels_case(ldim, dl, seed)
    got = check(reference, case)
    _, tables = E.vote_tables(case)
    assert (tables[0][2] > 1).any() and (tables[0][2] == 1).any()     # tied and untied voxels both occur
    v0 = np.searchsorted(got[3], E.voxel_keys(case.pts, case.dl)[0])
    assert got[2][v0].tolist() == [(E.INT_MAX, -1, 0, E.INT_MIN, 0)[l] for l in range(ldim)]
