"""GPU: ``grid_sub_sampling`` (ffb6d_grid_subsample_host) against the reference's own compiled
``grid_subsampling`` (oracle/_ref/libgrid_ref.so) at the edges of its voxel arithmetic (tests/grid_edges.py):
negative voxel indices, clouds 1e3 - 1e5 m from the origin, keys that wrap 2^64 (and voxels that share a key),
NaN and ±inf, one voxel of 2^24 + 3 points, N = 1, wide features and extreme labels.

Rows are matched by voxel key and must also come out by ascending key; barycentres and mean features are
compared bit for bit (NaNs by position); labels are exact except where several tie for the top count, where the
device's is the smallest of them and the reference's one of them."""
import resource
import time

import numpy as np
import pytest

import ffb6d_b200 as F
import grid_edges as E

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def reference():
    from oracle import ref_loader as R
    if not R.grid_available():
        pytest.fail("%s is missing: build() compiles the reference's grid_subsampling into it where the "
                    "reference's sources are present (make -C oracle ref), and the file must travel with the "
                    "tree; without it this file has nothing to compare with" % R.GRID_SO)

    def fn(pts, feats, labels, dl):
        out = R.grid_subsampling(pts, feats, labels, dl)
        return out[0], (out[1] if feats is not None else None), (out[-1] if labels is not None else None)
    return fn


def device(pts, feats, labels, dl):
    out = F.grid_sub_sampling(pts, features=feats, labels=labels, grid_size=dl)
    if not isinstance(out, tuple):
        out = (out,)
    return out[0], (out[1] if feats is not None else None), (out[-1] if labels is not None else None)


def check(reference, case):
    got = E.run(device, case)
    E.assert_matches_reference(got, E.run(reference, case), case)
    return got


def test_negative_index_four_points(cuda, reference):
    """min x = -3.7, dl = 0.02: the float32 origin -3.6999998 lies above the first point, whose x index -1 wraps
    into the (empty) voxel at the end of the row below: four voxels, as the reference returns."""
    case = E.Case(E.FOUR_POINTS, 0.02, np.arange(12, dtype=np.float32).reshape(4, 3), np.arange(4))
    assert E.voxel_indices(case.pts, case.dl)[0, 0] == 2 ** 64 - 1
    assert len(check(reference, case)[0]) == 4


@pytest.mark.parametrize("dl", E.NEG_DLS + (0.01, 0.05))
def test_negative_index_search(cuda, reference, dl):
    """Every (min, dl) pair the float32 search finds, with the -1 index on each axis in turn."""
    n = 0
    for m, a, case in E.negative_index_pair_clouds(dl):
        try:
            sp = check(reference, case)[0]
        except AssertionError as e:
            raise AssertionError("min %r on axis %d: %s" % (m, a, e)) from None
        assert len(sp) == (2 if a < 2 else 3), (m, a)
        n += 1
    print("dl=%g: %d (min, axis) clouds" % (dl, n))
    assert n >= 3 * 5, "the search found only %d clouds at dl=%g" % (n, dl)


@pytest.mark.parametrize("seed", [0, 1])
@pytest.mark.parametrize("axes", E.NEG_AXES)
@pytest.mark.parametrize("dl", E.NEG_DLS)
def test_negative_index_clouds(cuda, reference, dl, axes, seed):
    check(reference, E.negative_index_case(dl, axes, seed))


@pytest.mark.parametrize("lattice", [False, True])
@pytest.mark.parametrize("seed", [0, 1])
@pytest.mark.parametrize("dl", E.FAR_DLS)
@pytest.mark.parametrize("offset", E.FAR_OFFSETS)
def test_far_from_origin(cuda, reference, offset, dl, seed, lattice):
    check(reference, E.far_case(offset, dl, seed, lattice))


@pytest.mark.parametrize("seed", [0, 1])
@pytest.mark.parametrize("e", [0, 10, 20])
def test_key_collision(cuda, reference, e, seed):
    """NX = NY = 2^24: voxels 2^16 apart in z share a key, and the device merges them as the reference does."""
    case = E.key_collision_case(e, seed)
    sp = check(reference, case)[0]
    assert len(sp) < len(np.unique(E.voxel_indices(case.pts, case.dl), axis=0))


@pytest.mark.parametrize("seed", [0, 1])
@pytest.mark.parametrize("dl,extent", E.WIDE)
def test_key_overflow_wide(cuda, reference, dl, extent, seed):
    check(reference, E.wide_case(dl, extent, seed))


@pytest.mark.parametrize("seed", [0, 1])
@pytest.mark.parametrize("kind", E.NON_FINITE)
def test_non_finite(cuda, reference, kind, seed):
    check(reference, E.non_finite_case(kind, seed))


@pytest.mark.parametrize("n", [1, 100003])
def test_one_voxel(cuda, reference, n):
    assert len(check(reference, E.one_voxel_case(n, 0))[0]) == 1


def test_voxel_of_2_24_plus_3_points(cuda, reference):
    """One voxel of 2^24 + 3 points: the fp32 sum of the features (ones) stops at 2^24 and (float)count rounds
    to 2^24 + 4, so the mean is 2^24 / (2^24 + 4); the barycentre takes the double reciprocal of the count."""
    with open("/proc/self/statm") as fh:
        rss0 = int(fh.read().split()[1]) * resource.getpagesize() / 2 ** 20
    t0 = time.perf_counter()
    case = E.one_voxel_case(2 ** 24 + 3, 1)
    got = E.run(device, case, with_keys=False)
    t1 = time.perf_counter()
    want = E.run(reference, case, with_keys=False)
    t2 = time.perf_counter()
    assert len(got[0]) == len(want[0]) == 1
    E.same_bits(got[0], want[0], "barycentre")
    E.same_bits(got[1], want[1], "mean feature")
    assert got[1][0, 0] == np.float32(2 ** 24) / np.float32(2 ** 24 + 3) != 1
    assert got[2][0, 0] == want[2][0, 0] == 0
    peak = resource.getrusage(resource.RUSAGE_SELF).ru_maxrss / 1024
    print("2^24+3 points: inputs %.0f MB, device %.2f s, reference %.2f s; host RSS %.0f MB before the case, "
          "process peak %.0f MB" % ((case.pts.nbytes + case.feats.nbytes + case.labels.nbytes) / 2 ** 20,
                                    t1 - t0, t2 - t1, rss0, peak))


@pytest.mark.parametrize("seed", [0, 1])
@pytest.mark.parametrize("dl", [0.03, 0.1])
@pytest.mark.parametrize("fdim", E.FDIMS)
def test_features(cuda, reference, fdim, dl, seed):
    check(reference, E.features_case(fdim, dl, seed))


@pytest.mark.parametrize("seed", [0, 1])
@pytest.mark.parametrize("dl", [0.03, 0.1])
@pytest.mark.parametrize("ldim", E.LDIMS)
def test_labels(cuda, reference, ldim, dl, seed):
    case = E.labels_case(ldim, dl, seed)
    got = check(reference, case)
    v0 = np.searchsorted(got[3], E.voxel_keys(case.pts, case.dl)[0])
    assert got[2][v0].tolist() == [(E.INT_MAX, -1, 0, E.INT_MIN, 0)[l] for l in range(ldim)]
