"""CPU: the searches the scheduler does not run are exactly slices of searches it does run.

``tables.derived_searches`` (row prefixes: cloud level j = first rows of level i < j) and
``tables.derived_image_searches`` (strided pixel subsets: image level 2s = every other pixel of every other row of
level s) are checked on the point sets of a synthetic frame, and the index arrays the oracle computes for the child
searches are compared with the slices of the parents' arrays."""
import numpy as np

from conftest import frame_point_sets
from ffb6d_b200 import tables as T
from ffb6d_b200.synthetic import make_frame
from oracle import cpu_oracle as O

N_POINTS, H, W = 3072, 480, 640


def test_child_query_sets_are_slices_and_results_match():
    fr = make_frame(3, n_points=N_POINTS)
    sets = frame_point_sets(fr, N_POINTS)
    calls = T.knn_schedule(N_POINTS, H, W, 16)
    by_key = {key: (s, q, kk) for key, s, q, kk in calls}
    prefix = T.derived_searches(calls)
    strided = T.derived_image_searches(calls, H, W)
    assert len(prefix) == 4 and len(strided) == 3
    assert not set(prefix) & set(strided)
    assert all(p not in prefix and p not in strided for p in list(prefix.values()) + [p for p, _ in strided.values()])
    cache = {}

    def search(key):
        if key not in cache:
            s, q, kk = by_key[key]
            cache[key] = O.knn_search(sets[s][None], sets[q][None], kk)[0]
        return cache[key]

    for child, parent in prefix.items():
        (s_c, q_c, k_c), (s_p, q_p, k_p) = by_key[child], by_key[parent]
        assert s_c == s_p and k_c == k_p
        n = sets[q_c].shape[0]
        assert np.array_equal(sets[q_c], sets[q_p][:n])                      # the query set IS a row prefix
        assert np.array_equal(search(child), search(parent)[:n]), child
    for child, (parent, f) in strided.items():
        (s_c, q_c, k_c), (s_p, q_p, k_p) = by_key[child], by_key[parent]
        assert s_c == s_p and k_c == k_p == 1 and q_c[1] == q_p[1] * f
        hp, wp = H // q_p[1], W // q_p[1]
        sub = sets[q_p].reshape(hp, wp, 3)[::f, ::f].reshape(-1, 3)
        assert np.array_equal(sub, sets[q_c])                                # the query set IS the strided subset
        want = search(parent).reshape(hp, wp, 1)[::f, ::f].reshape(-1, 1)
        assert np.array_equal(search(child), want), child


def test_no_strided_derivation_for_indivisible_images():
    calls = T.knn_schedule(N_POINTS, 482, 642, 16)
    assert T.derived_image_searches(calls, 482, 642) == {}                   # not a multiple of 4: every search runs
    d = T.derived_image_searches(calls, 484, 644)                            # multiples of 4, not of 8
    assert set(d) == {"p2r_ds_nei_idx0"}

