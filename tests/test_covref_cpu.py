"""The K5 covariance reference (tests/covref.py) on the CPU: it agrees with the oracle's restatement of
computeCovariances, its far-face fixtures defeat the ring search's old stop rule, and each named way of getting K5
subtly wrong is caught by at least one fixture."""
import numpy as np
import pytest

import covref as CR
import gridref as GR

F32 = np.float32
KS = (3, 4, 20, 31, 32)


def _oracle_cov(oracle_mod, cloud, k, eps):
    o = oracle_mod.GICP(k_correspondences=k, gicp_epsilon=eps, max_iterations=1)
    o.set_target(cloud)
    o.set_source(cloud)
    o.align()
    return o.covariances("target")


@pytest.mark.parametrize("k", [4, 20])
def test_reference_matches_oracle(oracle_mod, k):
    for eps in (1e-3, 0.25):
        for name, c in CR.cov_fixtures(k).items():
            if name == "nonfinite" or len(c) < k:  # the oracle has no notion of non-finite rows
                continue
            # where C is an unrotated diagonal the oracle completes the columns of zero singular values by Gram-Schmidt,
            # which differs from Eigen's sort on diag(0, 0, s) alone (the "line z" fixture): compare its own rule there
            ref, info = CR.reference(c, k, eps, column="completion")
            bad, ratio, _ = CR.check(_oracle_cov(oracle_mod, c, k, eps), ref, info)
            assert not bad.any(), (name, k, eps, np.flatnonzero(bad)[:5])
            assert ratio <= 1.0


def test_exact_ties_take_eigens_column():
    # zero covariance: Eigen stops its sort at once, U = I, the last column is z
    ref, info = CR.reference(CR.dyadic_duplicates(20), 20)
    assert info["flat"].all() and np.all(info["C"] == 0)
    np.testing.assert_array_equal(np.diagonal(ref, axis1=1, axis2=2)[0], [1.0, 1.0, 1.0 - (1.0 - 1e-3)])
    # a line along y: diag(0, s, 0) -> the sort swaps y to the front and stops at the zero maximum: z is last
    assert CR.eigen_last_column([0.0, 2.0, 0.0]) == 2 and CR.eigen_last_column([0.0, 0.0, 2.0]) == 0
    assert CR.eigen_last_column([2.0, 0.0, 0.0]) == 2 and CR.eigen_last_column([1.0, 1.0, 3.0]) == 0
    assert CR.eigen_last_column([1.0, 1.0, 1.0]) == 2 and CR.eigen_last_column([3.0, 1.0, 1.0]) == 2


def test_knn_candidates_are_complete():
    """The cKDTree path (forced by brute_limit=0) returns the brute-force neighbours, ties and order included."""
    for name, c in (("lattice", GR.lattice((7, 6, 5), (1.0, 1.0, 0.5))), ("scene", CR.scene(1200, seed=3)),
                    ("nonfinite", GR.with_nonfinite_rows(CR.scene(600, seed=4), seed=4)[0][:, :3])):
        for k in (3, 20, 32):
            Ib, Db = CR.knn(c, k)
            It, Dt = CR.knn(c, k, brute_limit=0)
            np.testing.assert_array_equal(It, Ib, err_msg=f"{name} {k}")
            np.testing.assert_array_equal(Dt, Db, err_msg=f"{name} {k}")


def test_far_face_fixtures_defeat_the_old_stop_rule():
    f = CR.far_face_case("1nn")
    for rule, want in (("old", f["want"] - 1), ("sound", f["want"])):
        bi, _ = CR.ring_search(f["target"], f["query"][0], 1, rule)
        assert bi[0] == want, (rule, bi)
    assert GR.nn1_ref(f["target"], f["query"])[0][0] == f["want"]
    for k in KS:
        f = CR.far_face_case("knn", k)
        I, _ = CR.knn(f["target"], k)
        q = 8  # the query's own row
        assert f["want"] in I[q] and f["want"] - 1 not in I[q]
        old, _ = CR.ring_search(f["target"], f["query"][0], k, "old")
        sound, _ = CR.ring_search(f["target"], f["query"][0], k, "sound")
        assert set(old.tolist()) != set(I[q].tolist()) and f["want"] - 1 in old, k
        assert sound.tolist() == I[q].tolist(), k
    g = CR.far_face_gated()
    max_d2 = F32(F32(g["d2"]) * F32(1.0001)) + F32(1e-30)  # getFitnessScore(d2) and the correspondence search's slack
    assert len(CR.ring_search(g["target"], g["query"][0], 1, "old", max_d2=max_d2)[0]) == 0
    bi, bd = CR.ring_search(g["target"], g["query"][0], 1, "sound", max_d2=max_d2)
    assert bi[0] == g["want"] and bd[0] == g["d2"] and bd[0] < 0.99989 * float(g["geometry"]["h"]) ** 2


def test_face_queries_reach_the_last_cell():
    t = CR.corridor()
    g = GR.nn_geometry(t)
    q = CR.face_queries(t)
    cx = np.floor((q[:, 0] - g["origin"][0]) * g["inv_h"])
    assert g["dims"][0] > 1000 and cx.max() >= g["dims"][0] - 1 and len(q) >= 3 * (g["dims"][0] + 1)


MUTATIONS = {
    "higher-index ties at the k-th neighbour": dict(higher_index_ties=True),
    "the old stop rule": dict(stop_rule="old"),
    "f64 products": dict(f64_products=True),
    "the first-minimum column": dict(column="first"),
    "eps on the wrong column": dict(eps_column="largest"),
    "division by the neighbour count k - 1": "divisor",
}


@pytest.mark.parametrize("mutation", list(MUTATIONS))
def test_mutations_are_caught(mutation):
    caught = []
    for k in (4, 20):
        mut = MUTATIONS[mutation]
        mut = dict(divisor=k - 1) if mut == "divisor" else mut
        for name, c in CR.cov_fixtures(k).items():
            if len(c) < k or (mutation == "the old stop rule" and len(c) > 200):  # the restated walk is slow
                continue
            ref, info = CR.reference(c, k)
            got, _ = CR.reference(c, k, **mut)
            bad, _, _ = CR.check(got, ref, info)
            if bad.any():
                caught.append((k, name, int(bad.sum())))
    assert caught, mutation
