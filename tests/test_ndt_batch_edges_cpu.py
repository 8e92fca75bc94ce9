"""The generators of tests/ndtbatchref.py reach the edges they are named for, checked without a GPU: the size ladder lands
on both sides of every rows_for and staging boundary, the iteration limits give launches of 1, 2 and 4 registrations,
the job orders put the ladder top next to a 1-point job, same-size jobs differ on every evaluator CTA, the pageable scan
takes the four-thread staging path, every record stride keeps x, y, z where the solver reads them, the edge guesses
leave the fast controller in the float64 replay, the leaf-edge points sit where the multiply and divide cells disagree,
and K12's scan sizes straddle its tile multiples."""
import numpy as np
import pytest

import gridref as R
import ndtbatchref as B
import ndtctl_ref as X
import ndtref as N

F32 = np.float32


@pytest.mark.parametrize("n_sms", [B.H100_SXM_SMS, 100, 20])
def test_size_ladder_straddles_every_boundary(n_sms):
    e = B.n_eval(n_sms)
    assert B.n_eval(B.H100_SXM_SMS) == 129
    sizes = B.size_ladder(n_sms)
    assert sizes == sorted(sizes) and len(set(sizes)) == len(sizes)
    cap = B.staging_capacity(e)
    rows = [B.rows_for(n, e) for n in sizes]
    # ragged 32-point units, and rows_for stepping from one CTA to two at 128 / 129 points
    assert {31, 32, 33} <= set(sizes) and rows[sizes.index(128)] == 1 and rows[sizes.index(129)] == 2
    # the last size spread over fewer than all evaluators, then all of them
    assert B.rows_for(128 * e - 1, e) == e and B.rows_for(128 * (e - 1), e) == e - 1
    assert rows[sizes.index(128 * e)] == e == rows[sizes.index(128 * e + 1)]
    assert B.rows_for(128 * e - 129, e) == e - 1
    # the staging capacity: below it every point is staged, above it some thread reads from global memory
    for n, staged in ((cap - 33, True), (cap + 33, False), (sizes[-1], False)):
        units = (n + 31) // 32
        per_cta = -(-units // B.rows_for(n, e)) * 32
        assert (per_cta <= N.SMEM_POINTS) == staged, (n_sms, n)
    assert sizes[-1] > 2 * cap  # a thread of the top job evaluates three points, two of them read from global memory
    assert N.points_per_thread(sizes[-1], n_sms) >= 3
    # ndtref's points-per-thread depth sees the second point beyond the capacity
    assert N.points_per_thread(cap - 33, n_sms) == 1 and N.points_per_thread(cap + 33, n_sms) == 2


def test_ladder_order_puts_the_top_next_to_one_point():
    sizes = B.size_ladder(B.H100_SXM_SMS)
    order = B.ladder_order(sizes)
    assert len(order) >= 64
    seq = [sizes[i] for i in order]
    pairs = set(zip(seq, seq[1:]))
    assert (B.LADDER_TOP, 1) in pairs and (1, B.LADDER_TOP) in pairs
    assert all(seq.count(n) >= 5 for n in sizes)
    scan = np.random.default_rng(0).normal(size=(B.LADDER_TOP + 5000, 3)).astype(F32)
    jobs = B.ladder_jobs(scan, sizes, order, [np.eye(4, dtype=F32)])
    assert [len(p) for p, _ in jobs] == seq
    # equal sizes next to each other (where one copy ends and the next begins) never carry the same points
    for (a, _), (b, _) in zip(jobs, jobs[1:]):
        if len(a) == len(b):
            assert not np.array_equal(a, b)


def test_launch_arithmetic():
    assert B.per_launch(35) == 1538
    for pl, m in B.CHUNK_MAX_ITERATIONS.items():
        assert B.per_launch(m) == pl and B.per_launch(m - 1) >= pl
    assert B.per_launch(m + 1) == 1 and B.per_launch(10**6) == 1  # never fewer than one
    assert B.launch_counts(1) == [1, 2, 4]
    assert B.launch_counts(2) == [1, 2, 3, 7] and B.launch_counts(4) == [3, 4, 5, 13]
    for pl in B.CHUNK_MAX_ITERATIONS:
        cs = B.launch_counts(pl)
        assert max(cs) > pl and pl in cs and (-(-max(cs) // pl)) == 4


@pytest.mark.parametrize("n_sms", [B.H100_SXM_SMS, 40])
def test_same_size_pairs_differ_on_every_cta(n_sms):
    src = np.random.default_rng(1).normal(size=(B.LADDER_TOP, 3)).astype(F32)
    sizes = B.size_ladder(n_sms)
    pairs = B.same_size_pairs(src, sizes, seed=3)
    for k, (a, b) in enumerate(pairs):
        assert a.shape == b.shape == (sizes[k], 3) and a.dtype == b.dtype == F32
        differ, owners = B.ranks_that_differ(a, b, n_sms)
        assert differ == owners, (sizes[k], len(owners - differ))
        if k % 2 == 0 and sizes[k] > 1:  # the same points in another order
            assert np.array_equal(np.sort(a, axis=0), np.sort(b, axis=0))
        else:  # every point moved a little
            assert (a != b).any(axis=1).all() and np.abs(a - b).max() < 0.2


def test_record_builders():
    p = np.random.default_rng(2).normal(size=(1000, 3)).astype(F32)
    for stride in B.STRIDES:
        r = B.records(p, stride, seed=stride)
        assert r.strides[0] == stride and r.flags.c_contiguous and r.dtype == F32
        assert np.array_equal(r[:, :3], p)
        if stride == 16:
            assert np.isnan(r[::2, 3]).all() and np.isinf(r[1::4, 3]).all() and np.isfinite(r[3::4, 3]).all()
            assert (np.abs(r[3::4, 3]) > 1e3).mean() > 0.9  # garbage, not the homogeneous 1
        if stride > 16:
            assert np.isnan(r[:, 3:]).any() and (r[:, 3:] != 1).all()
    big = B.records(np.zeros((B.PAGEABLE_POINTS, 3), F32), 32)
    assert big.nbytes >= B.FOUR_THREAD_BYTES and big.strides[0] == 32


def test_edge_guesses_leave_the_fast_controller(oracle_mod, golden, pair_small):
    """On the golden PCD (resolution 1): the guess 10 km away has zero hits, so the first solve sees H = 0, which the fast
    path's LDL^T refuses; the ascent guesses reach an ascent round; the edge guesses a snap round; with max_iterations
    1 and 2 the solve ends at the iteration cap."""
    gs, gt = golden["source"], golden["target"]
    cfg = X.config()
    o = oracle_mod.NDT(resolution=1.0, num_threads=1)
    o.set_target(gt)
    o.set_source(gs)
    guesses = B.controller_edge_guesses()
    recs, res, infos = X.drive(o, B.far_guess(), cfg, len(gs))
    assert all(int(r["tot"][28]) == 0 and r["score"] == 0 for r in recs if r["evaluated"])
    first = infos[0]
    assert first["H_full"] is not None and not X.ldlt_accepts(first["H_full"]) and res["converged"]
    assert res["iterations"] == 0 and res["evaluations"] == 1 and np.array_equal(res["final_T"], B.far_guess())
    assert X.first_with(o, cfg, guesses, len(gs), X.is_ascent_round) is not None
    assert X.first_with(o, cfg, guesses, len(gs), X.is_snap_round) is not None
    osrc, otgt = X.origin_pair()
    oo = oracle_mod.NDT(resolution=2.0, num_threads=1)
    oo.set_target(otgt)
    oo.set_source(osrc)
    _, _, infos = X.drive(oo, np.eye(4, dtype=F32), cfg, len(osrc))
    assert any(i["H_full"] is not None and not X.ldlt_accepts(i["H_full"]) for i in infos)
    src, tgt, _ = pair_small
    for m in B.EDGE_MAX_ITERATIONS:
        c = X.config(max_iterations=m)
        om = oracle_mod.NDT(resolution=2.0, max_iterations=m, num_threads=1)
        om.set_target(tgt)
        om.set_source(src)
        _, r, _ = X.drive(om, np.eye(4, dtype=F32), c, len(src))
        assert r["iterations"] == m + 2 and r["converged"], (m, r)


@pytest.mark.parametrize("res", [0.3, 0.1])
def test_leaf_edge_points_disagree(res):
    src, tgt = B.leaf_edge_source(res)
    x = src[:, 0]
    assert len(x) >= 150
    assert (np.floor(x * (F32(1) / F32(res))) != np.floor(x / F32(res))).all()
    assert R.mul_div_disagree(x, res).all()
    for u in (-1, 1):
        # one ulp away, some points fall on the other side of the edge the lookup uses
        xn = B.nudged(src, u)[:, 0]
        assert (R.lookup_ref(xn, res) != R.lookup_ref(x, res)).any() and np.all(np.abs(xn - x) > 0)
    assert len(R.voxel_map_ref(tgt, res)["idx"]) > 0


def test_tile_sizes_straddle_multiples_of_1024():
    sizes = B.tile_sizes()
    tiles = [-(-n // B.SCORE_TILE) for n in sizes]
    for k in (1, 2, 3):
        m = B.SCORE_TILE * k
        assert {m - 1, m, m + 1} <= set(sizes)
        assert tiles[sizes.index(m - 1)] == tiles[sizes.index(m)] == k and tiles[sizes.index(m + 1)] == k + 1
    assert sizes[-1] % B.SCORE_TILE and sizes[-1] // B.SCORE_TILE >= 97
