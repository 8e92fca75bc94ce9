"""Fixture builders and launch arithmetic for the edge tests of the NDT batch solver (b200reg_ndt_align_batch /
_device) and of the pose scorer K12 (b200reg_ndt_score_poses). Nothing here needs a GPU except the pinned record
builder, which asks torch for page-locked memory.

What is restated, from ndt_solver.cu, capi.cu and cloud_codec.cu
  * rows_for(n, E): the evaluator CTAs a scan of n points is dealt over, E = SMs - 3 (132 - 3 = 129 on an H100 SXM).
  * staging_capacity(E) = 768 E: points beyond it are read from the caller's records (global memory) on every round.
  * per_launch(max_iterations) = max(1, 60000 // (max_iterations + 4)): a batch call is cut into launches of that many
    registrations; a call with more than one launch's worth also gives up the streaming upload for the unpack path.
  * staged_h2d stages a pageable source of 8 MiB or more with four host threads.
  * K12 stages the scan in tiles of 1024 points.

The generators, and the edge each reaches (tests/test_ndt_batch_edges_cpu.py checks every one):
  * size_ladder: both sides of every rows_for and staging boundary, topped by a scan read mostly from global memory;
  * ladder_order: a ladder-top job directly before a 1-point job and directly after one, 64 jobs or more;
  * same_size_pairs: two jobs of equal size whose points differ on every evaluator CTA (a re-staging shortcut keyed on
    the size would evaluate the first job's points for the second);
  * far_guess / controller_edge_guesses: registrations that leave the fast controller (zero hits, an indefinite Hessian,
    the 1e-4 angle snap) and EDGE_MAX_ITERATIONS, which end at the iteration cap;
  * records: the scan at every record stride the host path accepts, garbage in every float past x, y, z;
  * launch_counts / CHUNK_MAX_ITERATIONS: one launch short of, exactly at and past per_launch = 1, 2 and 4.
"""
from __future__ import annotations

import numpy as np

import ndtctl_ref as X
import ndtref as N

F32 = np.float32
MAX_ROUNDS_PER_LAUNCH = 60000  # NdtSolver::kMaxRoundsPerLaunch (engine.hpp)
H100_SXM_SMS = 132
FOUR_THREAD_BYTES = 8 << 20  # staged_h2d: pageable sources of this size or more are staged by four host threads
SCORE_TILE = 1024  # SCORE_TILE of ndt_score.cu
STRIDES = (12, 16, 20, 32, 48)  # bytes per host record
PAGEABLE_POINTS = 300_000  # x 32 B = 9.6 MB: above FOUR_THREAD_BYTES
LADDER_TOP = 250_000
# max_iterations -> per_launch of 4, 2 and 1
CHUNK_MAX_ITERATIONS = {4: 14996, 2: 29996, 1: 59996}
EDGE_MAX_ITERATIONS = (1, 2)
FAR = 10_000.0  # metres: a guess this far off leaves every point outside the grid (zero hits)


def n_eval(n_sms):
    """Evaluator CTAs of a solver launch: every SM but the NDT_MAX_SLOTS kept for controllers."""
    return max(1, n_sms - N.CTL_CTAS)


def rows_for(n, e):
    return max(1, min((n + 127) // 128, e))


def staging_capacity(e):
    return N.SMEM_POINTS * e


def per_launch(max_iterations):
    return max(1, MAX_ROUNDS_PER_LAUNCH // (max_iterations + 4))


def launch_counts(pl):
    """Batch sizes around a launch of pl registrations: one short of it (when that is a batch), one launch, one
    registration into the next launch, and three launches and one."""
    return [c for c in (pl - 1, pl, pl + 1, 3 * pl + 1) if c > 0]


def size_ladder(n_sms, top=LADDER_TOP):
    """Ragged units, one CTA's four warps, the last size spread over fewer than all evaluators, and both sides of the
    staging capacity; the top of the ladder reads most of its points from global memory."""
    e = n_eval(n_sms)
    cap = staging_capacity(e)
    return [1, 31, 32, 33, 127, 128, 129, 128 * e - 1, 128 * e, 128 * e + 1, cap - 33, cap + 33, top]


def ladder_order(sizes, copies=5):
    """Indices into `sizes` (ascending): the largest, the smallest, the second largest, the second smallest, ... and that
    order reversed, alternately, `copies` times: every copy puts the top job directly before or after a 1-point job."""
    asc = list(range(len(sizes)))
    desc = asc[::-1]
    half = (len(sizes) + 1) // 2
    one = [x for pair in zip(desc[:half], asc[:half]) for x in pair][:len(sizes)]
    assert sorted(one) == asc
    out = []
    for c in range(copies):
        out += one if c % 2 == 0 else one[::-1]
    return out


def tiled_scan(src, n, offsets=((0.0, 0.0, 0.0), (0.013, -0.007, 0.005), (-0.011, 0.009, -0.004), (0.006, 0.012, -0.009))):
    """At least n points: the scan repeated with millimetre offsets (a 128-ring sensor's density)."""
    reps = -(-n // len(src))
    assert reps <= len(offsets), (n, len(src))
    out = np.concatenate([np.asarray(src, F32)[:, :3] + F32(o) for o in np.array(offsets[:reps], dtype=F32)])
    return np.ascontiguousarray(out[:n], dtype=F32)


def ladder_jobs(scan, sizes, order, guesses, shift=1000):
    """The (points, guess) of each job of `order`: copy c of a size starts c * shift rows into `scan`, so two jobs of one
    size never hold the same points."""
    seen = {}
    out = []
    for k, i in enumerate(order):
        c = seen.get(i, 0)
        seen[i] = c + 1
        n = sizes[i]
        assert c * shift + n <= len(scan)
        out.append((np.ascontiguousarray(scan[c * shift:c * shift + n]), guesses[k % len(guesses)]))
    return out


def same_size_pairs(src, sizes, seed=0):
    """[(a, b)] with len(a) == len(b): b is a jittered copy of a (odd entries, and size 1) or a rotated copy of its rows
    (even entries)."""
    rng = np.random.default_rng(seed)
    out = []
    for k, n in enumerate(sizes):
        a = np.ascontiguousarray(np.asarray(src, F32)[:n, :3])
        if k % 2 or n == 1:
            b = a + rng.normal(0, 0.02, a.shape).astype(F32)
        else:
            b = np.roll(a, n // 2 + 1, axis=0)
        out.append((a, np.ascontiguousarray(b, dtype=F32)))
    return out


def ranks_that_differ(a, b, n_sms):
    """Evaluator CTAs whose points (ndtref.point_owner's deal) differ between two same-size scans, and the CTAs that own
    points at all."""
    rank, _, rows = N.point_owner(len(a), n_sms)
    diff = (np.asarray(a) != np.asarray(b)).any(axis=1)
    return set(np.unique(rank[diff]).tolist()), set(range(rows))


def far_guess(dist=FAR):
    T = np.eye(4, dtype=F32)
    T[0, 3], T[1, 3] = F32(dist), F32(-dist / 2)
    return T


def controller_edge_guesses():
    """ndtctl_ref's identity and ascent guesses (on the golden PCD at resolution 1: ascent and snap rounds) and a guess
    10 km away (zero hits: H = 0, which the fast path refuses)."""
    return X.edge_guesses() + [far_guess()]


def ordinary_guesses(n, seed=0):
    """Small, different perturbations of the identity."""
    import oracle

    rng = np.random.default_rng(seed)
    return [oracle.pose_to_matrix(np.r_[rng.uniform(-0.15, 0.15, 3), rng.uniform(-0.01, 0.01, 3)]).astype(F32)
            for _ in range(n)]


def records(points, stride, seed=0, pinned=False):
    """(n, stride / 4) float32 records with x, y, z first. Every float after them is garbage the solver must not read:
    the 16-byte records carry NaN in the fourth float of every other row and huge or infinite values in the rest,
    wider records random values and NaN. pinned: page-locked memory from torch."""
    p = np.asarray(points, F32)[:, :3]
    n, w = len(p), stride // 4
    assert stride % 4 == 0 and w >= 3
    if pinned:
        import torch

        out = torch.empty((n, w), dtype=torch.float32, pin_memory=True).numpy()
    else:
        out = np.empty((n, w), dtype=F32)
    out[:, :3] = p
    if w > 3:
        rng = np.random.default_rng(seed)
        junk = rng.uniform(-1e30, 1e30, (n, w - 3)).astype(F32)
        junk[::2, 0] = np.nan
        junk[1::4, 0] = np.inf
        if w > 4:
            junk[::3, -1] = np.nan
        out[:, 3:] = junk
    return out


def tile_sizes(ks=(1, 2, 3), big=100_003):
    """Scan sizes on both sides of K12's tile multiples 1024 k, and a scan of about a hundred tiles that ends ragged."""
    return [m for k in ks for m in (SCORE_TILE * k - 1, SCORE_TILE * k, SCORE_TILE * k + 1)] + [big]


def leaf_edge_source(res, seed=0):
    """(source, target): source points exactly on the floats where the builder's floor(x * inv_leaf) and the lookup's
    floor(x / leaf) disagree (x), inside cell 0 on y and z; target voxels in the cells on both sides of every such edge.
    At the identity the transformed point is the source point."""
    import gridref as R

    rng = np.random.default_rng(seed)
    x = R.leaf_edge_floats(res)
    x = x[R.mul_div_disagree(x, res)]
    cells = np.unique(np.concatenate([R.lookup_ref(x, res), R.build_ref(x, res)]))
    cells = np.unique(np.concatenate([cells - 1, cells, cells + 1]))
    tgt = R.cell_points(np.c_[cells, np.zeros((len(cells), 2))], res, 8, rng).astype(F32)
    yz = (rng.uniform(0.15, 0.85, size=(len(x), 2)) * F32(res)).astype(F32)
    return np.c_[x, yz].astype(F32), tgt


def nudged(src, ulps):
    """The source with x moved `ulps` float32 ulp (towards +inf for ulps > 0)."""
    out = np.array(src, dtype=F32)
    for _ in range(abs(ulps)):
        out[:, 0] = np.nextafter(out[:, 0], F32(np.inf if ulps > 0 else -np.inf), dtype=F32)
    return out
