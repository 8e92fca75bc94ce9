"""The on-disk form of a mapping session on the CPU: csrc/session_io.hpp compiled with g++ -ffp-contract=off
(tests/hostmath/session_io_host.cpp) against the Python restatement tests/sessionioref.py. The manifest and the g2o text
byte for byte for random sessions (one and several segments, no and many loop edges, with and without adjusted poses); the
parse of what was written bitwise over random bit patterns with -0.0, subnormals and the largest finite values; every kind
of malformed manifest refused with its line named; the g2o edges against pg::build_edges for merged segment layouts; and
the restatement told apart from its named mutations."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

import posegraphref as PG
import sessionioref as R
from oracle.scanmatcher import pose_matrix

HERE = os.path.dirname(os.path.abspath(__file__))
SRC = os.path.join(HERE, "hostmath", "session_io_host.cpp")
SC = (20, 60, 80.0, 2.0)


@pytest.fixture(scope="module")
def sioh(tmp_path_factory):
    lib = os.path.join(tmp_path_factory.mktemp("sioh"), "libsession_io_host.so")
    subprocess.check_call(["g++", "-O2", "-std=c++17", "-ffp-contract=off", "-fPIC", "-shared", "-x", "c++", SRC, "-o", lib])
    lib = C.CDLL(lib)
    vp, i, sz = C.c_void_p, C.c_int, C.c_size_t
    lib.sioh_write.argtypes = [i, vp, vp, i, i, vp, vp, vp, vp, i, i, vp, vp, vp, vp, sz]
    lib.sioh_write.restype = sz
    lib.sioh_parse.argtypes = [C.c_char_p, sz, vp, C.c_char_p, sz]
    lib.sioh_parsed.argtypes = [vp] * 9
    lib.sioh_edges.argtypes = [i, vp, i, i, vp, i, vp, vp, vp, vp, vp, vp, C.POINTER(i)]
    return lib


def _p(a):
    return None if a is None else a.ctypes.data


def _rand_pose(rng, span=50.0):
    q = rng.normal(size=4)
    return pose_matrix(rng.uniform(-span, span, 3), q / np.linalg.norm(q))


def _session(rng, n, seg_first, n_loops, adjusted, k=5):
    poses = [_rand_pose(rng) for _ in range(n)]
    loops = []
    for _ in range(n_loops):
        f, t = rng.choice(n, 2, replace=False)
        loops.append((int(f), int(t), _rand_pose(rng, 5.0)))
    return dict(sc=SC, seg_first=list(seg_first), points=rng.integers(0, 70000, n).tolist(), distances=rng.uniform(0, 500, n).tolist(),
                poses=poses, k=k, loops=loops, adjusted=[_rand_pose(rng) for _ in range(n)] if adjusted else None)


def _arrays(S):
    n = len(S["points"])
    col = lambda Ps: np.ascontiguousarray(np.array([np.asarray(P, dtype=np.float64).T.reshape(16) for P in Ps]).reshape(-1))  # noqa: E731
    L = len(S["loops"])
    return dict(
        sc_rs=np.array(S["sc"][:2], dtype=np.int32), sc_rh=np.array(S["sc"][2:], dtype=np.float64), n=n, m=len(S["seg_first"]),
        seg=np.array(S["seg_first"], dtype=np.int32), points=np.array(S["points"], dtype=np.uint64),
        dist=np.array(S["distances"], dtype=np.float64), pose=col(S["poses"]), k=int(S["k"]), L=L,
        loop_ft=np.array([(f, t) for f, t, _ in S["loops"]] or [(0, 0)], dtype=np.int32).reshape(-1),
        loop_rel=col([Z for _, _, Z in S["loops"]]) if L else np.zeros(16), adjusted=col(S["adjusted"]) if S["adjusted"] is not None else None)


def host_write(sioh, S, which):
    a = _arrays(S)
    args = [which, _p(a["sc_rs"]), _p(a["sc_rh"]), a["n"], a["m"], _p(a["seg"]), _p(a["points"]), _p(a["dist"]), _p(a["pose"]), a["k"],
            a["L"], _p(a["loop_ft"]), _p(a["loop_rel"]), _p(a["adjusted"])]
    size = sioh.sioh_write(*args, None, 0)
    buf = C.create_string_buffer(size + 1)
    sioh.sioh_write(*args, buf, size)
    return buf.raw[:size].decode()


def host_parse(sioh, text):
    """(True, dict of the parsed values) or (False, message)"""
    raw = text.encode() if isinstance(text, str) else text
    counts = np.zeros(6, dtype=np.int64)
    err = C.create_string_buffer(512)
    if not sioh.sioh_parse(raw, len(raw), _p(counts), err, 512):
        return False, err.value.decode()
    n, m, k, L, adj = (int(v) for v in counts[:5])
    out = dict(sc_rs=np.zeros(2, np.int32), sc_rh=np.zeros(2), seg=np.zeros(m, np.int32), points=np.zeros(n, np.uint64),
               dist=np.zeros(n), pose=np.zeros(16 * n), loop_ft=np.zeros(max(1, 2 * L), np.int32), loop_rel=np.zeros(max(1, 16 * L)),
               adjusted=np.zeros(16 * n) if adj else None)
    sioh.sioh_parsed(*(_p(out[key]) for key in ("sc_rs", "sc_rh", "seg", "points", "dist", "pose", "loop_ft", "loop_rel", "adjusted")))
    out.update(n=n, m=m, k=k, L=L)
    out["loop_ft"], out["loop_rel"] = out["loop_ft"][:2 * L], out["loop_rel"][:16 * L]
    return True, out


CASES = [  # (n, seg_first, loops, adjusted)
    (1, [0], 0, False),
    (7, [0], 0, True),
    (30, [0], 12, False),
    (30, [0], 12, True),
    (40, [0, 13, 14, 27], 0, True),
    (40, [0, 13, 14, 27], 25, False),
    (9, [0, 3, 6], 4, True),
]


@pytest.mark.parametrize("case", range(len(CASES)))
def test_manifest_and_g2o_are_the_restatements_bytes(sioh, case):
    n, segs, L, adj = CASES[case]
    rng = np.random.default_rng(100 + case)
    S = _session(rng, n, segs, L, adj, k=int(rng.integers(1, 6)))
    assert host_write(sioh, S, 0) == R.write_manifest(**S)
    g2o = R.write_g2o(S["poses"], S["k"], S["seg_first"], S["loops"], S["adjusted"])
    assert host_write(sioh, S, 1) == g2o
    lines = g2o.split("\n")[:-1]
    assert lines[0].startswith("VERTEX_SE3:QUAT 0 ") and lines[1] == "FIX 0" and all(l.endswith(" ") for l in lines if l != "FIX 0")
    assert sum(l.startswith("VERTEX_SE3:QUAT ") for l in lines) == n
    assert all(len(l.split()) == 31 for l in lines if l.startswith("EDGE_SE3:QUAT "))


@pytest.mark.parametrize("n", [0, 1, 17, 32768, 4194305])
def test_submap_header_is_pcl_binary(sioh, n):
    S = _session(np.random.default_rng(1), 1, [0], 0, False)
    S["points"] = [n]
    assert host_write(sioh, S, 2) == R.pcd_binary_header(n)
    assert R.pcd_binary_header(n).endswith(f"WIDTH {n}\nHEIGHT 1\nVIEWPOINT 0 0 0 1 0 0 0\nPOINTS {n}\nDATA binary\n")


def _special(rng, count):
    """random finite doubles from raw bit patterns, with -0.0, subnormals and +-max mixed in"""
    bits = rng.integers(0, 2 ** 64, count, dtype=np.uint64)
    v = bits.view(np.float64).copy()
    v[~np.isfinite(v)] = 1.5
    special = np.array([-0.0, 0.0, 5e-324, -5e-324, 2.2250738585072009e-308, np.finfo(np.float64).max, -np.finfo(np.float64).max,
                        np.finfo(np.float64).tiny, 1.0 / 3.0, -1e-310])
    v[: len(special)] = special
    return rng.permutation(v)


@pytest.mark.parametrize("adjusted", [False, True])
def test_parse_returns_every_number_bitwise(sioh, adjusted):
    rng = np.random.default_rng(7 + adjusted)
    n, L = 12, 5
    S = _session(rng, n, [0, 4, 9], L, adjusted)
    vals = _special(rng, 16 * n * 2 + 16 * L + n + 2)
    it = iter(vals)
    S["poses"] = [np.array([next(it) for _ in range(16)]).reshape(4, 4) for _ in range(n)]
    S["distances"] = [next(it) for _ in range(n)]
    S["loops"] = [(f, t, np.array([next(it) for _ in range(16)]).reshape(4, 4)) for f, t, _ in S["loops"]]
    if adjusted:
        S["adjusted"] = [np.array([next(it) for _ in range(16)]).reshape(4, 4) for _ in range(n)]
    S["sc"] = (20, 60, 5e-324, -0.0)  # max_radius > 0 (a subnormal), lidar_height -0.0
    text = host_write(sioh, S, 0)
    assert text == R.write_manifest(**S)
    ok, got = host_parse(sioh, text)
    assert ok, got
    a = _arrays(S)
    for key in ("sc_rs", "seg", "points", "loop_ft"):
        assert np.array_equal(got[key], a[key][: got[key].size]), key
    for key in ("sc_rh", "dist", "pose", "loop_rel") + (("adjusted",) if adjusted else ()):
        assert got[key].view(np.uint64).tolist() == a[key].view(np.uint64).tolist(), key
    assert (got["adjusted"] is None) == (not adjusted) and got["k"] == S["k"] and got["n"] == n and got["L"] == L
    ok, msg = host_parse(sioh, R.write_manifest(**S, mutations=("precision16",)))
    assert not ok or any(got2.view(np.uint64).tolist() != a2.view(np.uint64).tolist()
                         for got2, a2 in [(msg[k2], a[k2]) for k2 in ("dist", "pose")])


def _good():
    S = _session(np.random.default_rng(3), 6, [0, 3], 2, True, k=2)
    return R.write_manifest(**S).split("\n")[:-1]


def _with(lines, at, new):
    out = list(lines)
    if new is None:
        del out[at]
    else:
        out[at] = new
    return out


def _tok(lines, at, index, value):
    t = lines[at].split(" ")
    t[index] = value
    return _with(lines, at, " ".join(t))


# (name, corrupt(lines) -> lines, the 1-based line the error names). Layout of _good(): 1 version, 2 scan_context, 3 submaps,
# 4 segments, 5-10 submap, 11 odometry, 12 loops, 13-14 loop, 15 adjusted, 16-21 pose.
MALFORMED = [
    ("keyword", lambda L: _tok(L, 0, 0, "b200sm_sessions"), 1),
    ("version", lambda L: _tok(L, 0, 1, "2"), 1),
    ("sc_count", lambda L: _tok(L, 1, 1, "0"), 2),
    ("sc_nonfinite", lambda L: _tok(L, 1, 3, "inf"), 2),
    ("submaps_count", lambda L: _tok(L, 2, 1, "7"), 11),
    ("submaps_zero", lambda L: _tok(L, 2, 1, "0"), 3),
    ("segments_count", lambda L: _tok(L, 3, 1, "3"), 4),
    ("segments_not_at_0", lambda L: _with(L, 3, "segments 2 1 3"), 4),
    ("segments_not_increasing", lambda L: _with(L, 3, "segments 3 0 3 3"), 4),
    ("segments_past_n", lambda L: _with(L, 3, "segments 2 0 6"), 4),
    ("submap_index", lambda L: _tok(L, 5, 1, "2"), 6),
    ("submap_points", lambda L: _tok(L, 5, 2, "-1"), 6),
    ("token_not_whole", lambda L: _tok(L, 6, 7, "1.5x"), 7),
    ("token_nan", lambda L: _tok(L, 7, 9, "nan"), 8),
    ("token_inf", lambda L: _tok(L, 8, 3, "-inf"), 9),
    ("token_overflow", lambda L: _tok(L, 8, 4, "1e309"), 9),
    ("token_missing", lambda L: _with(L, 9, " ".join(L[9].split(" ")[:-1])), 10),
    ("double_space", lambda L: _with(L, 9, L[9].replace(" ", "  ", 1)), 10),
    ("odometry_zero", lambda L: _tok(L, 10, 1, "0"), 11),
    ("loops_count", lambda L: _tok(L, 11, 1, "3"), 15),
    ("loop_out_of_range", lambda L: _tok(L, 12, 2, "6"), 13),
    ("loop_negative", lambda L: _tok(L, 12, 1, "-1"), 13),
    ("loop_self", lambda L: _tok(_tok(L, 13, 1, "4"), 13, 2, "4"), 14),
    ("adjusted_value", lambda L: _tok(L, 14, 1, "2"), 15),
    ("pose_index", lambda L: _tok(L, 16, 1, "0"), 17),
    ("missing_line", lambda L: L[:-1], 21),
    ("extra_line", lambda L: L + ["pose 6 " + " ".join(["0"] * 16)], 22),
    ("adjusted_0_with_poses", lambda L: _tok(L, 14, 1, "0"), 16),
    ("no_final_newline", None, 21),
]


@pytest.mark.parametrize("kind", [m[0] for m in MALFORMED])
def test_malformed_manifest_names_its_line(sioh, kind):
    name, corrupt, line = next(m for m in MALFORMED if m[0] == kind)
    good = _good()
    assert host_parse(sioh, "".join(l + "\n" for l in good))[0]
    text = "".join(l + "\n" for l in good)[:-1] if corrupt is None else "".join(l + "\n" for l in corrupt(good))
    ok, msg = host_parse(sioh, text)
    assert not ok and msg.startswith(f"line {line}:"), (kind, msg)


@pytest.mark.parametrize("segs", [[0], [0, 10], [0, 1, 2, 20], [0, 6, 7, 8, 30]])
def test_g2o_edges_are_build_edges(sioh, segs):
    rng = np.random.default_rng(len(segs))
    S = _session(rng, 36, segs, 9, False, k=3)
    a = _arrays(S)
    E = 36 * 3 + 9
    ft_io, ft_pg = np.zeros(2 * E, np.int32), np.zeros(2 * E, np.int32)
    Z, Zinv = np.zeros(12 * E), np.zeros(12 * E)
    n_pg = C.c_int(0)
    n_io = sioh.sioh_edges(36, _p(a["pose"]), 3, a["m"], _p(a["seg"]), a["L"], _p(a["loop_ft"]), _p(a["loop_rel"]), _p(ft_io), _p(ft_pg),
                           _p(Z), _p(Zinv), C.byref(n_pg))
    assert n_io == n_pg.value and np.array_equal(ft_io[:2 * n_io], ft_pg[:2 * n_io])
    ref = R.graph_edges(S["poses"], 3, segs, S["loops"])
    assert [(f, t) for f, t, _ in ref] == [tuple(ft_io[2 * e:2 * e + 2]) for e in range(n_io)]
    for e in range(n_io):
        Ze = np.eye(4)
        Ze[:3] = Z[12 * e:12 * e + 12].reshape(3, 4)
        assert np.array_equal(Ze, ref[e][2]), e
        if e < n_io - len(S["loops"]):  # an odometry edge: build_edges keeps exactly the inverse of the measurement
            assert np.array_equal(PG.inverse(Ze)[:3].reshape(12), Zinv[12 * e:12 * e + 12]), e


def test_each_mutation_changes_an_outcome(sioh):
    rng = np.random.default_rng(29)
    S = _session(rng, 20, [0, 8], 3, True, k=2)
    S["distances"][0] = 0.1 + 0.2  # needs 17 significant digits
    caught = set()
    good_m, good_g = R.write_manifest(**S), R.write_g2o(S["poses"], S["k"], S["seg_first"], S["loops"], S["adjusted"])
    assert good_m == host_write(sioh, S, 0) and good_g == host_write(sioh, S, 1)
    for mut in R.MUTATIONS:
        m = R.write_manifest(**S, mutations=(mut,))
        g = R.write_g2o(S["poses"], S["k"], S["seg_first"], S["loops"], S["adjusted"], mutations=(mut,))
        if m != good_m or g != good_g:
            caught.add(mut)
    assert caught == set(R.MUTATIONS), set(R.MUTATIONS) - caught
    ok, got = host_parse(sioh, R.write_manifest(**S, mutations=("precision16",)))
    assert ok and got["dist"][0] != S["distances"][0]
