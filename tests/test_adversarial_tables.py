"""The adversarial table generators (tests/adversarial.py) reach what they are built for under the host mirror of the
key hash, the C oracle equals the Python oracle on them, and the DBSCAN rule the oracle and the kernels share agrees
with sklearn's algorithm written out literally.  No GPU needed."""
import functools

import numpy as np
import pytest

from oracle import c_oracle, tad_oracle as o
from tests import adversarial as A
from theia_b200 import sharding

U64 = np.uint64


@functools.lru_cache(maxsize=None)
def table(name):
    return {
        "collision": lambda: A.collision_table(seed=1),
        "probe_1024x3": lambda: A.probe_chain_table(1024, 3),
        "probe_4096x1": lambda: A.probe_chain_table(4096, 1),
        "lattice": lambda: A.dbscan_lattice_table(seed=2),
        "ewma": lambda: A.ewma_edge_table(seed=3),
        "timestamps": lambda: A.timestamp_table(seed=4),
        "duplicates": lambda: A.duplicate_table(seed=5),
    }[name]()


def test_inverse_hash_reaches_any_target():
    rng = np.random.default_rng(0)
    h = A.compose_hash(rng, 4096)
    assert np.array_equal(sharding.mix64(A.inv_mix64(h)), h)
    for proto in (0, 6, 17, 255):
        fs, sp, dp = A._random_b(rng, len(h))
        si, di = A.key_for_hash(h, A.key_b(fs, sp, dp), np.full(len(h), proto))
        t = {"src_ip": si, "dst_ip": di, "src_port": sp, "dst_port": dp, "flow_start": fs,
             "proto": np.full(len(h), proto, np.uint8), "flow_end": fs}
        assert np.array_equal(sharding.key_hash(t), h)
    # one target, four keys that differ in proto, flow_start or a port
    target = np.full(4, 0xdeadbeef12345678, U64)
    fs = np.array([100, 100, 101, 100], np.uint32)
    sp = np.array([1, 1, 1, 2], np.uint16)
    pr = np.array([6, 17, 6, 6], np.uint8)
    si, di = A.key_for_hash(target, A.key_b(fs, sp, np.zeros(4, np.uint16)), pr)
    t = {"src_ip": si, "dst_ip": di, "src_port": sp, "dst_port": np.zeros(4, np.uint16), "flow_start": fs, "proto": pr,
         "flow_end": fs}
    assert np.all(sharding.key_hash(t) == target) and A.n_connections(t) == 4


def test_collision_groups_and_twins():
    t, info = table("collision")
    for g in info["groups"]:
        gt = dict(g, flow_end=g["flow_start"])
        h = sharding.key_hash(gt)
        assert len(set(h.tolist())) == 1 and A.n_connections(gt) == len(h) >= 2
        present = {tuple(int(g[c][i]) for c in o.KEY_COLUMNS) for i in range(len(h))}
        rows = {tuple(int(t[c][i]) for c in o.KEY_COLUMNS) for i in np.flatnonzero(np.isin(t["src_ip"], g["src_ip"]))}
        assert present <= rows
    h = sharding.key_hash(t)
    for lo, hi in info["twins"]:
        assert lo != hi and lo >> (64 - A.TWIN_BITS) == hi >> (64 - A.TWIN_BITS)
        assert np.any(h == U64(lo)) and np.any(h == U64(hi))
        assert not np.any((h > U64(lo)) & (h < U64(hi))), "a hash between the twins: they are not neighbours"
        twin = (h == U64(lo)) | (h == U64(hi))
        for c in ("src_ip", "dst_ip", "src_port", "dst_port", "flow_start"):
            assert len(np.unique(t[c][twin])) == 1, c           # the twins differ in proto alone
        assert len(np.unique(t["proto"][twin])) == 2
    # the long twins overfill their bucket at every logB up to the one the table picks
    lo, hi = info["twins"][0]
    for logb in (1, 4, sharding.pick_logb(len(h))):
        b = A.bucket_of(U64(lo), logb)
        assert np.sum(A.bucket_of(h, logb) == b) > 4096
    assert info["series"] == o.run_job(t, o.JobSpec()).n_series


@pytest.mark.parametrize("points", [1, 3])
@pytest.mark.parametrize("cap", A.CLASS_CAPS)
def test_probe_chain_targets(cap, points):
    t, info = A.probe_chain_table(cap, points)
    h = sharding.key_hash(t)
    b = A.bucket_of(h, info["logb"])
    hist = np.bincount(b, minlength=16)
    assert hist[info["bucket"]] == cap and hist.max() == cap, hist
    mine = b == info["bucket"]
    assert np.all(A.start_slot(h[mine], info["logb"], cap) == 3 * cap // 2 - 1)
    assert A.n_connections({c: v[mine] for c, v in t.items()}) == info["series"]
    # distinct connections with one tag and one protocol byte: the full-key compare alone separates them
    word = (A.hash_tag(h[mine], info["logb"]) << 8) | t["proto"][mine].astype(np.int64)
    _, counts = np.unique(word, return_counts=True)
    assert counts.max() >= cap // points // 5


def test_one_bucket_overfills_the_overflow_list():
    t, info = A.one_bucket_table()
    n = len(t["value"])
    assert n == info["rows"] == 1_200_000
    h = sharding.key_hash(t)
    for logb in (1, 4, sharding.pick_logb(n), 22):
        assert len(np.unique(A.bucket_of(h, logb))) == 1
    overflow = n - 4096                            # the bucket's slot keeps 4096 rows
    assert overflow > max(1 << 20, n // 32)
    assert len(np.unique(h)) == info["series"]


def test_skewed_residues():
    t, info = A.skewed_residue_table()
    res = sharding.pass_of(t, 64)
    counts = np.bincount(res, minlength=64)
    assert counts.argmax() == info["residue"] and counts.max() == info["heavy_rows"]
    assert 0.77 < info["heavy_rows"] / info["rows"] < 0.83
    for P in (2, 4, 8, 64):          # halving the passes never splits the heavy residue
        largest = np.bincount(sharding.pass_of(t, P), minlength=P).max()
        assert largest >= info["heavy_rows"]


@pytest.mark.parametrize("name", ["ewma", "duplicates"])
def test_connections_alone_in_their_buckets(name):
    t, info = table(name)
    h = sharding.key_hash(t)
    logb = sharding.pick_logb(len(h))
    assert logb >= 5
    conn_per_bucket = {}
    for bkt, hv in zip(A.bucket_of(h, logb).tolist(), h.tolist()):
        conn_per_bucket.setdefault(bkt, set()).add(hv)
    assert all(len(s) == 1 for s in conn_per_bucket.values())
    assert len(conn_per_bucket) == info["series"] == A.n_connections(t)


def test_timestamp_edges():
    t, info = table("timestamps")
    fe = t["flow_end"].astype(np.int64)
    assert fe.min() == 0 and fe.max() == (1 << 32) - 1
    assert np.all(np.diff(fe) <= 0)                               # rows in descending time order
    assert np.any(t["flow_start"] == info["start_time"]) and np.any(t["flow_end"] == info["end_time"])
    res = o.run_job(t, o.JobSpec(start_time=info["start_time"], end_time=info["end_time"], emit_all=True))
    assert np.any(res.cols["flow_start"] == info["start_time"])    # kept: flow_start >= start
    assert not np.any(res.cols["flow_end"] >= info["end_time"])     # dropped: flow_end < end
    # a burst: most of one series inside 3 s, one row far away
    key = t["src_ip"].astype(np.int64) << 32 | t["dst_ip"].astype(np.int64)
    spans = [np.ptp(np.sort(fe[key == k])[:-1]) for k in np.unique(key)]
    assert sum(s <= 3 for s in spans) >= 8


def test_duplicate_sums_wrap():
    t, _ = table("duplicates")
    res = o.run_job(t, o.JobSpec(reducer=o.REDUCE_SUM, emit_all=True))
    exact = {}
    for i in range(len(t["value"])):
        k = (int(t["src_ip"][i]), int(t["dst_ip"][i]), int(t["flow_end"][i]))
        exact[k] = exact.get(k, 0) + int(t["value"][i])
    assert max(exact.values()) >= 1 << 64                       # the sum wraps
    assert res.n_points == len(exact)


# --------------------------------------------------------------------------------------------------------------------
# the C oracle equals the Python oracle
# --------------------------------------------------------------------------------------------------------------------
def _compare_oracles(t, spec):
    pr = o.run_job(t, spec)
    cc, ns, npts = c_oracle.run_job(t, algo=spec.algo, reducer=spec.reducer, start_time=spec.start_time,
                                    end_time=spec.end_time, emit_all=spec.emit_all, threads=4)
    cc = o.canonicalize(cc)
    assert ns == pr.n_series and npts == pr.n_points
    for k in pr.cols:
        assert np.array_equal(pr.cols[k], cc[k], equal_nan=True), k
    return pr


@pytest.mark.parametrize("algo", [o.ALGO_EWMA, o.ALGO_DBSCAN])
@pytest.mark.parametrize("name", ["collision", "probe_1024x3", "probe_4096x1", "lattice", "ewma", "timestamps",
                                  "duplicates"])
def test_c_oracle_equals_python(name, algo):
    t, info = table(name)
    for emit_all in (False, True):
        _compare_oracles(t, o.JobSpec(algo=algo, emit_all=emit_all))
    if name in ("timestamps", "duplicates"):
        _compare_oracles(t, o.JobSpec(algo=algo, reducer=o.REDUCE_SUM, emit_all=True))
    if name == "timestamps":
        _compare_oracles(t, o.JobSpec(algo=algo, start_time=info["start_time"], end_time=info["end_time"], emit_all=True))


# --------------------------------------------------------------------------------------------------------------------
# DBSCAN: sklearn's algorithm, literally
# --------------------------------------------------------------------------------------------------------------------
def sklearn_dbscan_noise(values, strict=False, expansion=None):
    """DBSCAN(eps=2.5e8, min_samples=4) on 1-D values as sklearn 1.3 runs it: float64 neighbourhoods (for n <= 11 the
    brute-force ``x^2 - 2xy + y^2`` distance against eps^2, the point itself always included; otherwise
    ``|xi - xj| <= eps``), core points with at least 4 neighbours counting themselves, clusters grown breadth-first from
    core points, noise = the points no cluster takes.  ``strict`` and ``expansion`` change one rule each."""
    x = np.asarray(values, dtype=U64).astype(np.float64)
    n = len(x)
    brute = n <= 11 if expansion is None else expansion
    eps = A.EPS * 1.0
    nbrs = []
    for i in range(n):
        if brute:
            d2 = (x[i] * x[i] + (-2.0 * (x[i] * x))) + x * x
            d2 = np.where(d2 > 0.0, d2, 0.0)
            nb = d2 < eps * eps if strict else d2 <= eps * eps
        else:
            d = np.abs(x[i] - x)
            nb = d < eps if strict else d <= eps
        nb[i] = True
        nbrs.append(np.flatnonzero(nb))
    core = np.array([len(nb) >= 4 for nb in nbrs], dtype=bool)
    label = np.full(n, -1)
    c = 0
    for i in range(n):
        if label[i] != -1 or not core[i]:
            continue
        label[i] = c
        queue = [i]
        while queue:
            p = queue.pop()
            for q in nbrs[p]:
                if label[q] == -1:
                    label[q] = c
                    if core[q]:
                        queue.append(q)
        c += 1
    return label == -1


def test_dbscan_rule_equals_sklearns_algorithm():
    _, info = table("lattice")
    differs_strict = differs_brute = differs_sweep = border = 0
    for v in info["values"]:
        want = sklearn_dbscan_noise(v)
        got = o.calculate_dbscan_anomaly(v)
        assert np.array_equal(got, want), len(v)
        assert np.array_equal(c_oracle.dbscan_series(v), want), len(v)
        differs_strict += not np.array_equal(sklearn_dbscan_noise(v, strict=True), want)
        if len(v) <= 11:
            differs_brute += not np.array_equal(sklearn_dbscan_noise(v, expansion=False), want)
        else:
            differs_sweep += not np.array_equal(sklearn_dbscan_noise(v, expansion=True), want)
        x = v.astype(np.float64)
        nb = np.abs(x[:, None] - x[None, :]) <= A.EPS if len(v) <= 600 else None
        if nb is not None:
            core = nb.sum(1) >= 4
            border += int(np.sum(~core & (nb & core[None, :]).any(1)))
    # the lattice decides on the edges: an eps tie, the brute-force expansion, border points
    assert differs_strict >= 20 and differs_brute >= 10 and border >= 100, (differs_strict, differs_brute, border)


def test_ewma_edges_decide_on_the_strict_compare():
    _, info = table("ewma")
    decided = 0
    for v in info["values"]:
        calc, flag, sd = c_oracle.ewma_series(v)
        if len(v) < 2:
            continue
        x = v.astype(np.float64)
        decided += int(np.sum(np.abs(x - calc) == sd))
        assert np.array_equal(flag, o.calculate_ewma_anomaly(v, o.stddev_samp(v)))
    assert decided >= 4 * 4095, decided


def test_arima_fixture_is_for_this_table():
    """tests/golden/adversarial_arima_series.json holds the ARIMA oracle's verdicts on arima_collision_table(): the
    fixture must be regenerated (tests/golden/make_adversarial_arima.py) whenever the table changes."""
    import json
    import os
    golden = json.load(open(os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden",
                                         "adversarial_arima_series.json")))
    t, info = A.arima_collision_table()
    assert golden["sha256"] == A.table_digest(t)
    assert golden["series"] == info["series"] and 100 <= len(golden["kept"]) < info["series"]
