"""The columnar oracle (oracle/columnar_oracle.py) equals the C oracle bit for bit on every adversarial table, the
golden e2e table and ragged make_flows tables with duplicates and values up to 2^64 -- both reducers, both values of
emit_all, time filters that cut series in the middle -- and each of its rules is needed: a mutant that changes one rule
differs from the C oracle on at least one of these tables.  No GPU needed."""
import functools
import json
import os

import numpy as np
import pytest

from oracle import c_oracle
from oracle import columnar_oracle as co
from oracle import tad_oracle
from tests import adversarial as A
from theia_b200 import synth

U64 = np.uint64
EWMA, DBSCAN = co.ALGO_EWMA, co.ALGO_DBSCAN
HERE = os.path.dirname(os.path.abspath(__file__))


def wide_flows(seed):
    """Ragged make_flows series with 10 % duplicates; a third of the connections moved up to values within 1e13 of
    2^64 - 1 and a third scaled by 2^20 (up to about 2^53), so the sum reducer wraps and u64 -> double rounds."""
    t = synth.make_flows(3000, 25, seed=seed, ragged=True, dup_frac=0.1)
    third = t["src_ip"] % np.uint32(3)
    v = t["value"]
    t["value"] = np.where(third == 0, U64((1 << 64) - 1) - v * U64(1000),
                          np.where(third == 1, v << U64(20), v)).astype(U64)
    return t


@functools.lru_cache(maxsize=None)
def table(name):
    """(table, time filters that cut series in the middle)."""
    if name == "golden":
        ref = json.load(open(os.path.join(HERE, "golden", "reference_test_vectors.json")))
        t = synth.golden_e2e_table(ref["throughput_list"], duplicates=2)
    elif name.startswith("flows"):
        t = wide_flows(int(name[5:]))
    else:
        t = {
            "collision": lambda: A.collision_table(seed=1),
            "probe_1024x3": lambda: A.probe_chain_table(1024, 3),
            "probe_4096x1": lambda: A.probe_chain_table(4096, 1),
            "one_bucket": lambda: A.one_bucket_table(n_series=100_000, seed=6),
            "skewed": lambda: A.skewed_residue_table(n_series=50_000, seed=7),
            "lattice": lambda: A.dbscan_lattice_table(seed=2),
            "ewma": lambda: A.ewma_edge_table(seed=3),
            "timestamps": lambda: A.timestamp_table(seed=4),
            "duplicates": lambda: A.duplicate_table(seed=5),
        }[name]()[0]
    fs = np.sort(np.unique(t["flow_start"]))
    fe = np.sort(np.unique(t["flow_end"]))
    return t, (int(fs[len(fs) // 4]), int(fe[len(fe) // 2]))


TABLES = ("collision", "probe_1024x3", "probe_4096x1", "one_bucket", "skewed", "lattice", "ewma", "timestamps",
          "duplicates", "golden", "flows1", "flows2")


def specs(name):
    """(reducer, emit_all, start_time, end_time) of the runs on a table."""
    _, (start, end) = table(name)
    return ((co.REDUCE_MAX, False, 0, 0), (co.REDUCE_MAX, True, 0, 0), (co.REDUCE_SUM, False, 0, 0),
            (co.REDUCE_SUM, True, 0, 0), (co.REDUCE_MAX, True, start, end), (co.REDUCE_SUM, False, 0, end))


@functools.lru_cache(maxsize=None)
def c_rows(name, algo, spec):
    reducer, emit_all, start, end = spec
    cols, ns, npts = c_oracle.run_job(table(name)[0], algo=algo, reducer=reducer, start_time=start, end_time=end,
                                      emit_all=emit_all)
    return tad_oracle.canonicalize(cols), ns, npts


def columnar_rows(name, algo, spec, **kw):
    reducer, emit_all, start, end = spec
    return co.run_job(table(name)[0], algo=algo, reducer=reducer, start_time=start, end_time=end, emit_all=emit_all,
                      **kw)


def same(got, want):
    """Equal counts and every column equal bit for bit (NaN stddev of one-point series included)."""
    (gc, gs, gp), (wc, ws, wp) = got, want
    if (gs, gp) != (ws, wp) or len(gc["flow_end"]) != len(wc["flow_end"]):
        return False
    return all(gc[c].dtype == wc[c].dtype and np.array_equal(gc[c].view(np.uint8), wc[c].view(np.uint8))
               for c in tad_oracle.OUT_COLUMNS)


@pytest.mark.parametrize("algo", [EWMA, DBSCAN])
@pytest.mark.parametrize("name", TABLES)
def test_equals_c_oracle(name, algo):
    n_rows = 0
    for spec in specs(name):
        want = c_rows(name, algo, spec)
        got = columnar_rows(name, algo, spec)
        assert same(got, want), (name, algo, spec)
        n_rows += len(want[0]["flow_end"])
    assert n_rows > 0


def test_filters_cut_series():
    """The end-time filter keeps the first part of series whose last part it drops."""
    t, (start, end) = table("flows1")
    cut = A.n_connections({c: v[t["flow_end"] < end] for c, v in t.items()})
    whole = A.n_connections({c: v[t["flow_end"] >= end] for c, v in t.items()})
    both = A.n_connections(t)
    assert cut + whole - both >= 100                     # connections on both sides of the cut
    _, ns, _ = c_rows("flows1", EWMA, (co.REDUCE_MAX, True, start, end))
    assert 0 < ns < cut


def test_torch_sort_and_pieces_equal_numpy():
    """The order from torch sorts and a table computed in pieces by source address give the same rows."""
    pytest.importorskip("torch")
    for name in ("collision", "lattice", "duplicates", "flows2"):
        for algo in (EWMA, DBSCAN):
            spec = (co.REDUCE_SUM, True, 0, 0)
            want = c_rows(name, algo, spec)
            assert same(columnar_rows(name, algo, spec, sort_device="cpu"), want), name
            rows = len(table(name)[0]["flow_end"])
            assert same(columnar_rows(name, algo, spec, max_chunk_rows=rows // 5 + 1), want), name
            assert same(columnar_rows(name, algo, spec, max_chunk_rows=rows // 5 + 1, workers=3), want), name


@pytest.mark.parametrize("words", [3, 2])
def test_a_wrong_sort_order_is_caught(monkeypatch, words):
    """An order from a sort that got it wrong -- of the rows by key (three words) or of a series' points by value (two
    words) -- stops the oracle instead of giving wrong rows."""
    right = co._argsort_lex

    def wrong(w, sort_device=None):
        o = right(w, sort_device)
        if len(w) == words:
            o[[0, -1]] = o[[-1, 0]]
        return o
    monkeypatch.setattr(co, "_argsort_lex", wrong)
    with pytest.raises(AssertionError, match="out of"):
        columnar_rows("flows1", DBSCAN, (co.REDUCE_MAX, False, 0, 0))


def test_canonicalize_equals_tad_oracle():
    t = table("flows1")[0]
    rng = np.random.default_rng(0)
    want = c_rows("flows1", EWMA, (co.REDUCE_MAX, True, 0, 0))[0]
    perm = rng.permutation(len(want["flow_end"]))
    got = co.canonicalize({c: v[perm] for c, v in want.items()})
    assert all(np.array_equal(got[c], want[c], equal_nan=True) for c in want)
    assert len(t["flow_end"]) > len(want["flow_end"])


# --------------------------------------------------------------------------------------------------------------------
# mutants: one rule changed each
# --------------------------------------------------------------------------------------------------------------------
def flag_ge(x, calc, sd_pt):
    return np.abs(x - calc) >= sd_pt


def two_pass_stddev(x, lens, base, counts):
    s = np.zeros(len(base))
    for i, c in enumerate(counts):
        s[:c] = s[:c] + x[base[:c] + i]
    mean = s / lens
    q = np.zeros(len(base))
    for i, c in enumerate(counts):
        d = x[base[:c] + i] - mean[:c]
        q[:c] = q[:c] + d * d
    with np.errstate(invalid="ignore", divide="ignore"):
        sd = np.sqrt(q / (lens - 1.0))
    sd[lens < 2] = np.nan
    return sd


def plain_distance(xi, xj):
    """|xi - xj| <= eps for n <= 11 as well: 0 inside the window, infinity outside."""
    return np.where(np.abs(xi - xj) <= A.EPS, 0.0, np.inf)


def saturating_sum(values, starts):
    lo = np.add.reduceat(values & U64(0xffffffff), starts)
    hi = np.add.reduceat(values >> U64(32), starts) + (lo >> U64(32))
    full = (hi << U64(32)) | (lo & U64(0xffffffff))
    return np.where(hi >> U64(32) != 0, U64((1 << 64) - 1), full).astype(U64)


MUTANTS = {
    "flag >=": ("ewma_flag", flag_ge, (EWMA,)),
    "two-pass stddev": ("welford", two_pass_stddev, (EWMA, DBSCAN)),
    "|xi - xj| for n <= 11": ("brute_d2", plain_distance, (DBSCAN,)),
    "sum without wrap": ("reduce_sum", saturating_sum, (EWMA, DBSCAN)),
}


@pytest.mark.parametrize("mutant", list(MUTANTS))
def test_every_mutant_is_caught(monkeypatch, mutant):
    attr, fn, algos = MUTANTS[mutant]
    monkeypatch.setattr(co, attr, fn)
    caught = []
    for name in TABLES:
        for algo in algos:
            for spec in specs(name):
                if not same(columnar_rows(name, algo, spec), c_rows(name, algo, spec)):
                    caught.append((name, algo, spec))
    assert caught, "mutant %r agrees with the C oracle on every table" % mutant
