"""Host mirror of the hash-range passes (sharding.pass_of): which rows a single-GPU job larger than its memory budget
runs together.  No GPU needed."""
import numpy as np
import pytest

from theia_b200 import sharding, synth


def _conn_ids(t):
    key = np.stack([t[c].astype(np.uint64) for c in ("src_ip", "dst_ip", "src_port", "dst_port", "proto", "flow_start")], 1)
    _, inv = np.unique(key, axis=0, return_inverse=True)
    return inv.ravel()


@pytest.mark.parametrize("passes", [1, 2, 4, 8, 64])
def test_every_connection_in_exactly_one_pass(passes):
    t = synth.make_flows(3000, 20, seed=1, dup_frac=0.1, ragged=True)
    p = sharding.pass_of(t, passes)
    assert p.min() >= 0 and p.max() < passes
    conn = _conn_ids(t)
    per_conn = np.full(conn.max() + 1, -1)
    per_conn[conn] = p
    assert np.array_equal(per_conn[conn], p)          # all rows of a connection share its pass
    assert np.bincount(p, minlength=passes).sum() == len(p)


def test_passes_split_by_the_next_hash_bit():
    """Pass v of P splits into passes v and v + P of 2P: a pass that does not fit is halved without re-planning the rest."""
    t = synth.make_flows(2000, 5, seed=2)
    for P in (1, 2, 4, 8, 16, 32):
        assert np.array_equal(sharding.pass_of(t, 2 * P) % P, sharding.pass_of(t, P))


@pytest.mark.parametrize("passes", [2, 8, 64])
def test_passes_are_balanced(passes):
    n_series = 64000
    t = synth.make_flows(n_series, 1, seed=3)            # one row per connection
    counts = np.bincount(sharding.pass_of(t, passes), minlength=passes)
    mean = n_series / passes
    assert np.all(np.abs(counts - mean) <= 5 * np.sqrt(mean)), counts      # binomial spread, 5 sigma


def test_pass_rows_cover_all_buckets_of_their_own_size():
    """The pass bits are the low hash bits; the bucket bits (top) of a pass's rows stay uniform, so a pass of n rows
    occupies every bucket of pick_logb(n) (mean 384..768 rows per bucket)."""
    t = synth.make_flows(40000, 50, seed=4)
    h = sharding.key_hash(t)
    for P in (2, 4, 8):
        p = sharding.pass_of(t, P)
        for v in range(P):
            hv = h[p == v]
            logb = sharding.pick_logb(len(hv))
            buckets = np.bincount((hv >> np.uint64(64 - logb)).astype(np.int64), minlength=1 << logb)
            assert len(buckets) == 1 << logb and buckets.min() > 0
            # and the 24-bit hash tag below the bucket bits is not biased by the pass either
            tag = (hv >> np.uint64(64 - logb - 24)) & np.uint64(0xffffff)
            assert 0.45 < float(np.mean(tag >= np.uint64(1 << 23))) < 0.55


def test_pass_of_rejects_bad_counts():
    t = synth.make_flows(10, 2, seed=5)
    for bad in (0, 3, 128):
        with pytest.raises(AssertionError):
            sharding.pass_of(t, bad)
