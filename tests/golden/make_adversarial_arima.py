#!/usr/bin/env python3
"""Generate tests/golden/adversarial_arima_series.json: the connections of tests/adversarial.arima_collision_table() for
which the ARIMA oracle (oracle/arima_oracle.calculate_arima) returns scores -- the series an ARIMA job keeps.  The Python
oracle takes about two seconds per series, too slow to run inside the GPU test, so its verdicts are committed here.

    python tests/golden/make_adversarial_arima.py [processes]
"""
import json
import os
import sys
from multiprocessing import Pool

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.join(HERE, "..", ".."))
from oracle import arima_oracle as ao, tad_oracle as o  # noqa: E402
from tests import adversarial as A  # noqa: E402

OUT = os.path.join(HERE, "adversarial_arima_series.json")


def kept(values):
    return ao.calculate_arima(np.asarray(values, dtype=np.uint64)) is not None


def main():
    t, _ = A.arima_collision_table()
    # stage A and B of the oracle: every series' reduced values in time order
    res = o.run_job(t, o.JobSpec(algo=o.ALGO_EWMA, emit_all=True))
    c = res.cols
    keys = np.stack([c[k].astype(np.int64) for k in o.KEY_COLUMNS], 1)
    _, first, inv = np.unique(keys, axis=0, return_index=True, return_inverse=True)
    inv = inv.ravel()
    series = [c["throughput"][inv == s].astype(np.uint64) for s in range(len(first))]
    with Pool(int(sys.argv[1]) if len(sys.argv) > 1 else os.cpu_count()) as p:
        ok = p.map(kept, series, chunksize=4)
    out = {
        "table": "tests/adversarial.py: arima_collision_table()",
        "sha256": A.table_digest(t),
        "key_columns": list(o.KEY_COLUMNS),
        "series": len(series),
        "kept": sorted(keys[first[s]].tolist() for s in range(len(series)) if ok[s]),
    }
    with open(OUT, "w") as f:
        json.dump(out, f, separators=(",", ":"))
        f.write("\n")
    print("%d of %d series kept -> %s" % (len(out["kept"]), len(series), OUT))


if __name__ == "__main__":
    main()
