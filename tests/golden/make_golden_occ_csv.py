"""Writes tests/golden/occupancy/occupancy_*.csv: the numpy mirror of the occupancy statistics
(ensemble.occupancy_from_rows) on small seeded inputs — a batch with a bad-status replica and an empty profile, a single
replica that counts, and none — so that a last-bit change in a mean, std, quantile or pooled curve fails a test.

    python tests/golden/make_golden_occ_csv.py
"""
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(os.path.dirname(HERE)))
OUT_DIR = os.path.join(HERE, "occupancy")
DC_NAMES = ["dc-a", "dc-b", "dc-c"]
SUMMARY_K = 24 + 8 * 8
F, B = 8, 128


def _rows(rng, n_dc, R, widths, total):
    """Seeded rows [1 + 8 n_dc + 2 * 128 n_dc, R] that satisfy the recorder's invariants (bins sum to profile_s)."""
    rows = np.zeros((1 + F * n_dc + 2 * B * n_dc, R))
    for r in range(R):
        prof = float(rng.uniform(50.0, 200.0))
        rows[0, r] = prof
        for d in range(n_dc):
            col = lambda f: 1 + f * n_dc + d  # noqa: E731
            q = rng.dirichlet(np.ones(6)) * prof
            qlen = rng.choice(np.arange(B), size=6, replace=False)
            qb = rows[1 + F * n_dc + d * B: 1 + F * n_dc + (d + 1) * B, r]
            np.add.at(qb, qlen, q)
            b = rng.dirichlet(np.ones(5)) * prof
            busy = rng.choice(np.arange(total[d] + 1), size=5, replace=False)
            bb = rows[1 + F * n_dc + (n_dc + d) * B: 1 + F * n_dc + (n_dc + d + 1) * B, r]
            np.add.at(bb, busy // widths[d], b)
            rows[col(0), r] = float(rng.uniform(0, 40)) * prof
            rows[col(1), r] = float(rng.uniform(0, 10)) * prof
            rows[col(2), r] = float(rng.uniform(0, total[d])) * prof
            rows[col(3), r] = float(rng.integers(0, 300))
            rows[col(4), r] = float(rng.integers(0, 90))
            rows[col(5), r] = float(q[qlen > 0].sum())
            rows[col(6), r] = float(b[busy == total[d]].sum())
            rows[col(7), r] = float(b[busy == 0].sum())
    return rows


def cases():
    """name -> (rows, summary, widths)."""
    rng = np.random.default_rng(20261016)
    out = {}
    widths, total = [1, 2, 1], [12, 200, 5]
    rows = _rows(rng, 3, 9, widths, total)
    summ = np.zeros((9, SUMMARY_K))
    summ[4, 0] = 1.0                                   # a replica with a bad status
    rows[:, 7] = 0.0                                   # and one whose run ended before its first event
    out["mixed"] = (rows, summ, widths)
    one = np.ones((9, SUMMARY_K))
    one[2, 0] = 0.0                                    # a single replica counts
    out["one_replica"] = (rows, one, widths)
    out["no_replica"] = (rows, np.ones((9, SUMMARY_K)), widths)   # none does
    return out


def main():
    from distributed_cluster_gpus_b200 import ensemble as EN
    os.makedirs(OUT_DIR, exist_ok=True)
    for name, (rows, summ, widths) in cases().items():
        EN.occupancy_from_rows(rows, summ, widths).to_csv(os.path.join(OUT_DIR, f"occupancy_{name}.csv"),
                                                          DC_NAMES[:len(widths)])


if __name__ == "__main__":
    main()
