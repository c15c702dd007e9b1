"""TEST-ONLY driver of the CUDA library built with -DDCSIM_TEST_HOOKS (tests/gpuhooks/_build, see __graft_entry__.build).

That build rounds every arrival and xfer_done instant up to a multiple of a time quantum on the device, like the
oracle's and the host build's hook, so that same-instant events become common.  It is loaded in a process of its own
(DCSIM_B200_LIB names it) so the test process keeps the product library.

    DCSIM_B200_LIB=<hook lib> python tests/gpuhooks/driver.py jobs.json out_dir

jobs.json: a list of {"name", "spec_hex", "n", "seed", "q", "rec", "trace_cap", "jobs_cap", "cluster_cap"}; each job
writes out_dir/<name>.npz with the summary, the event count and the trace, job log and cluster log of replica `rec`.

A job with "kind": "prepass" ({"name", "spec_hex", "n", "seed", "q", optional "first_replica_id", "rng", "replicas",
"reset"}) runs the arrival pre-pass and the list merge only (dcsim_prepare, no event loop) on buffers filled with 0xee
bytes first, and writes out_dir/<name>.npz with what they left for the local replicas listed in "replicas" (default:
all): arr_t, arr_raw, arr_meta, arr_pred, arr_tx, ml_t, ml_aux, ml_meta, hdr (raw dcsim_arrhdr_t bytes).  "reset":
{"seed", "first_replica_id"} reseeds the same handle afterwards and writes <name>__reset.npz the same way.
A job with "kind": "summary" ({"name", "spec_hex", "n", "seed", "q", optional "rng"}) writes the summary and the event
count of a whole run.
"""
import ctypes as C
import json
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)

from distributed_cluster_gpus_b200 import _native as N, spec as S  # noqa: E402
from distributed_cluster_gpus_b200.engine import BatchedEngine  # noqa: E402


PREPASS_ARRAYS = (("arr_t", np.float64, 1), ("arr_raw", np.float64, 1), ("arr_meta", np.uint32, 1), ("arr_pred", np.uint32, 1),
                  ("arr_tx", np.float64, 1), ("ml_t", np.float64, 2), ("ml_aux", np.float64, 2), ("ml_meta", np.uint32, 2))
HDR_BYTES = 32  # sizeof(dcsim_arrhdr_t)


def _fetch_prepass(lib, eng, replicas, cap_arr):
    """Poisoned buffers, dcsim_prepare, then the rows of `replicas`."""
    N.check(lib.dcsim_test_poison_prepass(eng._h), eng._h)
    eng.prepare()
    out = {k: np.zeros((len(replicas), w * cap_arr), dtype=dt) for k, dt, w in PREPASS_ARRAYS}
    out["hdr"] = np.zeros((len(replicas), HDR_BYTES), dtype=np.uint8)
    for i, r in enumerate(replicas):
        ptrs = [out[k][i].ctypes.data for k, _, _ in PREPASS_ARRAYS] + [out["hdr"][i].ctypes.data]
        N.check(lib.dcsim_test_fetch_prepass(eng._h, int(r), 1, *ptrs), eng._h)
    out["replicas"] = np.asarray(replicas, dtype=np.int64)
    return out


def run_prepass(lib, job, sp, out_dir):
    n = job["n"]
    replicas = job.get("replicas") or list(range(n))
    cap_arr = sp.cap_arrivals if sp.cap_arrivals > 0 else 16384
    with BatchedEngine(sp, n, base_seed=job["seed"], first_replica_id=job.get("first_replica_id", 0)) as eng:
        if job.get("rng", "philox") != "philox":
            eng.set_rng(job["rng"])
        np.savez(os.path.join(out_dir, job["name"] + ".npz"), **_fetch_prepass(lib, eng, replicas, cap_arr))
        if job.get("reset"):
            eng.reset(job["reset"]["seed"], job["reset"]["first_replica_id"])
            np.savez(os.path.join(out_dir, job["name"] + "__reset.npz"), **_fetch_prepass(lib, eng, replicas, cap_arr))


def main(jobs_path, out_dir):
    lib = N.load()
    if not hasattr(lib, "dcsim_test_set_time_quantum"):
        raise SystemExit(f"{N.LIB_PATH} is not the hook build (no dcsim_test_set_time_quantum)")
    lib.dcsim_test_set_time_quantum.restype = C.c_int
    lib.dcsim_test_set_time_quantum.argtypes = [C.c_double]
    lib.dcsim_test_poison_prepass.restype = C.c_int
    lib.dcsim_test_poison_prepass.argtypes = [C.c_void_p]
    lib.dcsim_test_fetch_prepass.restype = C.c_int
    lib.dcsim_test_fetch_prepass.argtypes = [C.c_void_p, C.c_uint64, C.c_uint64] + [C.c_void_p] * 9
    with open(jobs_path) as f:
        jobs = json.load(f)
    for job in jobs:
        N.check(lib.dcsim_test_set_time_quantum(float(job["q"])))   # read by dcsim_create
        sp = S.Spec.from_buffer_copy(bytes.fromhex(job["spec_hex"]))
        if job.get("kind") == "prepass":
            run_prepass(lib, job, sp, out_dir)
            continue
        if job.get("kind") == "summary":
            with BatchedEngine(sp, job["n"], base_seed=job["seed"]) as eng:
                if job.get("rng", "philox") != "philox":
                    eng.set_rng(job["rng"])
                events = eng.advance(0)
                np.savez(os.path.join(out_dir, job["name"] + ".npz"), summary=eng.summary(), events=events)
            continue
        with BatchedEngine(sp, job["n"], base_seed=job["seed"]) as eng:
            eng.set_trace(job["rec"], job["trace_cap"])
            eng.set_logging(job["rec"], job["jobs_cap"], job["cluster_cap"])
            events = eng.advance(0)
            np.savez(os.path.join(out_dir, job["name"] + ".npz"), summary=eng.summary(), events=events,
                     trace=eng.trace(), jobs=eng.job_log(), cluster=eng.cluster_log())
    N.check(lib.dcsim_test_set_time_quantum(0.0))


if __name__ == "__main__":
    main(sys.argv[1], sys.argv[2])
