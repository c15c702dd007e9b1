"""TEST-ONLY driver of the CUDA library built with -DDCSIM_TEST_HOOKS (tests/gpuhooks/_build, see __graft_entry__.build).

That build rounds every arrival and xfer_done instant up to a multiple of a time quantum on the device, like the
oracle's and the host build's hook, so that same-instant events become common.  It is loaded in a process of its own
(DCSIM_B200_LIB names it) so the test process keeps the product library.

    DCSIM_B200_LIB=<hook lib> python tests/gpuhooks/driver.py jobs.json out_dir

jobs.json: a list of {"name", "spec_hex", "n", "seed", "q", "rec", "trace_cap", "jobs_cap", "cluster_cap"}; each job
writes out_dir/<name>.npz with the summary, the event count and the trace, job log and cluster log of replica `rec`.
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


def main(jobs_path, out_dir):
    lib = N.load()
    if not hasattr(lib, "dcsim_test_set_time_quantum"):
        raise SystemExit(f"{N.LIB_PATH} is not the hook build (no dcsim_test_set_time_quantum)")
    lib.dcsim_test_set_time_quantum.restype = C.c_int
    lib.dcsim_test_set_time_quantum.argtypes = [C.c_double]
    with open(jobs_path) as f:
        jobs = json.load(f)
    for job in jobs:
        N.check(lib.dcsim_test_set_time_quantum(float(job["q"])))   # read by dcsim_create
        sp = S.Spec.from_buffer_copy(bytes.fromhex(job["spec_hex"]))
        with BatchedEngine(sp, job["n"], base_seed=job["seed"]) as eng:
            eng.set_trace(job["rec"], job["trace_cap"])
            eng.set_logging(job["rec"], job["jobs_cap"], job["cluster_cap"])
            events = eng.advance(0)
            np.savez(os.path.join(out_dir, job["name"] + ".npz"), summary=eng.summary(), events=events,
                     trace=eng.trace(), jobs=eng.job_log(), cluster=eng.cluster_log())
    N.check(lib.dcsim_test_set_time_quantum(0.0))


if __name__ == "__main__":
    main(sys.argv[1], sys.argv[2])
