"""TEST-ONLY plain reference of the list merge (dcsim_merge_arrivals in distributed_cluster_gpus_b200/csrc/dcsim_core.cuh).

Given one replica's arrivals as the pre-pass wrote them, it builds the time-ordered {arrival, xfer_done} list the event
loop reads, from the heap's own rule (simulator_paper_multi.py:160-166, "SIM"): events pop in (t, seq) order and seq
is push order.  Every push that reaches the list happens while an arrival is processed (its xfer_done first, then its
stream's next arrival, SIM:580-592), or in the constructor (each stream's first arrival, in stream order, SIM:154-156).
So the push rank
    first arrival of stream s    (-1, s)
    xfer_done of arrival j       (j, 0)
    arrival pushed by arrival j  (j, 1)
orders pushes like seq does, and the list is the stable sort of (t, rank).  No window, ring or running count is
involved: this is what the merge's per-arrival walks must reproduce, byte for byte (only IEEE adds, divides and ceil
produce the instants).
"""
import numpy as np

NO_PRED = 0xFFFFFFFF
ML_XFER = 1
ML_A_NEXT = 1 << 5
ML_A_XSCHED = 1 << 6
ML_A_XIN = 1 << 7
ST_XFER_OVERFLOW = 1  # DCSIM_ST_XFER_OVERFLOW


def quantize(t, q):
    """dcsim_test_quantize: round up to a multiple of q (q = 0: off); +inf stays +inf."""
    t = np.asarray(t, dtype=np.float64)
    if not q > 0.0:
        return t.copy()
    with np.errstate(invalid="ignore"):
        return np.where(t == np.inf, t, np.ceil(t / q) * q)


def xring_mask(spec):
    """dcsim_xring_entries(spec) - 1: the transfer-seq ring the merge checks max_ahead against."""
    cx = spec.cap_xfer if spec.cap_xfer > 0 else 64
    ring = 8
    while ring < 2 * cx:
        ring <<= 1
    return ring - 1


def hilo(hi, lo):
    """dcsim_hilo_f64: the double whose bit pattern is hi << 32 | lo."""
    return np.array([(int(hi) << 32) | int(lo)], dtype=np.uint64).view(np.float64)[0]


def merge(t, meta, pred, size, transfer_s, end_time, quantum=0.0, ring_mask=None):
    """One replica's list.  t / meta / pred / size: its arrivals in order (meta: stream bits 0-3, DC bits 4-6, the
    next-arrival bit 0x80; size: the job size the xfer_done entry carries); transfer_s[ingress][dc][jtype].
    -> {"ml_t", "ml_aux", "ml_meta", "ml_count", "max_ahead", "status", "tx"} (tx: the xfer_done instant of every
    arrival, +inf when none, what the merge leaves in arr_tx)."""
    t = np.asarray(t, dtype=np.float64)
    meta = np.asarray(meta, dtype=np.uint32)
    pred = np.asarray(pred, dtype=np.uint32)
    size = np.asarray(size, dtype=np.float64)
    n = len(t)
    stream = (meta & 15).astype(np.int64)
    jt, ing, dc = stream & 1, stream >> 1, ((meta >> 4) & 7).astype(np.int64)
    trans = np.array([transfer_s[i][d][j] for i, d, j in zip(ing, dc, jt)], dtype=np.float64)
    tx = quantize(t + trans, quantum)
    end = float(end_time)
    end_eps = end + 1e-9                                   # SIM:161
    xs = (tx != np.inf) & ~(tx > end_eps)                  # the push takes a seq
    xin = xs & ~(tx > end)                                 # ... and is processed: it is in the list

    k = np.arange(n, dtype=np.int64)
    first = pred == NO_PRED
    # entries: the n arrivals, then the listed xfer_done events
    xk = k[xin]
    ev_t = np.concatenate([t, tx[xin]])
    r0 = np.concatenate([np.where(first, -1, pred.astype(np.int64)), xk])
    r1 = np.concatenate([np.where(first, stream, 1), np.zeros(len(xk), dtype=np.int64)])
    order = np.lexsort((r1, r0, ev_t))                     # primary t, then rank
    pos = np.empty(len(order), dtype=np.int64)
    pos[order] = np.arange(len(order))
    pos_a, pos_x = pos[:n], pos[n:]

    m = len(order)
    ml_t = ev_t[order]
    ml_meta = np.zeros(m, dtype=np.uint32)
    ml_aux = np.zeros(m, dtype=np.float64)
    px_full = np.full(n, NO_PRED, dtype=np.int64)
    px_full[xk] = pos_x
    a_meta = ((stream << 1) | np.where(meta & 0x80, ML_A_NEXT, 0) | np.where(xs, ML_A_XSCHED, 0)
              | np.where(xin, ML_A_XIN, 0)).astype(np.uint32)
    ml_meta[pos_a] = a_meta
    ml_aux[pos_a] = px_full.astype(np.uint64).view(np.float64)   # hilo(0, pos_x)
    x_meta = (ML_XFER | (dc[xk] << 1) | (jt[xk] << 4) | (ing[xk] << 5) | (xk << 8)).astype(np.uint32)
    ml_meta[pos_x] = x_meta
    ml_aux[pos_x] = size[xk]
    ahead = int(np.max(pos_x - pos_a[xk])) if len(xk) else 0
    status = ST_XFER_OVERFLOW if ring_mask is not None and ahead > ring_mask else 0
    return {"ml_t": ml_t, "ml_aux": ml_aux, "ml_meta": ml_meta, "ml_count": m, "max_ahead": ahead,
            "status": status, "tx": tx}


def merge_spec(spec, t, meta, pred, size, quantum=0.0):
    """merge() with the transfer times, end_time and ring of a dcsim_spec_t (spec.Spec)."""
    tr = [[[spec.transfer_s[i][d][j] for j in range(2)] for d in range(spec.n_dc)] for i in range(spec.n_ing)]
    return merge(t, meta, pred, size, tr, spec.end_time, quantum, xring_mask(spec))
