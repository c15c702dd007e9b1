"""ctypes binding of csrc/libdcsim_b200.so (the C-ABI of include/dcsim_b200.h).

There is no CPU fallback: if the CUDA library is missing this module raises, and every engine call
surfaces the library's own error string.
"""
import ctypes as C
import os

from . import spec as S

_HERE = os.path.dirname(os.path.abspath(__file__))
# DCSIM_B200_LIB selects another build of the SAME CUDA library (tuning experiments); never a different backend.
LIB_PATH = os.environ.get("DCSIM_B200_LIB") or os.path.join(_HERE, "csrc", "libdcsim_b200.so")

OK, E_INVALID, E_CUDA, E_NOMEM, E_STATE, E_UNSUPPORTED = 0, -1, -2, -3, -4, -5

# every symbol include/dcsim_b200.h declares
EXPORTS = (
    "dcsim_sizeof_spec", "dcsim_abi_version", "dcsim_summary_k", "dcsim_create", "dcsim_reset", "dcsim_set_stream",
    "dcsim_set_trace", "dcsim_set_logging", "dcsim_prepare", "dcsim_advance", "dcsim_all_done", "dcsim_fetch_summary",
    "dcsim_summary_device_ptr", "dcsim_reduce_summary", "dcsim_enable_latency_histogram", "dcsim_fetch_latency_histogram", "dcsim_fetch_trace", "dcsim_fetch_job_log",
    "dcsim_fetch_cluster_log", "dcsim_launch_info", "dcsim_last_error", "dcsim_destroy", "dcsim_set_rng",
    "dcsim_recorder_counts", "dcsim_allreduce_summary", "dcsim_fetch_summary_host",
    "dcsim_enable_cluster_ensemble", "dcsim_cluster_ensemble_capacity", "dcsim_fetch_cluster_ensemble",
    "dcsim_ensemble_moments", "dcsim_ensemble_spread",
    "dcsim_enable_job_ensemble", "dcsim_job_ensemble_windows", "dcsim_fetch_job_ensemble", "dcsim_job_ensemble_moments",
    "dcsim_job_ensemble_spread", "dcsim_fetch_dc_latency_histogram",
    "dcsim_arrivals_compatible", "dcsim_create_shared", "dcsim_paired_moments", "dcsim_paired_spread",
    "dcsim_enable_power_profile", "dcsim_power_profile_range", "dcsim_fetch_power_profile", "dcsim_power_profile_moments",
    "dcsim_power_profile_spread",
    "dcsim_enable_job_waits", "dcsim_fetch_job_waits", "dcsim_job_waits_moments", "dcsim_job_waits_spread",
    "dcsim_fetch_dc_wait_histogram",
    "dcsim_enable_job_resources", "dcsim_fetch_job_resources", "dcsim_job_resources_moments", "dcsim_job_resources_spread",
    "dcsim_enable_occupancy", "dcsim_occupancy_bin_widths", "dcsim_fetch_occupancy", "dcsim_occupancy_moments",
    "dcsim_occupancy_spread",
    "dcsim_enable_tail_latency", "dcsim_fetch_tail_latency", "dcsim_fetch_tail_jobs", "dcsim_tail_latency_moments",
    "dcsim_tail_latency_spread",
    "dcsim_enable_energy_cost", "dcsim_fetch_energy_cost", "dcsim_energy_cost_moments", "dcsim_energy_cost_spread",
)

_lib = None


class NativeLibraryMissing(RuntimeError):
    pass


class DcsimError(RuntimeError):
    def __init__(self, code, message):
        super().__init__(f"dcsim error {code}: {message}")
        self.code = code


def load():
    """Loads the CUDA library (once) and declares prototypes."""
    global _lib
    if _lib is not None:
        return _lib
    if not os.path.exists(LIB_PATH):
        raise NativeLibraryMissing(
            f"{LIB_PATH} not found. Build it with `python -c 'import __graft_entry__ as g; g.build()'` "
            "(nvcc, sm_90a). The batched engine has no CPU fallback.")
    L = C.CDLL(LIB_PATH)
    vp, u64, u32, i32 = C.c_void_p, C.c_uint64, C.c_uint32, C.c_int
    L.dcsim_sizeof_spec.restype = C.c_size_t
    L.dcsim_abi_version.restype = u32
    L.dcsim_summary_k.restype = i32
    L.dcsim_create.restype = i32
    L.dcsim_create.argtypes = [vp, C.c_size_t, u64, u64, u64, i32, C.POINTER(vp)]
    L.dcsim_reset.restype = i32
    L.dcsim_reset.argtypes = [vp, u64, u64]
    L.dcsim_set_stream.restype = i32
    L.dcsim_set_stream.argtypes = [vp, vp]
    L.dcsim_set_trace.restype = i32
    L.dcsim_set_trace.argtypes = [vp, u64, u32]
    L.dcsim_set_logging.restype = i32
    L.dcsim_set_logging.argtypes = [vp, u64, u32, u32]
    L.dcsim_prepare.restype = i32
    L.dcsim_prepare.argtypes = [vp]
    L.dcsim_advance.restype = i32
    L.dcsim_advance.argtypes = [vp, u64, C.POINTER(u64)]
    L.dcsim_all_done.restype = i32
    L.dcsim_all_done.argtypes = [vp, C.POINTER(i32)]
    L.dcsim_fetch_summary.restype = i32
    L.dcsim_fetch_summary.argtypes = [vp, vp, C.c_size_t]
    L.dcsim_summary_device_ptr.restype = i32
    L.dcsim_summary_device_ptr.argtypes = [vp, C.POINTER(vp)]
    L.dcsim_reduce_summary.restype = i32
    L.dcsim_reduce_summary.argtypes = [vp, vp]
    L.dcsim_set_rng.restype = i32
    L.dcsim_set_rng.argtypes = [vp, C.c_int]
    L.dcsim_enable_latency_histogram.restype = i32
    L.dcsim_enable_latency_histogram.argtypes = [vp]
    L.dcsim_fetch_latency_histogram.restype = i32
    L.dcsim_fetch_latency_histogram.argtypes = [vp, vp, C.c_size_t]
    for name in ("dcsim_fetch_trace", "dcsim_fetch_job_log", "dcsim_fetch_cluster_log"):
        getattr(L, name).restype = i32
        getattr(L, name).argtypes = [vp, vp, u32, C.POINTER(u32)]
    if hasattr(L, "dcsim_allreduce_summary"):      # (older tuning builds selected with DCSIM_B200_LIB may lack the newest entry points)
        L.dcsim_allreduce_summary.restype = i32
        L.dcsim_allreduce_summary.argtypes = [vp, vp, vp]
    if hasattr(L, "dcsim_fetch_summary_host"):
        L.dcsim_fetch_summary_host.restype = i32
        L.dcsim_fetch_summary_host.argtypes = [vp, C.POINTER(C.POINTER(C.c_double))]
    if hasattr(L, "dcsim_recorder_counts"):
        L.dcsim_recorder_counts.restype = i32
        L.dcsim_recorder_counts.argtypes = [vp, C.POINTER(u32 * 3)]
    if hasattr(L, "dcsim_enable_cluster_ensemble"):
        L.dcsim_enable_cluster_ensemble.restype = i32
        L.dcsim_enable_cluster_ensemble.argtypes = [vp, u32]
        L.dcsim_cluster_ensemble_capacity.restype = i32
        L.dcsim_cluster_ensemble_capacity.argtypes = [vp, C.POINTER(u32)]
        L.dcsim_fetch_cluster_ensemble.restype = i32
        L.dcsim_fetch_cluster_ensemble.argtypes = [vp, vp, C.c_size_t]
        L.dcsim_ensemble_moments.restype = i32
        L.dcsim_ensemble_moments.argtypes = [vp, vp]
        L.dcsim_ensemble_spread.restype = i32
        L.dcsim_ensemble_spread.argtypes = [vp, vp, vp, vp, vp, vp]
    if hasattr(L, "dcsim_enable_job_ensemble"):
        L.dcsim_enable_job_ensemble.restype = i32
        L.dcsim_enable_job_ensemble.argtypes = [vp, C.c_double]
        L.dcsim_job_ensemble_windows.restype = i32
        L.dcsim_job_ensemble_windows.argtypes = [vp, C.POINTER(u32)]
        L.dcsim_fetch_job_ensemble.restype = i32
        L.dcsim_fetch_job_ensemble.argtypes = [vp, vp, C.c_size_t, vp, C.c_size_t]
        L.dcsim_job_ensemble_moments.restype = i32
        L.dcsim_job_ensemble_moments.argtypes = [vp, vp]
        L.dcsim_job_ensemble_spread.restype = i32
        L.dcsim_job_ensemble_spread.argtypes = [vp, vp, vp, vp, vp, vp]
        L.dcsim_fetch_dc_latency_histogram.restype = i32
        L.dcsim_fetch_dc_latency_histogram.argtypes = [vp, vp, C.c_size_t]
    if hasattr(L, "dcsim_create_shared"):
        L.dcsim_arrivals_compatible.restype = i32
        L.dcsim_arrivals_compatible.argtypes = [vp, C.c_size_t, vp, C.c_size_t, C.POINTER(i32)]
        L.dcsim_create_shared.restype = i32
        L.dcsim_create_shared.argtypes = [vp, C.c_size_t, vp, C.POINTER(vp)]
        L.dcsim_paired_moments.restype = i32
        L.dcsim_paired_moments.argtypes = [vp, vp, u64, vp]
        L.dcsim_paired_spread.restype = i32
        L.dcsim_paired_spread.argtypes = [vp, vp, u64, vp, vp, vp, vp, vp]
    if hasattr(L, "dcsim_enable_job_waits"):
        L.dcsim_enable_job_waits.restype = i32
        L.dcsim_enable_job_waits.argtypes = [vp]
        L.dcsim_fetch_job_waits.restype = i32
        L.dcsim_fetch_job_waits.argtypes = [vp, vp, C.c_size_t, vp, C.c_size_t]
        L.dcsim_job_waits_moments.restype = i32
        L.dcsim_job_waits_moments.argtypes = [vp, vp]
        L.dcsim_job_waits_spread.restype = i32
        L.dcsim_job_waits_spread.argtypes = [vp, vp, vp, vp, vp, vp]
        L.dcsim_fetch_dc_wait_histogram.restype = i32
        L.dcsim_fetch_dc_wait_histogram.argtypes = [vp, vp, C.c_size_t]
    if hasattr(L, "dcsim_enable_job_resources"):
        L.dcsim_enable_job_resources.restype = i32
        L.dcsim_enable_job_resources.argtypes = [vp]
        L.dcsim_fetch_job_resources.restype = i32
        L.dcsim_fetch_job_resources.argtypes = [vp, vp, C.c_size_t, vp, C.c_size_t, vp, C.c_size_t]
        L.dcsim_job_resources_moments.restype = i32
        L.dcsim_job_resources_moments.argtypes = [vp, vp]
        L.dcsim_job_resources_spread.restype = i32
        L.dcsim_job_resources_spread.argtypes = [vp, vp, vp, vp, vp, vp]
    if hasattr(L, "dcsim_enable_occupancy"):
        L.dcsim_enable_occupancy.restype = i32
        L.dcsim_enable_occupancy.argtypes = [vp]
        L.dcsim_occupancy_bin_widths.restype = i32
        L.dcsim_occupancy_bin_widths.argtypes = [vp, vp]
        L.dcsim_fetch_occupancy.restype = i32
        L.dcsim_fetch_occupancy.argtypes = [vp, vp, C.c_size_t]
        L.dcsim_occupancy_moments.restype = i32
        L.dcsim_occupancy_moments.argtypes = [vp, vp]
        L.dcsim_occupancy_spread.restype = i32
        L.dcsim_occupancy_spread.argtypes = [vp, vp, vp, vp, vp, vp]
    if hasattr(L, "dcsim_enable_tail_latency"):
        L.dcsim_enable_tail_latency.restype = i32
        L.dcsim_enable_tail_latency.argtypes = [vp, C.c_double]
        L.dcsim_fetch_tail_latency.restype = i32
        L.dcsim_fetch_tail_latency.argtypes = [vp, vp, C.c_size_t]
        L.dcsim_fetch_tail_jobs.restype = i32
        L.dcsim_fetch_tail_jobs.argtypes = [vp, u64, u64, vp, C.c_size_t]
        L.dcsim_tail_latency_moments.restype = i32
        L.dcsim_tail_latency_moments.argtypes = [vp, vp]
        L.dcsim_tail_latency_spread.restype = i32
        L.dcsim_tail_latency_spread.argtypes = [vp, vp, vp, vp, vp, vp]
    if hasattr(L, "dcsim_enable_power_profile"):
        L.dcsim_enable_power_profile.restype = i32
        L.dcsim_enable_power_profile.argtypes = [vp, C.c_double]
        L.dcsim_power_profile_range.restype = i32
        L.dcsim_power_profile_range.argtypes = [vp, C.POINTER(C.c_double)]
        L.dcsim_fetch_power_profile.restype = i32
        L.dcsim_fetch_power_profile.argtypes = [vp, vp, C.c_size_t]
        L.dcsim_power_profile_moments.restype = i32
        L.dcsim_power_profile_moments.argtypes = [vp, vp]
        L.dcsim_power_profile_spread.restype = i32
        L.dcsim_power_profile_spread.argtypes = [vp, vp, vp, vp, vp, vp]
    if hasattr(L, "dcsim_enable_energy_cost"):
        L.dcsim_enable_energy_cost.restype = i32
        L.dcsim_enable_energy_cost.argtypes = [vp]
        L.dcsim_fetch_energy_cost.restype = i32
        L.dcsim_fetch_energy_cost.argtypes = [vp, vp, C.c_size_t]
        L.dcsim_energy_cost_moments.restype = i32
        L.dcsim_energy_cost_moments.argtypes = [vp, vp]
        L.dcsim_energy_cost_spread.restype = i32
        L.dcsim_energy_cost_spread.argtypes = [vp, vp, vp, vp, vp, vp]
    L.dcsim_launch_info.restype = i32
    L.dcsim_launch_info.argtypes = [vp, C.POINTER(S.LaunchInfo)]
    L.dcsim_last_error.restype = C.c_char_p
    L.dcsim_last_error.argtypes = [vp]
    L.dcsim_destroy.restype = None
    L.dcsim_destroy.argtypes = [vp]
    if L.dcsim_sizeof_spec() != C.sizeof(S.Spec) or L.dcsim_abi_version() != S.ABI_VERSION or \
            L.dcsim_summary_k() != S.SUMMARY_K:
        raise RuntimeError("libdcsim_b200.so and spec.py disagree on the ABI (rebuild the library)")
    _lib = L
    return L


def check(rc, handle=None):
    if rc != OK:
        msg = load().dcsim_last_error(handle)
        raise DcsimError(rc, (msg or b"").decode("utf-8", "replace"))
