"""ctypes binding of libmvicp.so (include/mvicp.h).  No CPU fallback: if the library is missing it is built with
nvcc; if that fails, or no CUDA device exists at call time, the error is raised."""
import ctypes as C
import os
import subprocess

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_HERE, "libmvicp.so")
CSRC = os.path.join(_HERE, "csrc")


class Config(C.Structure):
    _fields_ = [("device", C.c_int32), ("flags", C.c_int32), ("stream", C.c_void_p)]


class LmOptions(C.Structure):
    _fields_ = [("max_num_iterations", C.c_int32), ("max_num_consecutive_invalid_steps", C.c_int32),
                ("jacobi_scaling", C.c_int32), ("reserved", C.c_int32),
                ("initial_trust_region_radius", C.c_double), ("max_trust_region_radius", C.c_double),
                ("min_trust_region_radius", C.c_double), ("min_relative_decrease", C.c_double),
                ("min_lm_diagonal", C.c_double), ("max_lm_diagonal", C.c_double),
                ("function_tolerance", C.c_double), ("gradient_tolerance", C.c_double),
                ("parameter_tolerance", C.c_double)]


class LmSummary(C.Structure):
    _fields_ = [("termination", C.c_int32), ("num_iterations", C.c_int32), ("num_successful_steps", C.c_int32),
                ("num_evaluations", C.c_int32), ("num_linear_solves", C.c_int32), ("reserved", C.c_int32),
                ("initial_cost", C.c_double), ("final_cost", C.c_double)]

    def asdict(self):
        return {k: getattr(self, k) for k, _ in self._fields_ if k != "reserved"}


class G2oOptions(C.Structure):
    _fields_ = [("iterations_per_call", C.c_int32), ("max_calls", C.c_int32), ("no_improvement_limit", C.c_int32),
                ("max_trials", C.c_int32), ("orthonormalize_after", C.c_int32), ("reserved", C.c_int32),
                ("tau", C.c_double), ("information_eps", C.c_double)]


class G2oSummary(C.Structure):
    _fields_ = [("calls", C.c_int32), ("iterations", C.c_int32), ("trials", C.c_int32), ("accepted", C.c_int32),
                ("evaluations", C.c_int32), ("ended", C.c_int32), ("last_call_end", C.c_int32), ("reserved", C.c_int32),
                ("chi2_initial", C.c_double), ("chi2_final", C.c_double)]

    def asdict(self):
        return {k: getattr(self, k) for k, _ in self._fields_ if k != "reserved"}


class Stats(C.Structure):
    _fields_ = [("knn_ms", C.c_float), ("select_ms", C.c_float), ("lm_eval_ms", C.c_float), ("lm_other_ms", C.c_float),
                ("correspond_ms", C.c_float), ("optimize_ms", C.c_float),
                ("kernel_launches", C.c_int64), ("queries", C.c_int64), ("correspondences", C.c_int64),
                ("select_guess_rounds", C.c_int64), ("select_guess_misses", C.c_int64),
                ("cert_rounds", C.c_int64), ("cert_reused", C.c_int64)]

    def asdict(self):
        return {k: getattr(self, k) for k, _ in self._fields_}


EXPORTS = ["mvicp_default_lm_options", "mvicp_last_error", "mvicp_create", "mvicp_destroy", "mvicp_set_frames",
           "mvicp_set_poses", "mvicp_get_poses", "mvicp_set_graph", "mvicp_pose_graph_knn", "mvicp_get_graph",
           "mvicp_correspond", "mvicp_get_edge", "mvicp_get_all_edges", "mvicp_get_nn", "mvicp_set_edge", "mvicp_closest_point",
           "mvicp_optimize", "mvicp_icp_round", "mvicp_pairwise", "mvicp_pairwise_closed", "mvicp_recompute_normals", "mvicp_get_normals", "mvicp_knn_self", "mvicp_nccl_unique_id", "mvicp_comm_init",
           "mvicp_get_stats", "mvicp_get_stream", "mvicp_sync", "mvicp_abi_version", "mvicp_host_alloc", "mvicp_host_free",
           "mvicp_default_g2o_options", "mvicp_optimize_g2o", "mvicp_pairwise_g2o", "mvicp_g2o_trace",
           "mvicp_closest_points", "mvicp_set_frames_device", "mvicp_set_edge_device", "mvicp_get_all_edges_device",
           "mvicp_closest_points_device", "mvicp_get_normals_device", "mvicp_knn_self_device",
           "mvicp_get_components", "mvicp_optimize_components", "mvicp_optimize_g2o_components", "mvicp_g2o_trace_component",
           "mvicp_covariance"]

COV_OK, COV_FIXED, COV_INDEPENDENT, COV_SINGULAR = 0, 1, 2, 3   # mvicp_covariance's per-pair status (MVICP_COV_*)


def build(force=False):
    """Compile libmvicp.so for sm_90a (nvcc cross-compiles without a GPU)."""
    srcs = [os.path.join(CSRC, f) for f in os.listdir(CSRC)] + [os.path.join(_HERE, "..", "include", "mvicp.h")]
    stale = force or not os.path.exists(LIB_PATH) or any(os.path.getmtime(s) > os.path.getmtime(LIB_PATH) for s in srcs)
    if stale:
        r = subprocess.run(["make", "-C", CSRC, "-s"], capture_output=True, text=True)
        if r.returncode != 0:
            raise RuntimeError("building libmvicp.so failed:\n" + r.stdout + r.stderr)
    return LIB_PATH


_lib = None


def _preload_nccl():
    """libmvicp.so needs libnccl.so.2.  PyTorch bundles a newer NCCL than the system one under the same soname; whichever
    is loaded first wins for the whole process, and torch fails to import on top of the older one.  Load torch's copy
    first when it exists (no torch import needed), so that both libraries share it regardless of import order."""
    import importlib.util
    try:
        spec = importlib.util.find_spec("nvidia")
        for base in (spec.submodule_search_locations if spec else []):
            p = os.path.join(base, "nccl", "lib", "libnccl.so.2")
            if os.path.exists(p):
                C.CDLL(p, mode=C.RTLD_GLOBAL)
                return p
    except Exception:
        pass
    return None


def lib():
    global _lib
    if _lib is None:
        build()
        _preload_nccl()
        _lib = C.CDLL(LIB_PATH)
        _lib.mvicp_last_error.restype = C.c_char_p
    return _lib


class MvicpError(RuntimeError):
    def __init__(self, code, msg):
        super().__init__(f"mvicp error {code}: {msg}")
        self.code = code


def check(rc):
    if rc != 0:
        raise MvicpError(rc, lib().mvicp_last_error().decode())
