"""karpenter-core_b200 — H100-native (sm_90a) drop-in for Karpenter's provisioning scheduler hot path.

Python is only the test / bench harness here: every call goes through the C-ABI library
`libksched.so` (include/ksched.h + the C++ host layer in host/). There is no Python or CPU
implementation of the solver in this package; without the CUDA extension the calls raise.

Names mirror the reference: `Scheduler.solve` <-> scheduling.Scheduler.Solve (scheduler.go:96),
`simulate_scheduling` <-> deprovisioning.simulateScheduling (helpers.go:42),
`MultiNodeConsolidation.first_n_node_consolidation_option` <-> multinodeconsolidation.go:74.
"""
import ctypes as C
import json
import weakref
from pathlib import Path

import numpy as np

PKG_DIR = Path(__file__).resolve().parent
LIB_PATH = PKG_DIR / "libksched.so"

KSCHED_OK = 0
KSCHED_ERR_INVALID = -1
KSCHED_ERR_UNSUPPORTED = -2
KSCHED_ERR_CUDA = -3
KSCHED_ERR_NCCL = -4
KSCHED_ERR_NO_DEVICE = -5
KSCHED_ERR_OVERFLOW = -6

# every symbol include/ksched.h declares
ABI_SYMBOLS = [
    "ksched_abi_version", "ksched_device_count", "ksched_create", "ksched_destroy", "ksched_last_error",
    "ksched_type_words", "ksched_load_catalog", "ksched_set_shard", "ksched_shard_range", "ksched_nccl_unique_id", "ksched_nccl_init",
    "ksched_solve", "ksched_upload", "ksched_run_resident", "ksched_download", "ksched_run_feasibility_only",
    "ksched_get_timings", "ksched_load_cluster", "ksched_simulate_batch", "ksched_simulate_full", "ksched_allgather", "ksched_rank_candidates",
]


class KschedError(RuntimeError):
    def __init__(self, code, message):
        super().__init__(f"ksched error {code}: {message}")
        self.code = code


class Timings(C.Structure):
    _fields_ = [("upload_us", C.c_double), ("sort_us", C.c_double), ("feasibility_us", C.c_double), ("pack_us", C.c_double),
                ("download_us", C.c_double), ("total_us", C.c_double), ("allreduce_us", C.c_double),
                ("feasibility_bytes", C.c_int64), ("pack_steps", C.c_int64),
                ("feasibility_launches", C.c_int32), ("pack_launches", C.c_int32), ("sort_launches", C.c_int32), ("pad", C.c_int32),
                ("h2d_bytes", C.c_int64), ("d2h_bytes", C.c_int64), ("class_feasibility_us", C.c_double),
                ("vt_build_us", C.c_double), ("vt_fetches", C.c_int64), ("run_derives", C.c_int64),
                ("pack_interval_ns", C.c_int64 * 2)]

    def as_dict(self):
        d = {k: getattr(self, k) for k, _ in self._fields_ if k != "pad"}
        d["pack_interval_ns"] = tuple(self.pack_interval_ns)
        return d


_model = None
MODEL_LIB_PATH = Path(__file__).resolve().parent / "libkmodel.so"


def model_lib():
    """libkmodel.so: the string-level model (JSON loader, synthetic BASELINE configurations, result accessors). No CUDA and
    no solver in it: the oracle's tests and the bench's reference arm load this library alone."""
    global _model
    if _model is not None:
        return _model
    if not MODEL_LIB_PATH.exists():
        raise RuntimeError(f"{MODEL_LIB_PATH} is missing: run `python -c 'import __graft_entry__ as g; g.build()'`")
    L = C.CDLL(str(MODEL_LIB_PATH))
    L.kh_last_error.restype = C.c_char_p
    L.kh_problem_from_json.restype = C.c_void_p
    L.kh_problem_from_json.argtypes = [C.c_char_p]
    L.kh_problem_synth.restype = C.c_void_p
    L.kh_problem_synth.argtypes = [C.c_int, C.c_longlong, C.c_longlong, C.c_ulonglong, C.c_longlong]
    L.kh_problem_free.argtypes = [C.c_void_p]
    L.kh_problem_counts.argtypes = [C.c_void_p, C.POINTER(C.c_longlong)]
    L.kh_parse_quantity.restype = C.c_longlong
    L.kh_parse_quantity.argtypes = [C.c_char_p]
    L.kh_result_new.restype = C.c_void_p
    L.kh_result_free.argtypes = [C.c_void_p]
    L.kh_result_error.restype = C.c_char_p
    L.kh_result_error.argtypes = [C.c_void_p]
    for name in ("kh_result_num_pods", "kh_result_num_new_nodes", "kh_result_num_existing", "kh_result_nodes_visited", "kh_result_add_calls"):
        getattr(L, name).restype = C.c_longlong
        getattr(L, name).argtypes = [C.c_void_p]
    L.kh_result_all_pods_scheduled.argtypes = L.kh_result_uninitialized_existing.argtypes = [C.c_void_p]
    L.kh_result_assign.argtypes = [C.c_void_p, C.c_void_p]
    L.kh_result_relax.argtypes = [C.c_void_p, C.c_void_p]
    L.kh_result_new_node_info.argtypes = [C.c_void_p, C.c_void_p]
    L.kh_result_new_node_options.restype = C.c_longlong
    L.kh_result_new_node_options.argtypes = [C.c_void_p, C.c_longlong, C.c_void_p, C.c_longlong]
    L.kh_result_digest.restype = C.c_ulonglong
    L.kh_result_digest.argtypes = [C.c_void_p]
    L.kh_result_to_json.restype = C.c_longlong
    L.kh_result_to_json.argtypes = [C.c_void_p, C.c_char_p, C.c_longlong]
    L.kh_result_to_json_brief.restype = C.c_longlong
    L.kh_result_to_json_brief.argtypes = [C.c_void_p, C.c_char_p, C.c_longlong]
    L.kh_problem_pod_summary.argtypes = [C.c_void_p, C.c_void_p]
    _model = L
    return L


_lib = None


def lib():
    """Load libksched.so (fails loudly when the extension was not built)."""
    global _lib
    if _lib is not None:
        return _lib
    if not LIB_PATH.exists():
        raise RuntimeError(f"{LIB_PATH} is missing: run `python -c 'import __graft_entry__ as g; g.build()'` "
                           "(there is no CPU fallback for the solver)")
    L = C.CDLL(str(LIB_PATH))
    L.kh_scheduler_error.restype = C.c_char_p
    L.kh_encoded_digest.restype = C.c_ulonglong
    L.kh_encoded_digest.argtypes = [C.c_void_p]
    L.kh_launch_table_selfcheck.argtypes = [C.c_void_p, C.c_void_p]
    L.kh_set_device.argtypes = [C.c_int]
    L.kh_set_count_visited.argtypes = [C.c_int]
    L.kh_handle.restype = C.c_void_p
    L.kh_scheduler_solve.argtypes = [C.c_void_p, C.POINTER(C.c_int), C.c_int, C.c_void_p]
    L.kh_scheduler_solve_timed.argtypes = [C.c_void_p, C.POINTER(C.c_int), C.c_int, C.c_void_p, C.POINTER(C.c_double)]
    L.kh_encode.restype = C.c_void_p
    L.kh_encode.argtypes = [C.c_void_p, C.POINTER(C.c_int), C.c_int]
    L.kh_encode_cluster.restype = C.c_void_p
    L.kh_encode_cluster.argtypes = [C.c_void_p, C.POINTER(C.c_int), C.c_int]
    L.kh_encoded_free.argtypes = [C.c_void_p]
    L.kh_encoded_dims.argtypes = [C.c_void_p, C.POINTER(C.c_longlong)]
    L.kh_encoded_key_info.argtypes = [C.c_void_p, C.c_char_p, C.POINTER(C.c_longlong)]
    L.kh_encoded_resource_id.argtypes = [C.c_void_p, C.c_char_p]
    L.kh_encoded_hostport.argtypes = [C.c_void_p, C.c_int, C.c_char_p, C.c_int]
    L.kh_encoded_volume_claim.argtypes = [C.c_void_p, C.c_int, C.c_char_p, C.c_int]
    L.kh_encoded_offering_slot.argtypes = [C.c_void_p, C.c_int, C.c_char_p, C.c_int]
    L.kh_encoded_offering_slots.argtypes = [C.c_void_p]
    L.kh_encoded_offering_slots.restype = C.c_longlong
    L.kh_encoded_hostname_req.argtypes = [C.c_void_p, C.c_int, C.POINTER(C.c_longlong), C.c_int]
    L.kh_encoded_class_hostname.argtypes = [C.c_void_p, C.c_int]
    L.kh_encoded_class_hostname.restype = C.c_longlong
    L.kh_encoded_pod_class.argtypes = [C.c_void_p, C.c_int]
    L.kh_encoded_pod_class.restype = C.c_longlong
    L.kh_encoded_group_total.argtypes = [C.c_void_p, C.c_int]
    L.kh_encoded_group_total.restype = C.c_longlong
    L.kh_value_class_selftest.argtypes = [C.c_uint, C.c_int]
    L.kh_gpu_load.argtypes = [C.c_void_p]
    L.kh_encoded_set_count_visited.argtypes = [C.c_void_p, C.c_int]
    L.kh_gpu_run.argtypes = [C.c_int]
    L.kh_gpu_run_feasibility.argtypes = [C.c_int, C.POINTER(C.c_float)]
    L.kh_gpu_download.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p]
    L.kh_gpu_timings.argtypes = [C.POINTER(Timings)]
    L.kh_gpu_solve_e2e.argtypes = [C.c_void_p, C.c_void_p, C.POINTER(C.c_double)]
    L.kh_gpu_load_catalog.argtypes = [C.c_void_p]
    L.kh_encoded_class_row.argtypes = [C.c_void_p, C.c_int, C.c_void_p]
    L.kh_gpu_k1_plan.argtypes = [C.POINTER(C.c_int)]
    L.kh_gpu_run_records.argtypes = [C.c_void_p, C.c_int]
    L.kh_gpu_set_shard.argtypes = [C.c_int, C.c_int]
    L.kh_consolidate.argtypes = [C.c_void_p, C.POINTER(C.c_int), C.POINTER(C.c_int), C.c_int, C.POINTER(C.c_int), C.POINTER(C.c_int), C.c_int,
                                 C.POINTER(C.c_int)]
    L.kh_consolidate_candidates.argtypes = [C.c_void_p]
    L.kh_cluster_open.restype = C.c_void_p
    L.kh_cluster_open.argtypes = [C.c_void_p, C.POINTER(C.c_int), C.POINTER(C.c_int)]
    L.kh_context_create.restype = C.c_void_p
    L.kh_context_create.argtypes = [C.c_int]
    L.kh_context_destroy.argtypes = [C.c_void_p]
    L.kh_context_solve.argtypes = [C.c_void_p, C.c_void_p, C.POINTER(C.c_int), C.c_int, C.c_void_p]
    L.kh_context_timings.argtypes = [C.c_void_p, C.POINTER(Timings)]
    L.kh_context_cluster_open.restype = C.c_void_p
    L.kh_context_cluster_open.argtypes = [C.c_void_p, C.c_void_p, C.POINTER(C.c_int), C.POINTER(C.c_int)]
    L.kh_cluster_close.argtypes = [C.c_void_p]
    L.kh_cluster_probe_sets.argtypes = [C.c_void_p, C.POINTER(C.c_int), C.POINTER(C.c_int), C.c_int, C.c_int, C.POINTER(C.c_int), C.POINTER(C.c_int), C.c_int,
                                        C.POINTER(C.c_int)]
    L.kh_cluster_candidates.argtypes = [C.c_void_p, C.POINTER(C.c_int), C.c_int]
    L.kh_cluster_simulate.argtypes = [C.c_void_p, C.POINTER(C.c_int), C.POINTER(C.c_int), C.c_int, C.POINTER(C.c_void_p)]
    L.kh_consolidate_single.argtypes = [C.c_void_p, C.c_int, C.c_int, C.c_int, C.POINTER(C.c_int), C.POINTER(C.c_int), C.POINTER(C.c_int), C.c_int]
    L.kh_consolidate_validated.argtypes = [C.c_void_p, C.c_void_p, C.POINTER(C.c_int), C.POINTER(C.c_int), C.c_int, C.POINTER(C.c_int), C.POINTER(C.c_int),
                                           C.c_int, C.POINTER(C.c_int), C.POINTER(C.c_int)]
    L.kh_consolidate_single_validated.argtypes = [C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.c_int, C.POINTER(C.c_int), C.POINTER(C.c_int),
                                                  C.POINTER(C.c_int), C.c_int, C.POINTER(C.c_int), C.POINTER(C.c_int), C.c_int, C.POINTER(C.c_int),
                                                  C.POINTER(C.c_int)]
    L.kh_cluster_validate.argtypes = [C.c_void_p, C.c_void_p, C.POINTER(C.c_int), C.POINTER(C.c_int), C.c_int, C.POINTER(C.c_int), C.POINTER(C.c_int),
                                      C.c_int, C.POINTER(C.c_int), C.POINTER(C.c_int)]
    L.kh_allgather_i32.argtypes = [C.POINTER(C.c_int), C.c_int, C.POINTER(C.c_int)]
    L.kh_nccl_init.argtypes = [C.c_void_p, C.c_int, C.c_int]
    L.kh_rank_candidates.argtypes = [C.c_void_p, C.POINTER(C.c_int), C.POINTER(C.c_double), C.c_int]
    L.kh_consolidate_probe.argtypes = [C.c_void_p, C.c_int, C.POINTER(C.c_int), C.c_int, C.POINTER(C.c_int)]
    L.kh_mask_intersection.argtypes = [C.c_char_p, C.c_char_p, C.c_char_p, C.c_char_p, C.POINTER(C.c_longlong)]
    L.kh_mask_allowed.restype = C.c_longlong
    L.kh_mask_allowed.argtypes = [C.c_char_p, C.c_char_p]
    L.kh_mask_compatible.argtypes = [C.c_char_p, C.c_char_p, C.c_int, C.c_char_p, C.c_char_p, C.c_int, C.c_int]
    L.ksched_device_count.restype = C.c_int
    L.ksched_abi_version.restype = C.c_int
    L.ksched_nccl_unique_id.argtypes = [C.c_void_p]
    L.ksched_nccl_init.argtypes = [C.c_void_p, C.c_void_p, C.c_int, C.c_int]
    L.ksched_set_shard.argtypes = [C.c_void_p, C.c_int, C.c_int]
    L.ksched_shard_range.argtypes = [C.c_int, C.c_int, C.c_int, C.POINTER(C.c_int), C.POINTER(C.c_int)]
    _lib = L
    return L


def device_count():
    n = lib().ksched_device_count()
    return max(n, 0)


def shard_range(n_words32, rank, world):
    """column words [begin, end) of the feasibility matrix that `rank` computes (SURVEY.md 8e)"""
    b, e = C.c_int(), C.c_int()
    rc = lib().ksched_shard_range(n_words32, rank, world, C.byref(b), C.byref(e))
    if rc != KSCHED_OK:
        raise KschedError(rc, "ksched_shard_range")
    return b.value, e.value


def set_shard(rank, world):
    """column shard of the process handle (ksched_set_shard): K1 computes only `rank`'s words of F and the pack kernel
    evaluates fresh nodes without F. (0, 1) computes every column."""
    _check(lib().kh_gpu_set_shard(rank, world))


def _check(rc):
    if rc != KSCHED_OK:
        raise KschedError(rc, lib().kh_scheduler_error().decode())


class Problem:
    """The inputs of NewScheduler + Solve (see host/model.h for the fields)."""

    def __init__(self, ptr):
        if not ptr:
            raise ValueError(model_lib().kh_last_error().decode())
        self.ptr = ptr

    @classmethod
    def from_dict(cls, d):
        return cls(model_lib().kh_problem_from_json(json.dumps(d).encode()))

    @classmethod
    def synth(cls, config, n_pods, n_types, seed=42, n_nodes=0):
        """BASELINE.json configurations C1..C5 (SURVEY.md 8d)."""
        return cls(model_lib().kh_problem_synth(config, n_pods, n_types, seed, n_nodes))

    def pod_summary(self):
        """[n_pods][6] int64: cpu milli, memory milli, app label id, self anti-affinity on hostname, zone spread skew, hostname spread skew"""
        n = self.counts()["pods"]
        out = np.zeros((max(n, 1), 6), dtype=np.int64)
        model_lib().kh_problem_pod_summary(self.ptr, out.ctypes.data_as(C.c_void_p))
        return out[:n]

    def counts(self):
        out = (C.c_longlong * 6)()
        model_lib().kh_problem_counts(self.ptr, out)
        return dict(zip(["pods", "instance_types", "provisioners", "nodes", "daemonset_pods", "bound_pods"], list(out)))

    def __del__(self):
        if getattr(self, "ptr", None) and _model is not None:
            _model.kh_problem_free(self.ptr)
            self.ptr = None


class Result:
    """([]*Node, []*ExistingNode) of Scheduler.Solve as flat data."""

    def __init__(self):
        self.ptr = model_lib().kh_result_new()

    def __del__(self):
        if getattr(self, "ptr", None) and _model is not None:
            _model.kh_result_free(self.ptr)
            self.ptr = None

    @property
    def error(self):
        return model_lib().kh_result_error(self.ptr).decode()

    @property
    def assign(self):
        n = model_lib().kh_result_num_pods(self.ptr)
        out = np.empty(n, dtype=np.int32)
        model_lib().kh_result_assign(self.ptr, out.ctypes.data)
        return out

    @property
    def relax_level(self):
        n = model_lib().kh_result_num_pods(self.ptr)
        out = np.empty(n, dtype=np.int32)
        model_lib().kh_result_relax(self.ptr, out.ctypes.data)
        return out

    @property
    def all_pods_scheduled(self):
        """simulateScheduling's allPodsScheduled (helpers.go:96-114): every pod was placed (GPU Solves and simulations)"""
        return bool(model_lib().kh_result_all_pods_scheduled(self.ptr))

    @property
    def uninitialized_existing(self):
        """an existing node of the result is not initialised: simulateScheduling then returns nil, false (helpers.go:104-110)"""
        return bool(model_lib().kh_result_uninitialized_existing(self.ptr))

    @property
    def num_new_nodes(self):
        return model_lib().kh_result_num_new_nodes(self.ptr)

    @property
    def num_existing(self):
        return model_lib().kh_result_num_existing(self.ptr)

    @property
    def nodes_visited(self):
        return model_lib().kh_result_nodes_visited(self.ptr)

    @property
    def add_calls(self):
        return model_lib().kh_result_add_calls(self.ptr)

    def new_node_info(self):
        """[n_new, 3] = (provisioner index in weight order, pod count, surviving instance-type options)"""
        n = self.num_new_nodes
        out = np.empty((n, 3), dtype=np.int32)
        model_lib().kh_result_new_node_info(self.ptr, out.ctypes.data)
        return out

    def new_node_options(self, i):
        cap = 1 << 16
        out = np.empty(cap, dtype=np.int32)
        n = model_lib().kh_result_new_node_options(self.ptr, i, out.ctypes.data, cap)
        return out[:n].copy()

    def digest(self):
        return model_lib().kh_result_digest(self.ptr)

    def to_dict(self, brief=False):
        """brief: per-node instance-type lists replaced by their length (full-size problems)"""
        fn = model_lib().kh_result_to_json_brief if brief else model_lib().kh_result_to_json
        need = fn(self.ptr, None, 0)
        buf = C.create_string_buffer(need)
        fn(self.ptr, buf, need)
        return json.loads(buf.value.decode())


def _cand_array(candidates):
    arr = (C.c_int * max(1, len(candidates)))(*candidates)
    return arr, len(candidates)


class Context:
    """A scheduler context: a device handle of its own (kh_context_create). Schedulers and sessions made with context=ctx
    run on it; two contexts can be used from two threads at once, and their kernels overlap on one device. One context is
    used by one thread at a time. Without a context, everything shares the process-wide handle, one call at a time."""

    def __init__(self, device=0):
        self.ptr = lib().kh_context_create(int(device))
        if not self.ptr:
            msg = lib().kh_scheduler_error().decode()
            raise KschedError(KSCHED_ERR_NO_DEVICE if "no usable CUDA device" in msg else KSCHED_ERR_INVALID, msg)
        self.device = int(device)
        self._sessions = weakref.WeakSet()  # open ClusterSessions on this context: destroy() refuses while there are any

    def handle(self):
        """the context's pointer for the C calls; refuses a destroyed context"""
        if not self.ptr:
            raise KschedError(KSCHED_ERR_INVALID, "the context has been destroyed")
        return self.ptr

    def timings(self):
        """ksched_get_timings of the context's handle, as a dict (pack_interval_ns: its last pack launch in device ns)"""
        t = Timings()
        _check(lib().kh_context_timings(self.handle(), C.byref(t)))
        return t.as_dict()

    def destroy(self):
        """frees the context's handle; refused while a session opened on it is still open (close it first)"""
        if getattr(self, "ptr", None) and any(s.ptr for s in self._sessions):
            raise KschedError(KSCHED_ERR_INVALID, "the context still has open sessions")
        if getattr(self, "ptr", None) and _lib is not None:
            _lib.kh_context_destroy(self.ptr)
        self.ptr = None

    def __del__(self):  # an open session keeps its context alive, so none is open here
        if getattr(self, "ptr", None) and _lib is not None:
            _lib.kh_context_destroy(self.ptr)
        self.ptr = None


class Scheduler:
    """scheduling.Scheduler: NewScheduler(...) then Solve(pods). GPU only. context: a Context to solve on (default: the
    process-wide handle)."""

    def __init__(self, problem: Problem, context: "Context | None" = None):
        self.problem = problem
        self.context = context

    def solve(self, candidates=(), count_visited=True):
        """count_visited=False is the production setting: the exact nodes_visited statistic is dropped and the pack
        kernel may use its steady-state paths (failure memo, class run, existing-node run)."""
        lib().kh_set_count_visited(int(count_visited))
        res = Result()
        arr, n = _cand_array(list(candidates))
        if self.context is None:
            rc = lib().kh_scheduler_solve(self.problem.ptr, arr, n, res.ptr)
        else:
            rc = lib().kh_context_solve(self.context.handle(), self.problem.ptr, arr, n, res.ptr)
        _check(rc)
        return res


def solve_timed(problem: Problem, candidates=(), count_visited=False):
    """Scheduler.solve with its host phases timed: (Result, {encode_us, catalog_us, solve_us, decode_us, total_us})."""
    lib().kh_set_count_visited(int(count_visited))
    res = Result()
    arr, n = _cand_array(list(candidates))
    ph = (C.c_double * 5)()
    _check(lib().kh_scheduler_solve_timed(problem.ptr, arr, n, res.ptr, ph))
    return res, dict(zip(["encode_us", "catalog_us", "solve_us", "decode_us", "total_us"], list(ph)))


def simulate_scheduling(problem: Problem, nodes_to_delete):
    """deprovisioning.simulateScheduling (helpers.go:42): re-run Solve with the candidates' pods added."""
    return Scheduler(problem).solve(candidates=nodes_to_delete)


class ClusterSession:
    """One consolidation pass over a cluster: the candidates ranked once, the cluster resident on the device once
    (ksched_load_cluster), every computeConsolidation one entry of a ksched_simulate_batch call."""
    OPTIONS_STRIDE = 2048

    def __init__(self, problem: Problem, context: "Context | None" = None):
        self.problem = problem
        self.context = context  # kept alive as long as the session
        res, n = C.c_int(), C.c_int()
        if context is None:
            self.ptr = lib().kh_cluster_open(problem.ptr, C.byref(res), C.byref(n))
        else:
            self.ptr = lib().kh_context_cluster_open(context.handle(), problem.ptr, C.byref(res), C.byref(n))
            if self.ptr:
                context._sessions.add(self)
        if not self.ptr:
            msg = lib().kh_scheduler_error().decode()
            raise KschedError(KSCHED_ERR_NO_DEVICE if "no usable CUDA device" in msg else KSCHED_ERR_INVALID, msg)
        self.resident = bool(res.value)
        self.n_candidates = n.value

    def candidate_nodes(self):
        arr = (C.c_int * max(1, self.n_candidates))()
        lib().kh_cluster_candidates(self.ptr, arr, self.n_candidates)
        return list(arr[:self.n_candidates])

    def probe_sets(self, sets, multi):
        """computeConsolidation for every candidate set (positions in the disruption order) in one device batch ->
        [(action, options)]"""
        if not sets:
            return []
        flat = [i for s_ in sets for i in s_]
        off = [0]
        for s_ in sets:
            off.append(off[-1] + len(s_))
        stride = self.OPTIONS_STRIDE
        actions = (C.c_int * len(sets))()
        nopt = (C.c_int * len(sets))()
        opts = (C.c_int * (stride * len(sets)))()
        _check(lib().kh_cluster_probe_sets(self.ptr, (C.c_int * max(1, len(flat)))(*flat), (C.c_int * len(off))(*off), len(sets), int(multi), actions, opts, stride,
                                           nopt))
        return [(int(actions[q]), list(opts[q * stride:q * stride + min(nopt[q], stride)])) for q in range(len(sets))]

    def simulate(self, sets):
        """simulateScheduling's whole result (helpers.go:42-115) for every set of node indices of the problem, in the order
        Expiration, Drift or computeConsolidation picked them, in one device call -> [Result], each what
        Scheduler(problem).solve(candidates=set) returns (nodes_visited aside: a simulation also counts the removed nodes it
        skips), with all_pods_scheduled and uninitialized_existing set. The nodes must be candidates of the session."""
        if not sets:
            return []
        flat = [int(i) for s_ in sets for i in s_]
        off = [0]
        for s_ in sets:
            off.append(off[-1] + len(s_))
        out = [Result() for _ in sets]
        ptrs = (C.c_void_p * len(sets))(*[r.ptr for r in out])
        _check(lib().kh_cluster_simulate(self.ptr, (C.c_int * max(1, len(flat)))(*flat), (C.c_int * len(off))(*off), len(sets), ptrs))
        return out

    def validate(self, after: Problem, commands):
        """Validation.IsValid (validation.go:63-172) of commands against `after`, the cluster when the TTL ends, in one device
        batch. commands = [(positions in the disruption order, action 1 or 2, options)], as probe_sets returns them -> [bool].
        The session keeps the snapshot of `after` until it closes or is handed a different problem."""
        if not commands:
            return []
        flat = [i for s_, _, _ in commands for i in s_]
        off = [0]
        for s_, _, _ in commands:
            off.append(off[-1] + len(s_))
        stride = max(1, max(len(o) for _, _, o in commands))
        opts = (C.c_int * (stride * len(commands)))()
        for q, (_, _, o) in enumerate(commands):
            opts[q * stride:q * stride + len(o)] = list(o)
        n = len(commands)
        valid = (C.c_int * n)()
        self._after = after   # the session's snapshot of `after` lives as long as the session or the next validate
        _check(lib().kh_cluster_validate(self.ptr, after.ptr, (C.c_int * max(1, len(flat)))(*flat), (C.c_int * len(off))(*off), n,
                                         (C.c_int * n)(*[a for _, a, _ in commands]), opts, stride, (C.c_int * n)(*[len(o) for _, _, o in commands]), valid))
        return [bool(v) for v in valid]

    def close(self):
        if getattr(self, "ptr", None) and _lib is not None:
            _lib.kh_cluster_close(self.ptr)
            self.ptr = None

    __del__ = close


def rank_candidates(problem: Problem, cap=65536):
    """deprovisioning candidates in disruption order (device kernels: costs, lifetime scaling, order) -> (node indices, costs)"""
    order = (C.c_int * cap)()
    cost = (C.c_double * cap)()
    n = lib().kh_rank_candidates(problem.ptr, order, cost, cap)
    if n < 0:
        _check(n)
    return list(order[:n]), list(cost[:n])


def nccl_allgather_i32(values, world):
    """one ncclAllGather of `values` (ints) on the scheduler handle's communicator -> [per-rank list]"""
    n = len(values)
    send = (C.c_int * max(1, n))(*values)
    recv = (C.c_int * max(1, n * world))()
    _check(lib().kh_allgather_i32(send, n, recv))
    return [list(recv[r * n:(r + 1) * n]) for r in range(world)]


class MultiNodeConsolidation:
    """context: the Context its session() opens on (default: the process-wide handle); the one-call searches below run on
    the process-wide handle."""

    def __init__(self, problem: Problem, context: "Context | None" = None):
        self.problem = problem
        self.context = context
        self._session = None

    def session(self):
        if self._session is None:
            self._session = ClusterSession(self.problem, context=self.context)
        return self._session

    def first_n_node_consolidation_option(self):
        out4 = (C.c_int * 4)()
        opts = (C.c_int * 8192)()
        probes = (C.c_int * 256)()
        acts = (C.c_int * 256)()
        npr = C.c_int()
        rc = lib().kh_consolidate(self.problem.ptr, out4, opts, 8192, probes, acts, 256, C.byref(npr))
        _check(rc)
        return {"action": out4[0], "nodes_removed": out4[1], "simulations": out4[2], "options": list(opts[:out4[3]]),
                "probes": list(probes[:npr.value]), "probe_actions": list(acts[:npr.value])}

    def compute_command(self, after: Problem):
        """MultiNodeConsolidation.ComputeCommand (multinodeconsolidation.go:41-70): the search, then Validation.IsValid of its
        command against `after`, the cluster when the TTL ends. A command that fails validation is retry (action 3).
        validations = the verdicts of the validations run (none when the search finds nothing)."""
        out4 = (C.c_int * 4)()
        opts = (C.c_int * 8192)()
        probes = (C.c_int * 256)()
        acts = (C.c_int * 256)()
        npr, verdict = C.c_int(), C.c_int()
        _check(lib().kh_consolidate_validated(self.problem.ptr, after.ptr, out4, opts, 8192, probes, acts, 256, C.byref(npr), C.byref(verdict)))
        return {"action": out4[0], "nodes_removed": out4[1], "simulations": out4[2], "options": list(opts[:out4[3]]),
                "probes": list(probes[:npr.value]), "probe_actions": list(acts[:npr.value]),
                "validations": [] if verdict.value < 0 else [bool(verdict.value)]}

    def candidates(self):
        return int(lib().kh_consolidate_candidates(self.problem.ptr))

    def probe(self, count):
        """computeConsolidation over the `count` cheapest candidates (one simulation on this rank's GPU, cluster resident)."""
        return self.session().probe_sets([list(range(int(count)))], True)[0]

    def first_n_node_consolidation_option_sharded(self, rank=0, world=1, all_gather=None):
        """The same binary search with its probes sharded over ranks (SURVEY section 8e: consolidation probes are
        independent simulations). Each round evaluates, in parallel, every probe the sequential search could reach within
        the next log2(world+1) steps and then replays the sequential decisions on the gathered outcomes, so the command
        is identical to first_n_node_consolidation_option for any world size. `all_gather(obj) -> [obj per rank]`
        (e.g. nccl_allgather_i32 on the verdicts; None = single process)."""
        n = self.candidates()

        def probe_many(counts):
            mine = {c: self.probe(c) for i, c in enumerate(counts) if i % world == rank}
            if all_gather is None or world == 1:
                return mine
            merged = {}
            for part in all_gather(mine):
                merged.update(part)
            return merged

        action, count, options, rounds, probes = speculative_binary_search(n, probe_many, world)
        return {"action": action, "nodes_removed": count, "options": options, "rounds": rounds, "probes": probes}


class SingleNodeConsolidation:
    """SingleNodeConsolidation.ComputeCommand (singlenodeconsolidation.go:43-84): the candidates in disruption order, the
    first whose computeConsolidation yields delete / replace wins. The simulations are independent: a rank sweeps its share
    `batch` simulations per device call."""

    def __init__(self, problem: Problem):
        self.problem = problem

    def compute_command(self, first=0, last=-1, batch=64, after=None):
        """after = the cluster when the TTL ends: each batch's actionable commands are validated against it in one more device
        call, the first valid one wins, and none after a failed validation is retry (action 3). The result then also carries
        "validations" = [(position, valid)] of what the sequential loop validates and "failed_validation"."""
        out4 = (C.c_int * 4)()
        node = C.c_int()
        opts = (C.c_int * 8192)()
        if after is None:
            _check(lib().kh_consolidate_single(self.problem.ptr, int(first), int(last), int(batch), out4, C.byref(node), opts, 8192))
            return {"action": out4[0], "position": out4[1], "simulations": out4[2], "node": node.value, "options": list(opts[:out4[3]])}
        cap = 1 << 16
        trace, valid = (C.c_int * cap)(), (C.c_int * cap)()
        ntr, failed = C.c_int(), C.c_int()
        _check(lib().kh_consolidate_single_validated(self.problem.ptr, after.ptr, int(first), int(last), int(batch), out4, C.byref(node), opts, 8192,
                                                     trace, valid, cap, C.byref(ntr), C.byref(failed)))
        return {"action": out4[0], "position": out4[1], "simulations": out4[2], "node": node.value, "options": list(opts[:out4[3]]),
                "validations": [(trace[i], bool(valid[i])) for i in range(min(ntr.value, cap))], "failed_validation": bool(failed.value)}


def merge_single_node_shares(shares):
    """SingleNodeConsolidation.ComputeCommand of a sweep split into shares [first, last) in order: the first share with a
    winner gives the command; the trace is every earlier share's trace and the winner's; with no winner the result is retry
    when any share failed a validation, else nothing."""
    trace = []
    for r in shares:
        trace += r["validations"]
        if r["action"] in (1, 2):
            return dict(r, validations=trace, failed_validation=any(not v for _, v in trace))
    failed = any(r["failed_validation"] for r in shares)
    return {"action": 3 if failed else 0, "position": -1, "node": -1, "options": [], "validations": trace, "failed_validation": failed}


def speculation_frontier(lo, hi, width):
    """Probe sizes (mid+1) of the binary-search decision tree rooted at [lo, hi], breadth first, at most `width` of them
    and always whole levels first (multinodeconsolidation.go:84-112 visits exactly one root-to-leaf path of this tree)."""
    out, level = [], [(lo, hi)]
    while level and len(out) < width:
        nxt = []
        for (a, b) in level:
            if a > b:
                continue
            mid = (a + b) // 2
            if len(out) < width:
                out.append(mid + 1)
            nxt.append((mid + 1, b))
            nxt.append((a, mid - 1))
        level = nxt
    return out


def speculative_binary_search(n_candidates, probe_many, width):
    """firstNNodeConsolidationOption (multinodeconsolidation.go:74-114) with `width` probes evaluated per round.
    probe_many(list of probe sizes) -> {size: (action, options)}. Returns (action, nodes_removed, options, rounds, probes):
    the decisions replayed are the sequential ones, so the answer does not depend on `width`."""
    if n_candidates < 2:
        return 0, 0, [], 0, []
    lo, hi = 1, n_candidates - 1
    last = (0, 0, [])
    rounds, path = 0, []
    while lo <= hi:
        known = probe_many(speculation_frontier(lo, hi, max(1, width)))
        rounds += 1
        while lo <= hi:
            mid = (lo + hi) // 2
            if mid + 1 not in known:
                break
            action, options = known[mid + 1]
            path.append(mid + 1)
            if action in (1, 2):
                last = (action, mid + 1, options)
                lo = mid + 1
            else:
                hi = mid - 1
    return last[0], last[1], last[2], rounds, path


class ResidentSolve:
    """Encode once, keep the problem in HBM, run the kernels repeatedly (bench / kernel tests)."""

    def __init__(self, problem: Problem, candidates=()):
        self.problem = problem
        arr, n = _cand_array(list(candidates))
        self.enc = lib().kh_encode(problem.ptr, arr, n)
        if not self.enc:
            msg = lib().kh_scheduler_error().decode()
            raise KschedError(KSCHED_ERR_UNSUPPORTED if msg.startswith("unsupported:") else KSCHED_ERR_INVALID, msg)
        d = (C.c_longlong * 20)()
        lib().kh_encoded_dims(self.enc, d)
        self.dims = dict(zip(["pods", "classes", "existing", "groups", "types", "templates", "keys", "resources", "type_words", "class_topo",
                              "taintsets", "resources_ext", "hostports", "hostport_ext_words", "hostname_reqs", "hostname_words",
                              "itype_reqs", "itype_filter_terms", "volume_claims", "volume_ext_words"], list(d)))
        self.dims["offering_slots"] = lib().kh_encoded_offering_slots(self.enc)

    def hostname_reqs(self):
        """every hostname requirement of this encoding in entry order, as (admits new nodes, [admitted existing slots])"""
        out, buf = [], (C.c_longlong * (self.dims["existing"] + 1))()
        for i in range(self.dims["hostname_reqs"]):
            n = lib().kh_encoded_hostname_req(self.enc, i, buf, len(buf))
            assert n >= 0, n
            out.append((bool(buf[0]), list(buf[1:n + 1])))
        return out

    def pod_class(self, i):
        """the initial class of pod i of Solve's pod list"""
        return lib().kh_encoded_pod_class(self.enc, i)

    def class_hostname_req(self, c):
        """the hostname_reqs entry of class c, or None without a hostname requirement"""
        i = lib().kh_encoded_class_hostname(self.enc, c)
        return None if i < 0 else i

    def group_total(self, g):
        """the initial count of topology group g summed over its domains (countDomains)"""
        return lib().kh_encoded_group_total(self.enc, g)

    def hostports(self):
        """the host-port entries of this encoding in id order, as (ip, port, protocol): the ones the encoder kept"""
        out, buf = [], C.create_string_buffer(256)
        while lib().kh_encoded_hostport(self.enc, len(out), buf, len(buf)) == 0:
            ip, port, proto = buf.value.decode().split(" ")
            out.append((ip, int(port), proto))
        return out

    def volume_claims(self):
        """the tracked volume claims of this encoding in id order, as (driver, claim)"""
        out, buf = [], C.create_string_buffer(1024)
        while lib().kh_encoded_volume_claim(self.enc, len(out), buf, len(buf)) == 0:
            driver, claim = buf.value.decode().split(" ", 1)
            out.append((driver, claim))
        return out

    def offering_slots(self):
        """the dense offering slots of this encoding in slot order, as (capacity type, zone); [] for the ct*16 + zone layout"""
        out, buf = [], C.create_string_buffer(1024)
        while lib().kh_encoded_offering_slot(self.enc, len(out), buf, len(buf)) == 0:
            ct, zone = buf.value.decode().split(" ", 1)
            out.append((ct, zone))
        return out

    def key_info(self, key):
        """dictionary of one mask key: {values, representatives (of unnamed value classes, 0 = none), thresholds}, or None
        when the key is not a mask key of this encoding"""
        out = (C.c_longlong * 3)()
        if lib().kh_encoded_key_info(self.enc, key.encode(), out) != 0:
            return None
        return dict(zip(["values", "representatives", "thresholds"], list(out)))

    def class_row(self, c):
        """the 32 u64 words of class c's pod row as the device receives it (include/ksched.h: ksched_pod_row)"""
        out = np.zeros(32, dtype=np.uint64)
        if lib().kh_encoded_class_row(self.enc, c, out.ctypes.data) != 0:
            raise IndexError(c)
        return out

    @staticmethod
    def k1_plan():
        """the process handle's last K1 class pass: {blocks, chunk (class rows per warp), cacheable, alloc_in_smem,
        tables_in_smem}"""
        out = (C.c_int * 5)()
        _check(lib().kh_gpu_k1_plan(out))
        return dict(zip(["blocks", "chunk", "cacheable", "alloc_in_smem", "tables_in_smem"], list(out)))

    RUN_REC_DTYPE = np.dtype([("ok", "<i4"), ("n_host", "<i4"), ("n_mask", "<i4"), ("h_row", "<i4", 4), ("h_group", "<i4", 4),
                              ("h_lim", "<i4", 4), ("m_group", "<i4", 2), ("m_skew", "<i4", 2), ("m_neutral", "<u4", 2),
                              ("m_tallow", "<u4", 2), ("m_dict", "<u4", 2), ("h_times", "u1", 4), ("m_key", "u1", 2),
                              ("m_self", "u1", 2), ("m_rec", "u1", 2), ("m_wk", "u1", 2), ("pad", "<u4", 4)])

    def run_records(self):
        """the class runs' relation tables of this problem's last run(): one record per class (csrc/pack_state.cuh: RunRec)
        as a structured array, or None when that Solve built none (class runs could not run)"""
        out = np.zeros(max(self.dims["classes"], 1), dtype=self.RUN_REC_DTYPE)
        n = lib().kh_gpu_run_records(out.ctypes.data, self.dims["classes"])
        _check(min(n, 0))
        return out[:self.dims["classes"]] if n > 0 else None

    def resource_id(self, name):
        """id of a resource in this encoding: a row slot below 8, an ext resource from 8 on; -1 when it is not carried"""
        return lib().kh_encoded_resource_id(self.enc, name.encode())

    def set_count_visited(self, on):
        """exact nodes_visited statistic on/off (off for timed runs: it costs a pass over all in-flight nodes per pod)"""
        lib().kh_encoded_set_count_visited(self.enc, int(on))

    def load(self):
        _check(lib().kh_gpu_load(self.enc))

    def load_catalog(self):
        _check(lib().kh_gpu_load_catalog(self.enc))

    def solve_e2e(self, want_result=False):
        """ksched_solve with host buffers: upload + kernels + download. Returns (wall microseconds, Result|None)."""
        us = C.c_double()
        res = Result() if want_result else None
        _check(lib().kh_gpu_solve_e2e(self.enc, res.ptr if res else None, C.byref(us)))
        return us.value, res

    def run(self, flush_l2=False):
        _check(lib().kh_gpu_run(int(flush_l2)))

    def run_feasibility(self, flush_l2=False):
        us = C.c_float()
        _check(lib().kh_gpu_run_feasibility(int(flush_l2), C.byref(us)))
        return us.value

    def download(self, want_feasibility=False):
        res = Result()
        feas = best = None
        fptr = bptr = None
        if want_feasibility:
            d = self.dims
            feas = np.zeros((d["pods"], d["templates"], d["type_words"]), dtype=np.uint64)
            best = np.zeros(d["pods"], dtype=np.uint64)
            fptr, bptr = feas.ctypes.data, best.ctypes.data
        _check(lib().kh_gpu_download(self.enc, res.ptr, fptr, bptr))
        return (res, feas, best) if want_feasibility else res

    def timings(self):
        t = Timings()
        lib().kh_gpu_timings(C.byref(t))
        return t.as_dict()

    def __del__(self):
        if getattr(self, "enc", None) and _lib is not None:
            _lib.kh_encoded_free(self.enc)
            self.enc = None
