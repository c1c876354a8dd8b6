"""ctypes access to the CPU oracle (oracle/_build/liboracle.so) — test infrastructure only."""
import ctypes as C
import subprocess
from pathlib import Path

ROOT = Path(__file__).resolve().parent.parent
_lib = None


class Oracle:
    def __init__(self, lib):
        self.lib = lib
        lib.oracle_req_render.argtypes = [C.c_char_p, C.c_char_p, C.c_int]
        lib.oracle_req_intersection.argtypes = [C.c_char_p, C.c_char_p, C.c_char_p, C.c_int]
        lib.oracle_req_has.argtypes = [C.c_char_p, C.c_char_p]
        lib.oracle_req_operator.argtypes = [C.c_char_p]
        lib.oracle_req_len.argtypes = [C.c_char_p]
        lib.oracle_req_len.restype = C.c_longlong
        lib.oracle_req_string.argtypes = [C.c_char_p, C.c_char_p, C.c_char_p, C.c_int]
        lib.oracle_reqs_compatible.argtypes = [C.c_char_p, C.c_char_p, C.c_char_p, C.c_int]
        lib.oracle_normalize_key.argtypes = [C.c_char_p, C.c_char_p, C.c_int]
        lib.oracle_solve.argtypes = [C.c_void_p, C.POINTER(C.c_int), C.c_int, C.c_void_p]
        lib.oracle_consolidate_probe.argtypes = [C.c_void_p, C.c_int, C.POINTER(C.c_int), C.c_int, C.POINTER(C.c_int), C.c_char_p, C.c_int]
        lib.oracle_consolidate.argtypes = [C.c_void_p, C.POINTER(C.c_int), C.POINTER(C.c_int), C.POINTER(C.c_int), C.c_int,
                                           C.POINTER(C.c_int), C.POINTER(C.c_int), C.POINTER(C.c_int), C.c_int,
                                           C.POINTER(C.c_int), C.c_char_p, C.c_int]

        lib.oracle_consolidate_single.argtypes = [C.c_void_p, C.c_int, C.POINTER(C.c_int), C.POINTER(C.c_int), C.c_int, C.POINTER(C.c_int),
                                                  C.POINTER(C.c_int), C.c_char_p, C.c_int]
        lib.oracle_rank_candidates.argtypes = [C.c_void_p, C.POINTER(C.c_int), C.POINTER(C.c_double), C.c_int]

    def consolidate_single(self, problem, only_candidate=-1):
        """SingleNodeConsolidation.ComputeCommand -> {action, node, options, simulations}; only_candidate = one position"""
        node, nopt, npr = C.c_int(), C.c_int(), C.c_int()
        opts = (C.c_int * 8192)()
        err = C.create_string_buffer(1024)
        action = self.lib.oracle_consolidate_single(problem.ptr, int(only_candidate), C.byref(node), opts, 8192, C.byref(nopt), C.byref(npr), err, 1024)
        if action < 0:
            raise RuntimeError(err.value.decode())
        return {"action": action, "node": node.value, "options": list(opts[:nopt.value]), "simulations": npr.value}

    def rank_candidates(self, problem, cap=65536):
        order = (C.c_int * cap)()
        cost = (C.c_double * cap)()
        n = self.lib.oracle_rank_candidates(problem.ptr, order, cost, cap)
        return list(order[:n]), list(cost[:n])

    def _s(self, fn, *args):
        buf = C.create_string_buffer(4096)
        n = fn(*[a.encode() if isinstance(a, str) else a for a in args], buf, 4096)
        assert n >= 0
        return buf.value.decode()

    def intersection(self, a, b):
        return self._s(self.lib.oracle_req_intersection, a, b)

    def render(self, a):
        return self._s(self.lib.oracle_req_render, a)

    def has(self, a, v):
        return bool(self.lib.oracle_req_has(a.encode(), v.encode()))

    def operator(self, a):
        return ["In", "NotIn", "Exists", "DoesNotExist", "Gt", "Lt"][self.lib.oracle_req_operator(a.encode())]

    def length(self, a):
        return self.lib.oracle_req_len(a.encode())

    def string(self, a, b=""):
        return self._s(self.lib.oracle_req_string, a, b)

    def compatible(self, key, a, b, well_known=True):
        return bool(self.lib.oracle_reqs_compatible(key.encode(), a.encode(), b.encode(), int(well_known)))

    def normalize(self, k):
        return self._s(self.lib.oracle_normalize_key, k)

    def solve(self, problem, result, candidates=()):
        arr = (C.c_int * max(1, len(candidates)))(*candidates)
        rc = self.lib.oracle_solve(problem.ptr, arr, len(candidates), result.ptr)
        return rc

    def solve_dict(self, pkg, prob, candidates=(), fast=False):
        """Solve a problem dict, in fast mode if asked (the literal path again afterwards) -> (problem, result)"""
        problem = pkg.Problem.from_dict(prob)
        res = pkg.Result()
        self.lib.oracle_set_fast(int(fast))
        try:
            assert self.solve(problem, res, candidates) == 0, res.error
        finally:
            self.lib.oracle_set_fast(0)
        return problem, res

    def assert_fast_equals_literal(self, pkg, prob):
        """Fast mode's shortcuts are result-neutral on this problem: digest and whole result -> (literal, fast) results"""
        literal, fast = (self.solve_dict(pkg, prob, fast=f)[1] for f in (False, True))
        assert fast.digest() == literal.digest() and fast.to_dict() == literal.to_dict()
        return literal, fast

    def consolidate_probe(self, problem, count):
        """computeConsolidation over the `count` cheapest candidates -> (action, options)"""
        nopt = C.c_int()
        opts = (C.c_int * 8192)()
        err = C.create_string_buffer(1024)
        action = self.lib.oracle_consolidate_probe(problem.ptr, int(count), opts, 8192, C.byref(nopt), err, 1024)
        if action < 0:
            raise RuntimeError(err.value.decode())
        return action, list(opts[:nopt.value])

    def consolidate(self, problem):
        nr, sims, nopt, npr = C.c_int(), C.c_int(), C.c_int(), C.c_int()
        opts = (C.c_int * 8192)()
        probes = (C.c_int * 256)()
        acts = (C.c_int * 256)()
        err = C.create_string_buffer(1024)
        action = self.lib.oracle_consolidate(problem.ptr, C.byref(nr), C.byref(sims), opts, 8192, C.byref(nopt), probes, acts, 256,
                                             C.byref(npr), err, 1024)
        if action < 0:
            raise RuntimeError(err.value.decode())
        return {"action": action, "nodes_removed": nr.value, "simulations": sims.value,
                "options": list(opts[:nopt.value]), "probes": list(probes[:npr.value]), "probe_actions": list(acts[:npr.value])}


def load():
    global _lib
    if _lib is None:
        so = ROOT / "oracle" / "_build" / "liboracle.so"
        if not so.exists():
            subprocess.check_call(["make", "-C", str(ROOT / "oracle")])
        _lib = Oracle(C.CDLL(str(so)))
    return _lib
