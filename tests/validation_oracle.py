"""ctypes access to the validation oracle (oracle/validation.cc -> oracle/_build/libvalidation_oracle.so, linked to
liboracle.so) - test infrastructure only. `before` / `after` are (dict, Problem) pairs, as the tests build them; only the
Problem crosses into the oracle. Actions: 0 nothing, 1 delete, 2 replace, 3 retry."""
import ctypes as C
import subprocess

import oracle_lib

_lib = None


def lib():
    global _lib
    if _lib is None:
        oracle_lib.load()   # builds liboracle.so when missing
        so = oracle_lib.ROOT / "oracle" / "_build" / "libvalidation_oracle.so"
        if not so.exists():
            subprocess.check_call(["make", "-C", str(oracle_lib.ROOT / "oracle"), "-f", "validation.mk"])
        L = C.CDLL(str(so))
        P = C.POINTER(C.c_int)
        L.oracle_is_valid.argtypes = [C.c_void_p, C.c_void_p, P, C.c_int, C.c_int, P, C.c_int, C.c_char_p, C.c_int]
        L.oracle_single_compute_command.argtypes = [C.c_void_p, C.c_void_p, C.c_int, C.c_int, P, P, C.c_int, P, P, P, C.c_int, P, P, C.c_char_p, C.c_int]
        L.oracle_multi_compute_command.argtypes = [C.c_void_p, C.c_void_p, P, P, C.c_int, P, P, P, C.c_int, P, P, C.c_char_p, C.c_int]
        _lib = L
    return _lib


def _ints(xs):
    return (C.c_int * max(1, len(xs)))(*xs)


def is_valid(before, after, nodes, action, options):
    """Validation.IsValid of the command removing before's nodes (Problem.nodes indices), action 1 / 2, options (before's
    instance-type indices), against after"""
    err = C.create_string_buffer(1024)
    rc = lib().oracle_is_valid(before[1].ptr, after[1].ptr, _ints(nodes), len(nodes), int(action), _ints(options), len(options), err, 1024)
    if rc < 0:
        raise RuntimeError(err.value.decode())
    return bool(rc)


def single_compute_command(before, after, first=0, last=-1):
    """SingleNodeConsolidation.ComputeCommand over positions [first, last): validations = [(position, valid)]"""
    out3, nopt, ntr, failed = (C.c_int * 3)(), C.c_int(), C.c_int(), C.c_int()
    opts, cap = (C.c_int * 8192)(), 1 << 16
    trace, valid = (C.c_int * cap)(), (C.c_int * cap)()
    err = C.create_string_buffer(1024)
    if lib().oracle_single_compute_command(before[1].ptr, after[1].ptr, int(first), int(last), out3, opts, 8192, C.byref(nopt), trace, valid, cap,
                                           C.byref(ntr), C.byref(failed), err, 1024) < 0:
        raise RuntimeError(err.value.decode())
    return {"action": out3[0], "position": out3[1], "node": out3[2], "options": list(opts[:nopt.value]),
            "validations": [(trace[i], bool(valid[i])) for i in range(ntr.value)], "failed_validation": bool(failed.value)}


def multi_compute_command(before, after):
    """MultiNodeConsolidation.ComputeCommand: the search's fields plus validations = [valid] (empty: nothing to validate)"""
    out3, nopt, npr, verdict = (C.c_int * 3)(), C.c_int(), C.c_int(), C.c_int()
    opts, probes, acts = (C.c_int * 8192)(), (C.c_int * 256)(), (C.c_int * 256)()
    err = C.create_string_buffer(1024)
    if lib().oracle_multi_compute_command(before[1].ptr, after[1].ptr, out3, opts, 8192, C.byref(nopt), probes, acts, 256, C.byref(npr),
                                          C.byref(verdict), err, 1024) < 0:
        raise RuntimeError(err.value.decode())
    return {"action": out3[0], "nodes_removed": out3[1], "simulations": out3[2], "options": list(opts[:nopt.value]),
            "probes": list(probes[:npr.value]), "probe_actions": list(acts[:npr.value]),
            "validations": [] if verdict.value < 0 else [bool(verdict.value)]}
