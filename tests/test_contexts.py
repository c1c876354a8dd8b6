"""Scheduler contexts without a device: creating one fails with KSCHED_ERR_NO_DEVICE (there is no CPU path), and the
Python wrappers refuse a destroyed context before anything reaches the library."""
import ctypes as C

import pytest


def test_context_create_without_device_fails(pkg):
    if pkg.device_count() > 0:
        pytest.skip("a CUDA device is visible")
    assert not pkg.lib().kh_context_create(0)
    with pytest.raises(pkg.KschedError) as e:
        pkg.Context()
    assert e.value.code == pkg.KSCHED_ERR_NO_DEVICE


def test_null_context_is_refused(pkg):
    problem = pkg.Problem.synth(1, 10, 4, 42, 0)
    res = pkg.Result()
    arr = (C.c_int * 1)()
    assert pkg.lib().kh_context_solve(None, problem.ptr, arr, 0, res.ptr) == pkg.KSCHED_ERR_INVALID
    assert not pkg.lib().kh_context_cluster_open(None, problem.ptr, None, None)


def test_destroyed_context_is_refused(pkg):
    ctx = object.__new__(pkg.Context)  # what destroy() leaves behind, without needing a device to create one
    ctx.ptr = None
    problem = pkg.Problem.synth(1, 10, 4, 42, 0)
    with pytest.raises(pkg.KschedError):
        pkg.Scheduler(problem, context=ctx).solve()
    with pytest.raises(pkg.KschedError):
        pkg.ClusterSession(problem, context=ctx)
    with pytest.raises(pkg.KschedError):
        ctx.timings()
    ctx.destroy()  # a second destroy is a no-op
