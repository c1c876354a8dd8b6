"""The GPU path's Solve against the oracle's, field by field: shared by the GPU differential tests (test_gpu_parity,
test_gpu_fuzz, test_gpu_runs)."""
import pytest

INSTANCE_TYPE = "node.kubernetes.io/instance-type"


def compare(pkg, oracle, problem, candidates=(), add_calls=True, refusal_skips=False):
    """Solve on the GPU twice (nodes_visited counted, then the production setting without it) and compare with the oracle:
    assignment, relaxation levels, existing nodes, every new node (provisioner, pods in Add order, surviving instance-type
    options, requests, final requirements, launch choice) and nodes_visited. refusal_skips: a KSCHED_ERR_UNSUPPORTED
    refusal skips the test instead of failing it (random problems may leave the supported envelope)."""
    want = pkg.Result()
    assert oracle.solve(problem, want, candidates) == 0, want.error
    try:
        got = pkg.Scheduler(problem).solve(candidates)
    except pkg.KschedError as e:
        if refusal_skips and e.code == pkg.KSCHED_ERR_UNSUPPORTED:
            pytest.skip(f"refused loudly: {e}")
        raise
    w, g = want.to_dict(), got.to_dict()
    assert g["assign"] == w["assign"]
    assert g["relax"] == w["relax"]
    assert g["existing"] == w["existing"]
    assert len(g["newNodes"]) == len(w["newNodes"])
    for i, (a, b) in enumerate(zip(g["newNodes"], w["newNodes"])):
        assert a["provisioner"] == b["provisioner"], i
        assert a["pods"] == b["pods"], i
        assert a["options"] == b["options"], i
        assert a["requests"] == b["requests"], i
        assert a["requirements"] == {k: v for k, v in b["requirements"].items() if k != INSTANCE_TYPE}, i
        assert a.get("launch") == b.get("launch") and a.get("launch") is not None, i  # launch choice (device kernel vs oracle)
    assert got.nodes_visited == want.nodes_visited
    if add_calls:
        assert got.add_calls == want.add_calls
    # production setting (no nodes_visited statistic): the steady-state kernel paths must give the identical result
    f = pkg.Scheduler(problem).solve(candidates, count_visited=False).to_dict()
    assert f["assign"] == w["assign"] and f["relax"] == w["relax"] and f["existing"] == w["existing"]
    assert f["newNodes"] == g["newNodes"]
    return got, want
