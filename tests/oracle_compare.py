"""The GPU path's Solve, consolidation and validation against the oracles', field by field, and the pack kernel's mode
switches: shared by the GPU differential tests (test_gpu_parity, test_gpu_fuzz, test_gpu_runs, test_gpu_cluster, ...)."""
import pytest

import validation_oracle as vo

INSTANCE_TYPE = "node.kubernetes.io/instance-type"

# Each switch turns off one closed-form mode of the pack kernel, the class-run loop or one of its steps (read per Solve,
# csrc/ksched.cu): the per-pod loop or the generic step then places the same pods one at a time, with the same result.
MODE_SWITCHES = ("KSCHED_NO_CLASSRUN", "KSCHED_NO_LEVELRUN", "KSCHED_NO_LEVELWARP", "KSCHED_NO_MASKRUN", "KSCHED_NO_VARSTORE",
                 "KSCHED_NO_ROUNDSTRETCH")


def set_modes(monkeypatch, *specs):
    """Clear every mode switch and KSCHED_PACK_THREADS, then set the variables the specs name: each spec is a comma-separated
    list of NAME (set to 1) or NAME=value; empty specs set nothing."""
    for v in MODE_SWITCHES + ("KSCHED_PACK_THREADS",):
        monkeypatch.delenv(v, raising=False)
    for spec in specs:
        for kv in (spec or "").split(","):
            if kv:
                k, _, v = kv.partition("=")
                monkeypatch.setenv(k, v or "1")


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


def compare_probes(pkg, oracle, problem, cs, prefixes, singles):
    """The session's batched simulations against the oracle: each prefix set (the cheapest candidates, multi-node) is
    computeConsolidation over that many candidates, each single set is single-node consolidation of that candidate."""
    for s_, g in zip(prefixes, cs.probe_sets(prefixes, True)):
        assert g == oracle.consolidate_probe(problem, len(s_)), ("prefix", len(s_))
    for s_, g in zip(singles, cs.probe_sets(singles, False)):
        w = oracle.consolidate_single(problem, s_[0])
        assert g == (w["action"], w["options"]), ("single", s_)


def compare_searches(pkg, oracle, problem):
    """The multi-node binary search (command and probe trace) and the single-node sweep against the oracle."""
    got = pkg.MultiNodeConsolidation(problem).first_n_node_consolidation_option()
    want = oracle.consolidate(problem)
    keys = ("action", "nodes_removed", "options", "probes", "probe_actions")
    assert {k: got[k] for k in keys} == {k: want[k] for k in keys}
    got = pkg.SingleNodeConsolidation(problem).compute_command()
    want = oracle.consolidate_single(problem)
    keys = ("action", "node", "options")
    assert {k: got[k] for k in keys} == {k: want[k] for k in keys}


def compare_cluster(pkg, oracle, problem, min_candidates=2):
    """The device-resident consolidation session of a cluster probe for probe (every prefix, every single candidate) and
    both searches against the oracle; returns the session."""
    cs = pkg.ClusterSession(problem)
    assert cs.resident
    n = cs.n_candidates
    assert n >= min_candidates
    compare_probes(pkg, oracle, problem, cs, [list(range(c)) for c in range(1, n + 1)], [[i] for i in range(n)])
    compare_searches(pkg, oracle, problem)
    return cs


VALIDATION_KEYS = ("action", "position", "node", "options", "validations", "failed_validation")
MULTI_VALIDATION_KEYS = ("action", "nodes_removed", "options", "probes", "probe_actions", "validations")


def compare_validation(pkg, before_dict, after_dict, label=None):
    """Both consolidations of `before_dict` validated against the cluster after the TTL, `after_dict`, against the
    validation oracle: single-node at batch 1 and 64, then multi-node. Returns the device's (single, multi) commands."""
    before = (before_dict, pkg.Problem.from_dict(before_dict))
    after = (after_dict, pkg.Problem.from_dict(after_dict))
    want = vo.single_compute_command(before, after)
    for batch in (1, 64):
        got = pkg.SingleNodeConsolidation(before[1]).compute_command(batch=batch, after=after[1])
        assert {k: got[k] for k in VALIDATION_KEYS} == {k: want[k] for k in VALIDATION_KEYS}, (label, batch)
    got_m = pkg.MultiNodeConsolidation(before[1]).compute_command(after[1])
    want_m = vo.multi_compute_command(before, after)
    assert {k: got_m[k] for k in MULTI_VALIDATION_KEYS} == {k: want_m[k] for k in MULTI_VALIDATION_KEYS}, label
    return got, got_m
