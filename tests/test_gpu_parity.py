"""GPU parity: the CUDA path (through the C-ABI / host facade) against the CPU oracle, bit-exact.

Compared per problem: the pod->node assignment vector, relaxation levels, and for every new node its
provisioner, pods in Add order, surviving instance-type options, requests and final requirements."""
import pytest

from oracle_compare import compare

pytestmark = pytest.mark.gpu

SMALL = [
    # (config, pods, types, nodes, seed)
    (1, 100, 10, 0, 42),
    (2, 1000, 500, 0, 42),
    (2, 3000, 500, 0, 7),
    (2, 10000, 500, 0, 42),
    (2, 6000, 40, 0, 5),
    (3, 1500, 1000, 0, 42),
    (3, 1000, 1000, 0, 3),
    (4, 1500, 1000, 0, 42),
    (4, 1000, 1000, 0, 11),
]


@pytest.mark.parametrize("config,pods,types,nodes,seed", SMALL)
def test_synthetic_configs_match_oracle(pkg, oracle, config, pods, types, nodes, seed):
    problem = pkg.Problem.synth(config, pods, types, seed, nodes)
    compare(pkg, oracle, problem)


def test_simulation_with_candidates_matches_oracle(pkg, oracle):
    problem = pkg.Problem.synth(5, 600, 1000, 42, 60)
    for cands in ([0], [3, 4, 5], list(range(10))):
        compare(pkg, oracle, problem, cands)


def test_multi_node_consolidation_matches_oracle(pkg, oracle):
    problem = pkg.Problem.synth(5, 400, 1000, 42, 40)
    want = oracle.consolidate(problem)
    got = pkg.MultiNodeConsolidation(problem).first_n_node_consolidation_option()
    assert got == want


@pytest.mark.parametrize("width", [1, 3, 7])
def test_sharded_consolidation_search_matches_oracle(pkg, oracle, width):
    """Probes evaluated `width` at a time (what `width` ranks would do) give the oracle's sequential command."""
    problem = pkg.Problem.synth(5, 400, 1000, 43, 40)
    want = oracle.consolidate(problem)
    mnc = pkg.MultiNodeConsolidation(problem)
    assert mnc.candidates() == 40
    seen = []

    def probe_many(counts):
        seen.append(list(counts))
        return {c: mnc.probe(c) for c in counts}

    action, count, options, rounds, path = pkg.speculative_binary_search(mnc.candidates(), probe_many, width)
    assert (action, count, options) == (want["action"], want["nodes_removed"], want["options"])
    assert path == want["probes"]
    assert rounds <= len(want["probes"])
    single = mnc.first_n_node_consolidation_option_sharded()
    assert (single["action"], single["nodes_removed"], single["options"]) == (want["action"], want["nodes_removed"], want["options"])


def test_feasibility_matrix_matches_fresh_node_options(pkg, oracle):
    """K1: F[p, v, :] must equal the option set of a fresh node of template v that holds only pod p
    (Node.Add on a new node, node.go:62-107) — checked for every (pod, provisioner) pair against the oracle."""
    import copy
    from fuzz_problems import random_problem
    checked = 0
    for seed in range(60):
        prob = random_problem(seed)
        prob["nodes"] = []
        prob["daemonSetPods"] = []
        for pr in prob["provisioners"]:
            pr.pop("limits", None)
        for pd in prob["pods"]:
            for k in ("topologySpreadConstraints", "podAntiAffinity", "podAffinity"):
                pd.pop(k, None)
        # weight order is the template order of the kernel
        order = sorted(range(len(prob["provisioners"])), key=lambda i: -prob["provisioners"][i].get("weight", 0))
        problem = pkg.Problem.from_dict(prob)
        rs = pkg.ResidentSolve(problem)
        rs.load()
        rs.run()
        _, feas, best = rs.download(want_feasibility=True)
        n_types = len(prob["instanceTypes"])
        for p_i, pd in enumerate(prob["pods"]):
            for v, prov_i in enumerate(order):
                single = copy.deepcopy(prob)
                single["pods"] = [pd]
                single["provisioners"] = [prob["provisioners"][prov_i]]
                want = pkg.Result()
                assert oracle.solve(pkg.Problem.from_dict(single), want) == 0, want.error
                w = want.to_dict()
                # relaxation changes the pod: K1's row describes the unrelaxed pod only
                expect = w["newNodes"][0]["options"] if (w["assign"][0] >= 0 and w["relax"][0] == 0) else None
                got = [i for i in range(n_types) if (int(feas[p_i][v][i // 64]) >> (i % 64)) & 1]
                if expect is None:
                    if w["relax"][0] == 0:
                        assert got == [], (seed, p_i, v)
                else:
                    assert got == expect, (seed, p_i, v)
                checked += 1
            any_col = any(int(x) for x in feas[p_i].ravel())
            assert (int(best[p_i]) != 2 ** 64 - 1) == any_col
    assert checked > 1500


def test_two_handles_on_one_device_solve_concurrently(pkg, oracle):
    """The pack kernel's parameters live in one __constant__ block per device: two handles driven by two host threads must
    still each reproduce their own result (device-side ordering in run_pack)."""
    a = pkg.Problem.synth(4, 1500, 1000, 5, 0)
    b = pkg.Problem.synth(3, 2000, 1000, 6, 0)
    assert pkg.lib().kh_selftest_two_handles(a.ptr, b.ptr, 6) == 0
    # and the singleton handle still agrees with the oracle afterwards
    compare(pkg, oracle, a, [])


from consolidation_answers import CASES as _CONS, CPU_ONLY_CASES as _CONS_LATE

CONSOLIDATION_CASES = _CONS + _CONS_LATE


@pytest.mark.parametrize("name,ref,build", CONSOLIDATION_CASES, ids=[c[0] for c in CONSOLIDATION_CASES])
def test_consolidation_known_answers_match_oracle(pkg, oracle, name, ref, build):
    """deprovisioning/suite_test.go cases: the product's probe / search must satisfy the same checks AND equal the oracle"""
    prob, check = build()
    problem = pkg.Problem.from_dict(prob)
    mnc = pkg.MultiNodeConsolidation(problem)

    def search():
        out = mnc.first_n_node_consolidation_option()
        want = oracle.consolidate(problem)
        assert (out["action"], out["nodes_removed"], out["options"], out["probes"]) == (want["action"], want["nodes_removed"], want["options"], want["probes"])
        return out

    def probe(count):
        got = mnc.probe(count)
        assert got == oracle.consolidate_probe(problem, count)
        return got

    check(probe, search)


CLASS_RUN_SWITCHES = ("KSCHED_NO_LEVELWARP", "KSCHED_NO_MASKRUN", "KSCHED_NO_LEVELRUN", "KSCHED_NO_CLASSRUN", "KSCHED_NO_LEVELSTEP", "KSCHED_WARPLOOP")


@pytest.mark.parametrize("config,pods,types,seed", [(4, 6000, 1000, 7), (4, 2500, 1000, 3), (3, 5000, 1000, 7), (2, 3000, 500, 7), (2, 4000, 40, 9)])
def test_class_run_modes_agree(pkg, monkeypatch, config, pods, types, seed):
    """The closed-form steps of the class-run loop (level / fill steps and fresh nodes in bulk, their one-warp form, the mask
    run with its rounds) are exact: with each of them switched off (KSCHED_NO_*: the per-pod loop or the generic step then
    places the same pods one at a time) the whole result is the same, bit for bit (scheduler.go:174-219 is one pod at a
    time; DESIGN.md section 4 says why several at once give the same answer)."""
    problem = pkg.Problem.synth(config, pods, types, seed, 0)
    rs = pkg.ResidentSolve(problem)
    rs.set_count_visited(False)
    rs.load()
    digests = {}
    for off in ("", "KSCHED_NO_LEVELWARP", "KSCHED_NO_MASKRUN", "KSCHED_NO_LEVELRUN,KSCHED_NO_MASKRUN", "KSCHED_NO_CLASSRUN", "KSCHED_NO_LEVELSTEP",
                "KSCHED_WARPLOOP"):
        for v in CLASS_RUN_SWITCHES:
            monkeypatch.delenv(v, raising=False)
        for v in off.split(","):
            if v:
                monkeypatch.setenv(v, "1")
        rs.run()
        res = rs.download()
        digests[off or "all on"] = (int(res.digest()), int(res.num_new_nodes), int((res.assign >= 0).sum()))
    for v in CLASS_RUN_SWITCHES:
        monkeypatch.delenv(v, raising=False)
    assert len(set(digests.values())) == 1, digests
