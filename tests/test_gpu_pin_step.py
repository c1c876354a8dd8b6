"""GPU: the mask run's pin step (csrc/pack_kernel.cuh, DESIGN.md section 4) against the oracle. A zone-spread run meets
nodes an earlier class opened without pinning them to a zone; the pin step places pods on the next of them, one each, in
bulk. Each scenario ends its stretches by a different rule: the end of the staged entries, of the unpinned nodes or of the
32 lanes; an unpinned node with another pod count; an unpinned node behind a pinned head; a pod whose domain cannot be
pinned without narrowing the node's instance types. Spreads with max skew 1 and 2, and one whose selector does not match
its own pods (the domain counts stay), cover run_pick's order."""
import random

import pytest

import fixtures as fx
import run_problems as rp
from fixtures import HOSTNAME, ZONE
from oracle_compare import compare

pytestmark = pytest.mark.gpu

TINY = {"cpu": "50m", "memory": "64Mi"}


def _spread(app, seed):
    """zone spread of `app` pods: self-selecting with skew 1 or 2, or (seed 2) counting the pods of another deployment"""
    if seed % 3 == 2:
        return {"labels": {"app": app}, "topologySpreadConstraints": [fx.spread(ZONE, {"app": "other"})]}
    return rp.zone_spread(app, skew=1 + seed % 2)


def one_pod_nodes(seed):
    """an anti-affinity run opens one-pod nodes in no particular zone; zone-spread runs of 33-250 pods follow"""
    rng = random.Random(seed)
    zs = rp.zone_names(3, "eu-south")
    its = rp.zonal_types(zs, [(2, 4), (8, 32)])
    r = rp.Runs("one")
    r.run("other", 7, {"cpu": "1500m", "memory": "1Gi"}, **rp.zone_spread("other"))
    r.run("anti", rng.choice([40, 70, 129]), {"cpu": "1", "memory": "1Gi"}, labels={"app": "anti"},
          podAntiAffinity={"required": [fx.affinity_term(HOSTNAME, {"app": "anti"})]})
    r.run("spread", rng.choice([33, 129, 250]), TINY, **_spread("spread", seed))
    return fx.problem(r.pods, instance_types=its, provisioners=[rp.unlimited()])


def mixed_counts(seed):
    """a plain run after the anti-affinity run gives some of its nodes a second pod: the unpinned list holds nodes with one
    pod, then nodes with two"""
    rng = random.Random(seed)
    zs = rp.zone_names(4, "ap-east")
    its = rp.zonal_types(zs, [(2, 4), (8, 32)])
    r = rp.Runs("mix")
    r.run("other", 5, {"cpu": "1500m", "memory": "1Gi"}, **rp.zone_spread("other"))
    r.run("anti", rng.choice([40, 60]), {"cpu": "1", "memory": "1Gi"}, labels={"app": "anti"},
          podAntiAffinity={"required": [fx.affinity_term(HOSTNAME, {"app": "anti"})]})
    r.run("plain", rng.choice([9, 15, 21]), {"cpu": "200m", "memory": "256Mi"}, labels={"app": "plain"})
    r.run("spread", rng.choice([129, 250]), TINY, **_spread("spread", seed))
    return fx.problem(r.pods, instance_types=its, provisioners=[rp.unlimited()])


def interleaved_pins(seed):
    """two deployments alternate pod by pod, one node each (shared anti-affinity): one pins its nodes to a zone, the other
    does not, so pinned and unpinned nodes of one pod alternate in the order"""
    rng = random.Random(seed)
    zs = rp.zone_names(3, "us-west")
    its = rp.zonal_types(zs, [(2, 4), (8, 32)])
    r = rp.Runs("alt")
    anti = {"required": [fx.affinity_term(HOSTNAME, {"tier": "solo"})]}
    spec_p = {"labels": {"app": "p", "tier": "solo"}, "podAntiAffinity": anti,
              "nodeAffinity": {"required": [[{"key": ZONE, "operator": "In", "values": [zs[1 + seed % 2]]}]]}}
    spec_u = {"labels": {"app": "u", "tier": "solo"}, "podAntiAffinity": anti}
    r.interleave("p", "u", rng.choice([20, 40]), {"cpu": "1", "memory": "1Gi"}, spec_p, spec_u)
    r.run("spread", rng.choice([60, 129]), TINY, **_spread("spread", seed))
    return fx.problem(r.pods, instance_types=its, provisioners=[rp.unlimited()])


def partial_zone(seed):
    """the largest instance type is not offered in the last zone: pinning a node to that zone can narrow its types, so the
    pod that would pin it is left to the per-pod path"""
    rng = random.Random(seed)
    zs = rp.zone_names(3, "sa-west")
    its = rp.zonal_types(zs, [(2, 4), (4, 16)]) + rp.zonal_types(zs[:2], [(16, 64)], prefix="x")
    r = rp.Runs("part")
    r.run("anti", rng.choice([40, 70]), {"cpu": "1", "memory": "1Gi"}, labels={"app": "anti"},
          podAntiAffinity={"required": [fx.affinity_term(HOSTNAME, {"app": "anti"})]})
    r.run("spread", rng.choice([33, 129]), TINY, **_spread("spread", seed))
    return fx.problem(r.pods, instance_types=its, provisioners=[rp.unlimited()])


SCENARIOS = {"one_pod_nodes": one_pod_nodes, "mixed_counts": mixed_counts, "interleaved_pins": interleaved_pins,
             "partial_zone": partial_zone}
CASES = [(name, seed) for name in SCENARIOS for seed in (0, 1, 2)]


@pytest.mark.parametrize("name,seed", CASES, ids=[f"{n}-{s}" for n, s in CASES])
def test_pin_step_matches_oracle(pkg, oracle, name, seed):
    compare(pkg, oracle, pkg.Problem.from_dict(SCENARIOS[name](seed)))


@pytest.mark.parametrize("name", list(SCENARIOS))
def test_pin_step_every_block_size_and_without_mask_run(pkg, oracle, monkeypatch, name):
    """warp 0 drives the mask run at every block size; KSCHED_NO_MASKRUN places the same pods by the per-pod loop"""
    problem = pkg.Problem.from_dict(SCENARIOS[name](0))
    want = pkg.Result()
    assert oracle.solve(problem, want) == 0, want.error
    rs = pkg.ResidentSolve(problem)
    rs.set_count_visited(False)
    rs.load()
    monkeypatch.delenv("KSCHED_NO_MASKRUN", raising=False)
    for env in [("KSCHED_PACK_THREADS", str(t)) for t in (32, 64, 128, 256, 512)] + [("KSCHED_NO_MASKRUN", "1")]:
        monkeypatch.delenv("KSCHED_PACK_THREADS", raising=False)
        monkeypatch.setenv(*env)
        rs.run()
        res = rs.download()
        assert (res.assign == want.assign).all(), env
        assert res.digest() == want.digest(), env
        monkeypatch.delenv(env[0])
