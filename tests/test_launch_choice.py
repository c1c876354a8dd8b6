"""Launch choice of a finished node (SURVEY section 8f-2; fake/cloudprovider.go:74-84 + cloudprovider/types.go:120-145).
Three independent statements of it are pinned against each other on the CPU:
  * the oracle's (oracle/oracle.cc: launch_choice, strings),
  * the Python restatement the known-answer tests already use (tests/fixtures.py: launch),
  * the product's encoded offering table walked by the shared host/device core (csrc/launch.cuh) — kh_launch_table_selfcheck.
The device kernel itself is compared with the oracle in the GPU suites (every parity / fuzz / known-answer comparison)."""
import pytest

import fixtures as fx
from fuzz_problems import random_problem

ZONE, CT, ARCH = "topology.kubernetes.io/zone", "karpenter.sh/capacity-type", "kubernetes.io/arch"


@pytest.mark.parametrize("seed", range(40))
def test_oracle_launch_equals_python_restatement_and_encoded_table(pkg, oracle, seed):
    prob = random_problem(seed)
    problem, res = oracle.solve_dict(pkg, prob)
    d = res.to_dict()
    for node in d["newNodes"]:
        want = fx.launch(prob, node)
        assert want is not None
        got = node["launch"]
        assert (got["price"], prob["instanceTypes"][got["type"]]["name"], got["zone"]) == want
        it = prob["instanceTypes"][got["type"]]
        assert any(o["capacityType"] == got["capacityType"] and o["zone"] == got["zone"] and o["price"] == got["price"] and o.get("available", True)
                   for o in it["offerings"])
    try:
        bad = pkg.lib().kh_launch_table_selfcheck(problem.ptr, res.ptr)
    except Exception:  # pragma: no cover
        raise
    if bad == pkg.KSCHED_ERR_UNSUPPORTED:
        pytest.skip("encoder refuses this problem loudly")
    assert bad == 0


def _assorted():
    its = []
    for cpu in (1, 2, 4, 8):
        for mem in (2, 8):
            for zone in fx.ZONES:
                for ct in ("spot", "on-demand"):
                    for arch in ("amd64", "arm64"):
                        res = {"cpu": str(cpu), "memory": f"{mem}Gi", "pods": "10"}
                        its.append(fx.instance_type(f"{cpu}c-{mem}g-{arch}-{zone}-{ct}", res,
                                                    offerings=[{"capacityType": ct, "zone": zone, "price": fx.price_from_resources(res), "available": True}],
                                                    arch=arch, oses=("linux",)))
    return its


def _aff(key, value):
    return {"nodeAffinity": {"required": [[{"key": key, "operator": "In", "values": [value]}]]}}


def _min_price(its, pred):
    return min(o["price"] for it in its if pred(it) for o in it["offerings"])


def _arch(it):
    return next(r["values"][0] for r in it["requirements"] if r["key"] == ARCH)


# instance_selection_test.go:72-230 restated: the node is launched on one of the cheapest valid instance types
CASES = [
    ("any", {}, {}, lambda it: True),
    ("pod arch amd64", _aff(ARCH, "amd64"), {}, lambda it: _arch(it) == "amd64"),
    ("pod arch arm64", _aff(ARCH, "arm64"), {}, lambda it: _arch(it) == "arm64"),
    ("prov zone 2", {}, {"requirements": [{"key": ZONE, "operator": "In", "values": ["test-zone-2"]}]},
     lambda it: it["offerings"][0]["zone"] == "test-zone-2"),
    ("pod zone 2", _aff(ZONE, "test-zone-2"), {},
     lambda it: it["offerings"][0]["zone"] == "test-zone-2"),
    ("prov spot", {}, {"requirements": [{"key": CT, "operator": "In", "values": ["spot"]}]}, lambda it: it["offerings"][0]["capacityType"] == "spot"),
    ("pod on-demand", _aff(CT, "on-demand"), {},
     lambda it: it["offerings"][0]["capacityType"] == "on-demand"),
]


@pytest.mark.parametrize("name,pod_kw,prov_kw,pred", CASES, ids=[c[0] for c in CASES])
def test_launches_on_one_of_the_cheapest_valid_instances(pkg, oracle, name, pod_kw, prov_kw, pred):
    its = _assorted()
    prob = fx.problem([fx.pod(**pod_kw)], instance_types=its, provisioners=[fx.provisioner(**prov_kw)])
    problem, res = oracle.solve_dict(pkg, prob)
    d = res.to_dict()
    assert d["assign"] == [0] and len(d["newNodes"]) == 1
    node = d["newNodes"][0]
    assert node["launch"]["price"] == _min_price(its, pred)
    assert pred(its[node["launch"]["type"]])
    for idx in node["options"]:  # every option handed to the cloud provider is valid too
        assert pred(its[idx])
    assert pkg.lib().kh_launch_table_selfcheck(problem.ptr, res.ptr) == 0
