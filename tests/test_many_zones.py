"""CPU: catalogs that offer instance types in more than 16 zones or 4 capacity types (tests/zone_problems.py) encode without
refusal. The dense offering slots equal the (capacity type, zone) pairs of available offerings restated on strings, catalogs
that fit ct*16 + zone keep that layout (no slot tables, digest as before), and more than 64 pairs is refused. The oracle's
launch choice equals the Python restatement and the encoded offering table walked by the shared core, every option of
every new node has an offering its requirements admit, and the oracle's fast mode equals its literal path."""
import json
from pathlib import Path

import pytest

import fixtures as fx
import zone_problems as zp

CORPUS = zp.corpus()
IDS = [c[0] for c in CORPUS]
GOLDEN = Path(__file__).parent / "golden" / "zone_layout_digests.json"


@pytest.mark.parametrize("name,prob,table", CORPUS, ids=IDS)
def test_encoder_takes_the_scenario(pkg, name, prob, table):
    rs = pkg.ResidentSolve(pkg.Problem.from_dict(prob))
    assert (rs.dims["offering_slots"] > 0) == table


@pytest.mark.parametrize("name,prob,table", [c for c in CORPUS if c[2]], ids=[c[0] for c in CORPUS if c[2]])
def test_slots_equal_the_pair_rule(pkg, name, prob, table):
    rs = pkg.ResidentSolve(pkg.Problem.from_dict(prob))
    keys = [rs.key_info(k) for k in (fx.ZONE, fx.CAPACITY_TYPE)]
    assert all(k is None or k["representatives"] == 0 for k in keys)  # no value folded into a class
    want = zp.pairs(prob, keys[0] is not None, keys[1] is not None)
    assert rs.offering_slots() == want
    assert rs.dims["offering_slots"] == len(want) <= 64


def test_old_layout_keeps_its_encoding(pkg):
    """16 zones x 4 capacity types, and the capacity-type typo without a fifth value, fit ct*16 + zone: no slot tables, and
    the same digest as before the slot tables existed"""
    golden = json.loads(GOLDEN.read_text())
    for name, prob in (("zones16x4", zp.zonal(16, cts=("capacity-block", "on-demand", "reserved", "spot"))),
                       ("ct-typo-one", zp.ct_typo(False))):
        rs = pkg.ResidentSolve(pkg.Problem.from_dict(prob))
        assert rs.dims["offering_slots"] == 0 and rs.offering_slots() == []
        assert f"{pkg.lib().kh_encoded_digest(rs.enc):016x}" == golden[name], name


def test_more_than_64_pairs_is_refused(pkg):
    with pytest.raises(pkg.KschedError) as e:
        pkg.ResidentSolve(pkg.Problem.from_dict(zp.near_miss()))
    assert e.value.code == pkg.KSCHED_ERR_UNSUPPORTED
    assert "66 pairs" in str(e.value)


@pytest.mark.parametrize("name,prob,table", CORPUS, ids=IDS)
def test_launch_choice_three_ways(pkg, oracle, name, prob, table):
    problem, res = oracle.solve_dict(pkg, prob)
    d = res.to_dict()
    for node in d["newNodes"]:
        got = node["launch"]
        assert (got["price"], prob["instanceTypes"][got["type"]]["name"], got["zone"]) == fx.launch(prob, node)
    assert pkg.lib().kh_launch_table_selfcheck(problem.ptr, res.ptr) == 0


@pytest.mark.parametrize("name,prob,table", CORPUS, ids=IDS)
def test_every_option_has_an_admitted_offering(pkg, oracle, name, prob, table):
    _, res = oracle.solve_dict(pkg, prob)
    for node in res.to_dict()["newNodes"]:
        assert node["options"]
        assert all(zp.has_offering(prob, node, i) for i in node["options"])


@pytest.mark.parametrize("name,prob,table", CORPUS, ids=IDS)
def test_oracle_fast_mode_equals_literal(pkg, oracle, name, prob, table):
    oracle.assert_fast_equals_literal(pkg, prob)


def test_scenarios_cross_what_they_were_built_for(pkg, oracle):
    # the capacity-type typo: the plain pods schedule on one new node, the two typo pods do not
    _, res = oracle.solve_dict(pkg, zp.ct_typo())
    d = res.to_dict()
    assert d["assign"][:5] == [d["assign"][0]] * 5 and d["assign"][0] >= 0 and d["assign"][5:] == [-1, -1]
    # a zone only a pod names pushes the last offered zone to id 16
    rs = pkg.ResidentSolve(pkg.Problem.from_dict(zp.pod_named_zone(0)))
    assert rs.dims["offering_slots"] == 16 and rs.key_info(fx.ZONE)["values"] == 17
    # Local-Zone pods land in their Local Zone
    prob = zp.local_pinned(0)
    d = oracle.solve_dict(pkg, prob)[1].to_dict()
    lz = prob["pods"][33]["nodeSelector"][fx.ZONE]
    n_ex = len(d["existing"])
    nodes = {d["assign"][i] for i in range(33, 45)}
    assert all(a >= n_ex and d["newNodes"][a - n_ex]["launch"]["zone"] == lz for a in nodes)
    # the consolidation cluster prices a replacement in a Local Zone
    cands = [i for i, n in enumerate(zp.cluster(0)["nodes"]) if n.get("candidate")]
    for prob in (zp.cluster(0), zp.after(0)):
        assert pkg.ResidentSolve(pkg.Problem.from_dict(prob), candidates=cands).dims["offering_slots"] > 0
