"""CPU: clusters and batches whose pods mount more than 64 volume claims that the sharing rule would track
(tests/volume_problems.py) encode without refusal, in plain and superset form. The encoder's tracked claims are the rule
restated from the problem's strings; problems that fit the word get no table; more than 4 limited drivers stay refused. The
oracle's results keep every existing node within its volume limits, and its fast mode equals the literal path."""
import ctypes as C

import pytest

import fixtures as fx
import volume_problems as vp

CORPUS = vp.corpus()
IDS = [c[0] for c in CORPUS]
CLUSTERS = vp.clusters()
CIDS = [c[0] for c in CLUSTERS]


def _words(n):
    return (n - 64 + 63) // 64 if n > 64 else 0


def _candidates(prob):
    return [i for i, n in enumerate(prob["nodes"]) if n.get("candidate")]


def _encode(pkg, prob, cands, superset):
    """(tracked claims, dims) of kh_encode / kh_encode_cluster; raises KschedError on a refusal"""
    problem = pkg.Problem.from_dict(prob)
    arr = (C.c_int * max(1, len(cands)))(*cands)
    f = pkg.lib().kh_encode_cluster if superset else pkg.lib().kh_encode
    enc = f(problem.ptr, arr, len(cands))
    if not enc:
        msg = pkg.lib().kh_scheduler_error().decode()
        raise pkg.KschedError(pkg.KSCHED_ERR_UNSUPPORTED if msg.startswith("unsupported:") else pkg.KSCHED_ERR_INVALID, msg)
    try:
        d = (C.c_longlong * 20)()
        pkg.lib().kh_encoded_dims(enc, d)
        out, buf = [], C.create_string_buffer(1024)
        while pkg.lib().kh_encoded_volume_claim(enc, len(out), buf, len(buf)) == 0:
            out.append(tuple(buf.value.decode().split(" ", 1)))
        return out, {"volume_claims": d[18], "volume_ext_words": d[19]}
    finally:
        pkg.lib().kh_encoded_free(enc)


def _check(pkg, prob, cands, superset):
    claims, dims = _encode(pkg, prob, cands, superset)
    want = vp.tracked_claims(prob, cands, superset)
    assert claims == want
    assert dims == {"volume_claims": len(want), "volume_ext_words": _words(len(want))}
    return claims


@pytest.mark.parametrize("name,prob,table", CORPUS, ids=IDS)
def test_batches_track_the_rule(pkg, name, prob, table):
    claims = _check(pkg, prob, [], False)
    assert (len(claims) > 64) == table
    rs = pkg.ResidentSolve(pkg.Problem.from_dict(prob))
    assert rs.volume_claims() == claims
    assert rs.dims["volume_claims"] == len(claims) and rs.dims["volume_ext_words"] == _words(len(claims))


@pytest.mark.parametrize("name,prob,table", CLUSTERS, ids=CIDS)
def test_clusters_encode_in_both_forms(pkg, name, prob, table):
    cands = _candidates(prob)
    assert vp.shared_count(prob, cands, True) > 64  # refused before the rule
    for p in (prob, vp.after(prob, 0)):
        _check(pkg, p, cands, False)
        assert (len(_check(pkg, p, cands, True)) > 64) == table
        _check(pkg, p, [], False)


def test_statefulset_pods_of_one_shape_share_a_class(pkg):
    """private claims do not split classes: 100 StatefulSet pods, one claim each, are one class of a Solve batch"""
    prob = vp.statefulsets(100, 1, 1)
    rs = pkg.ResidentSolve(pkg.Problem.from_dict(prob), candidates=_candidates(prob))
    assert rs.dims["volume_claims"] == 0 and rs.dims["pods"] == 100
    assert len({rs.pod_class(i) for i in range(100)}) == 2  # with and without a PD claim


def test_boundaries():
    assert [len(vp.tracked_claims(vp.boundary(k))) for k in ("fit64", "one65", "edge128", "edge129", "narrow65")] == [64, 65, 128, 129, 64]


def test_traps(pkg):
    prob = vp.traps(0)
    rs = pkg.ResidentSolve(pkg.Problem.from_dict(prob))
    claims = rs.volume_claims()
    for c in ("z/high-only", "z/twin-1", "z/twin-2"):
        assert claims.index((vp.EBS, c)) >= 64
    assert not any(c[0] == vp.EFS or c[0] == "" for c in claims)  # no limit for the driver, or no driver: never tracked
    assert (vp.EBS, "dup/d-0") not in claims                        # one pod mounting a claim twice does not share it
    # the twins differ only in a claim beyond 64: two classes
    twins = [i for i, p in enumerate(prob["pods"]) if p["labels"]["app"] == "twin"]
    assert len({rs.pod_class(i) for i in twins}) == 2


def test_more_than_four_limited_drivers_stay_refused(pkg):
    nodes = [fx.state_node(f"n-{i}", "fake-it-7", volumeLimits={f"d{i}.csi": 5}) for i in range(5)]
    prob = fx.problem([fx.pod({"cpu": "100m"}, volumes=[vp.vol("d0.csi", "x/a")])], instance_types=fx.fake_instance_types(16), nodes=nodes)
    with pytest.raises(pkg.KschedError) as e:
        pkg.ResidentSolve(pkg.Problem.from_dict(prob))
    assert "more than 4 CSI drivers" in str(e.value)


@pytest.mark.parametrize("name,prob,table", CORPUS, ids=IDS)
def test_oracle_keeps_volume_limits(pkg, oracle, name, prob, table):
    d = oracle.solve_dict(pkg, prob)[1].to_dict()
    assert vp.volume_violations(prob, d) == []
    with_claims = [i for i, p in enumerate(prob["pods"]) if p.get("volumes")]
    assert any(d["assign"][i] >= 0 for i in with_claims)


@pytest.mark.parametrize("name,prob,table", CORPUS, ids=IDS)
def test_oracle_fast_mode_equals_literal(pkg, oracle, name, prob, table):
    oracle.assert_fast_equals_literal(pkg, prob)
