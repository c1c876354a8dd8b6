"""Known answers for consolidation validation (validation.go:63-172 and its two callers), restated from
pkg/controllers/deprovisioning/suite_test.go plus one case per branch of IsValid / ValidateCommand. Each case builds
((before, after), check); check(single, multi) receives SingleNodeConsolidation.ComputeCommand's and
MultiNodeConsolidation.ComputeCommand's results (action 0 nothing, 1 delete, 2 replace, 3 retry; "validations" = the trace)."""
import copy

import consolidation_answers as ca
import fixtures as fx

CASES = []


def case(ref):
    def deco(fn):
        CASES.append((fn.__name__, ref, fn))
        return fn
    return deco


def _cluster(n=3, pod_cpu="1"):
    """n nodes of the most expensive on-demand type, one small pod each: every node can be deleted on its own (its pod fits on
    a neighbour), and the multi-node search replaces all of them with one cheaper node"""
    its = ca.assorted()
    big = ca.on_demand_by_price(its)[-1]
    nodes = [ca.node_of_type(f"node{i + 1}", big, [fx.pod({"cpu": pod_cpu}, nodeName=f"node{i + 1}")], 1.0) for i in range(n)]
    return fx.problem([], instance_types=its, provisioners=[fx.provisioner(consolidationEnabled=True)], nodes=nodes, deriveCandidates=True)


def _pair(before, mutate=None):
    after = copy.deepcopy(before)
    if mutate:
        mutate(after)
    return before, after


@case("deprovisioning/suite_test.go:2246-2337")
def single_node_command_stands_on_an_unchanged_cluster():
    def check(single, multi):
        assert single["action"] == 1 and single["position"] == 0 and single["validations"] == [(0, True)]
    return _pair(_cluster()), check


@case("deprovisioning/suite_test.go:2721-2810")
def multi_node_command_stands_on_an_unchanged_cluster():
    def check(single, multi):
        assert multi["action"] == 2 and multi["nodes_removed"] == 3 and multi["options"] and multi["validations"] == [True]
    return _pair(_cluster()), check


@case("validation.go:85-91")
def nominated_node_fails_and_the_next_candidate_wins():
    def mutate(a):
        a["nodes"][0]["nominated"] = True
    def check(single, multi):
        assert single["action"] == 1 and single["position"] == 1 and single["validations"] == [(0, False), (1, True)]
        assert multi["action"] == 3 and multi["validations"] == [False]
    return _pair(_cluster(), mutate), check


@case("validation.go:112-116 (node gone)")
def removed_node_maps_to_nothing():
    def mutate(a):
        del a["nodes"][0]
    def check(single, multi):
        assert single["validations"][:2] == [(0, False), (1, True)] and single["action"] == 1
    return _pair(_cluster(), mutate), check


@case("validation.go:112-116 (marked for deletion)")
def node_marked_for_deletion_maps_to_nothing():
    def mutate(a):
        a["nodes"][0]["markedForDeletion"] = True
    def check(single, multi):
        assert single["validations"][:2] == [(0, False), (1, True)]
    return _pair(_cluster(), mutate), check


@case("helpers.go:328-337")
def multi_node_command_with_one_node_left_still_validates():
    def mutate(a):
        del a["nodes"][1]
    def check(single, multi):
        assert multi["action"] == 2 and multi["nodes_removed"] == 3 and multi["validations"] == [True]
    return _pair(_cluster(), mutate), check


@case("validation.go:85-91 (multi-node)")
def nominated_node_alone_fails_a_multi_node_delete():
    """a roomy node that is not a candidate takes every pod, so the search deletes all three candidates; in `after` node1 is
    nominated. Its partners still map and would validate on their own (their pods fit on the spare node): only the
    nominated check fails the command"""
    def with_spare(d):
        spare = copy.deepcopy(d["nodes"][0])
        spare.update(name="spare", pods=[], doNotConsolidate="true")
        spare["labels"][fx.HOSTNAME] = "spare"
        d["nodes"].append(spare)
        return d
    def mutate(a):
        a["nodes"][0]["nominated"] = True
    def check(single, multi):
        assert multi["action"] == 3 and multi["validations"] == [False] and multi["nodes_removed"] == 0
    return _pair(with_spare(_cluster()), mutate), check


@case("validation.go:122-124 + singlenodeconsolidation.go:80-83")
def pending_pods_that_do_not_fit_make_every_command_retry():
    def mutate(a):
        a["pods"] = [fx.pod({"cpu": "1000"})]
    def check(single, multi):
        assert single["action"] == 3 and single["validations"] == [(0, False), (1, False), (2, False)] and single["failed_validation"]
        assert multi["action"] == 3 and multi["options"] == [] and multi["validations"] == [False]
    return _pair(_cluster(), mutate), check


@case("validation.go:132-140")
def replace_with_room_elsewhere_needs_no_new_node():
    def mutate(a):
        spare = copy.deepcopy(a["nodes"][0])
        spare.update(name="spare", pods=[], doNotConsolidate="true")
        spare["labels"][fx.HOSTNAME] = "spare"
        a["nodes"].append(spare)
    def check(single, multi):
        assert single["action"] == 3 and single["validations"] == [(0, False)]
    return _pair(_cluster(1), mutate), check


@case("validation.go:147-151")
def delete_that_now_needs_a_new_node():
    def mutate(a):
        for n in a["nodes"][1:]:
            n["allocatable"] = {"cpu": "1", "memory": "64Gi", "pods": "100"}
    def check(single, multi):
        assert single["validations"][0] == (0, False)
    return _pair(_cluster(), mutate), check


@case("validation.go:142-145")
def two_new_nodes_are_never_valid():
    def mutate(a):
        for n in a["nodes"][1:]:
            n["allocatable"] = {"cpu": "1", "memory": "64Gi", "pods": "100"}
        a["nodes"][0]["pods"] += [fx.pod({"cpu": "20"}, nodeName="node1") for _ in range(2)]
    def check(single, multi):
        assert single["validations"][0] == (0, False)
    return _pair(_cluster(), mutate), check


@case("validation.go:153-171 (subset holds)")
def replacement_options_are_a_subset():
    def check(single, multi):
        assert single["action"] == 2 and single["options"] and single["validations"] == [(0, True)]
    return _pair(_cluster(1)), check


@case("validation.go:164-166 (subset fails)")
def replacement_needs_a_bigger_type_after_the_ttl():
    def mutate(a):
        a["nodes"][0]["pods"] = [fx.pod({"cpu": "20"}, nodeName="node1")]
    def check(single, multi):
        assert single["action"] == 3 and single["validations"] == [(0, False)]
    return _pair(_cluster(1), mutate), check


@case("helpers.go:106-113")
def uninitialised_node_in_after_fails_every_command():
    def mutate(a):
        n = copy.deepcopy(a["nodes"][0])
        n.update(name="fresh", pods=[])
        n["labels"][fx.HOSTNAME] = "fresh"
        n["labels"].pop(fx.INITIALIZED)
        a["nodes"].append(n)
    def check(single, multi):
        assert single["action"] == 3 and multi["action"] == 3
    return _pair(_cluster(), mutate), check


@case("validation.go:78-83 (no sortAndFilterCandidates)")
def node_a_pdb_now_blocks_is_still_validated():
    def mutate(a):
        a["nodes"][0]["pods"][0]["labels"] = {"app": "guarded"}
        a["pdbs"] = [{"namespace": "default", "selector": {"matchLabels": {"app": "guarded"}}, "disruptionsAllowed": 0}]
    def check(single, multi):
        assert single["action"] == 1 and single["validations"] == [(0, True)]
    return _pair(_cluster(), mutate), check
