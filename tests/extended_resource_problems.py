"""Seeded corpus of GPU-fleet-shaped batches whose pods request more than 8 distinct resources (DESIGN.md §3, ext resources).
cpu, memory, pods, ephemeral-storage, `nvidia.com/gpu` (named by a provisioner limit) and `hugepages-2Mi` (requested by a
daemonset) take row slots; the rest (MIG profiles, EFA, hugepages-1Gi, Neuron, pod ENIs, FPGAs, ...) are ext resources.

 * fleet(seed, extra): GPU and CPU instance types, two pools (one with a GPU limit), a hugepages daemonset, existing nodes
   that alone advertise MIG profiles, and deployments that request ext resources in containers and init containers, with a
   zone spread and a hostname anti-affinity, plus two deployments identical except for one MIG amount;
 * cluster(seed) / after(seed): a consolidation cluster of GPU nodes and the same cluster after the TTL;
 * near misses that must still be refused: 33 read resources, and 9 resources that need a row slot.
"""
import copy
import random

import fixtures as fx
from fixtures import HOSTNAME, ZONE

MIG = ("nvidia.com/mig-1g.10gb", "nvidia.com/mig-3g.40gb", "nvidia.com/mig-7g.80gb")
EXT = ("vpc.amazonaws.com/efa", "hugepages-1Gi", "aws.amazon.com/neuron", "vpc.amazonaws.com/pod-eni", "example.com/fpga")


def instance_types():
    out = fx.fake_instance_types(8)
    for it in out:
        it["capacity"] = dict(it["capacity"], **{"ephemeral-storage": "100Gi", "hugepages-2Mi": "1Gi"})
    for i, (gpus, efa) in enumerate(((1, 0), (4, 1), (8, 4))):
        out.append(fx.instance_type(f"gpu-{gpus}x", {"cpu": str(8 * gpus), "memory": f"{32 * gpus}Gi", "pods": "110", "nvidia.com/gpu": str(gpus),
                                                   "vpc.amazonaws.com/efa": str(efa), "hugepages-2Mi": "2Gi", "hugepages-1Gi": str(gpus) + "Gi",
                                                   "ephemeral-storage": "500Gi", "vpc.amazonaws.com/pod-eni": str(4 * gpus)}))
    out.append(fx.instance_type("inf-2", {"cpu": "16", "memory": "64Gi", "pods": "58", "aws.amazon.com/neuron": "2", "hugepages-2Mi": "1Gi",
                                          "ephemeral-storage": "200Gi", "example.com/fpga": "1"}))
    out.append(fx.instance_type("inf-8", {"cpu": "32", "memory": "128Gi", "pods": "58", "aws.amazon.com/neuron": "8", "hugepages-2Mi": "1Gi",
                                          "ephemeral-storage": "200Gi"}))
    return out


def pools():
    gpu = fx.provisioner("gpu", weight=10, limits={"cpu": "4000", "nvidia.com/gpu": "24"})
    return [gpu, fx.provisioner("general")]


def daemonsets():
    return [fx.pod({"cpu": "100m", "memory": "128Mi", "hugepages-2Mi": "256Mi"}, name="ds-hugepages", isDaemonSet=True)]


def _mig_node(name, rng, mig_amounts, pool="gpu"):
    alloc = {"cpu": "63900m", "memory": "250Gi", "pods": "110", "nvidia.com/gpu": "0", "ephemeral-storage": "500Gi", "hugepages-2Mi": "2Gi"}
    for m, a in zip(MIG, mig_amounts):
        alloc[m] = str(a)
    return fx.state_node(name, "gpu-8x", zone=rng.choice(fx.ZONES[:3]), provisioner_name=pool, allocatable=alloc, capacity=dict(alloc))


def _gpu_node(name, rng, it="gpu-4x", pods_=None):
    g = int(it.split("-")[1][:-1])
    alloc = {"cpu": f"{8 * g * 1000 - 100}m", "memory": f"{32 * g - 1}Gi", "pods": "110", "nvidia.com/gpu": str(g), "vpc.amazonaws.com/efa": str(1 if g == 4 else 4 if g == 8 else 0),
             "hugepages-2Mi": "2Gi", "hugepages-1Gi": f"{g}Gi", "ephemeral-storage": "500Gi", "vpc.amazonaws.com/pod-eni": str(4 * g)}
    return fx.state_node(name, it, zone=rng.choice(fx.ZONES[:3]), provisioner_name="gpu", allocatable=alloc, capacity=dict(alloc), pods_=pods_ or [])


def _pods(n, requests, **kw):
    return [fx.pod(dict(requests), **kw) for _ in range(n)]


def _init_pods(n, containers, init, **kw):
    return [fx.pod(None, containers=[{"requests": dict(containers)}], initContainers=[{"requests": dict(init)}], **kw) for _ in range(n)]


def workload(rng, extra=()):
    pods = []
    pods += _pods(40, {"cpu": "1", "memory": "2Gi"}, labels={"app": "web"})
    pods += _pods(20, {"cpu": "2", "memory": "4Gi", "ephemeral-storage": "10Gi"}, labels={"app": "batch"})
    pods += _pods(12, {"cpu": "4", "memory": "16Gi", "nvidia.com/gpu": "1"}, labels={"app": "train"})
    pods += _pods(6, {"cpu": "8", "memory": "32Gi", "nvidia.com/gpu": "4", "vpc.amazonaws.com/efa": "1", "hugepages-1Gi": "2Gi"}, labels={"app": "dist"})
    # two deployments identical except for the amount of an ext resource (few pods request neuron): the larger one fits
    # inf-8 only, so a row or variant shared between the two classes would be wrong
    pods += _pods(4, {"cpu": "1", "memory": "4Gi", "aws.amazon.com/neuron": "1"}, labels={"app": "neuron"})
    pods += _pods(4, {"cpu": "1", "memory": "4Gi", "aws.amazon.com/neuron": "4"}, labels={"app": "neuron"})
    pods += _pods(6, {"cpu": "1", "memory": "4Gi", MIG[0]: "1"}, labels={"app": "infer"})
    pods += _pods(4, {"cpu": "2", "memory": "8Gi", MIG[1]: "1"}, labels={"app": "mid"})
    pods += _pods(2, {"cpu": "4", "memory": "16Gi", MIG[2]: "1"}, labels={"app": "big"})
    pods += _pods(6, {"cpu": "2", "memory": "8Gi", "example.com/fpga": "1"}, labels={"app": "inf"})
    pods += _init_pods(5, {"cpu": "1", "memory": "1Gi"}, {"cpu": "1", "vpc.amazonaws.com/pod-eni": "2", "hugepages-1Gi": "1Gi"}, labels={"app": "init"})
    pods += _pods(9, {"cpu": "2", "memory": "8Gi", "nvidia.com/gpu": "1", "vpc.amazonaws.com/pod-eni": "1"}, labels={"app": "spread"},
                  topologySpreadConstraints=[fx.spread(ZONE, {"app": "spread"})])
    pods += _pods(4, {"cpu": "2", "memory": "8Gi", "vpc.amazonaws.com/efa": "1"}, labels={"app": "anti"},
                  podAntiAffinity={"required": [fx.affinity_term(HOSTNAME, {"app": "anti"})]})
    for r in extra:
        pods += _pods(2, {"cpu": "1", r: "1"}, labels={"app": "extra"})
    rng.shuffle(pods)
    return pods


def fleet(seed, extra=(), existing=True):
    """existing=False: no existing nodes, so the pack kernel's closed-form modes (class run and its steps, variant store,
    failure memo) run for the classes that request no ext resource, between the generic steps of those that do"""
    rng = random.Random(seed * 31 + 7)
    nodes = [_mig_node(f"mig-{i}", rng, (rng.choice([2, 4, 7]), rng.choice([0, 1, 2]), rng.choice([0, 1]))) for i in range(4)]
    nodes += [_gpu_node(f"gpu-{i}", rng, rng.choice(["gpu-4x", "gpu-8x"])) for i in range(3)]
    if not existing:
        nodes = []
    its = instance_types()
    for r in extra:  # extra resources every instance type offers
        for it in its:
            it["capacity"][r] = "4"
    return fx.problem(workload(rng, extra), instance_types=its, provisioners=pools(), nodes=nodes, daemonSetPods=daemonsets())


def cluster(seed):
    """GPU nodes of the `gpu` pool, half of them consolidation candidates, running GPU and MIG pods"""
    rng = random.Random(seed * 17 + 3)
    nodes = []
    for i in range(10):
        bound = []
        name = f"gn-{i}"
        for _ in range(rng.choice([0, 1, 2])):
            bound.append(fx.pod({"cpu": "2", "memory": "8Gi", "nvidia.com/gpu": "1", "vpc.amazonaws.com/pod-eni": "1"}, labels={"app": "train"},
                                nodeName=name))
        if i % 3 == 0:
            bound.append(fx.pod({"cpu": "1", "memory": "2Gi", "hugepages-1Gi": "1Gi", "vpc.amazonaws.com/efa": "1"}, labels={"app": "net"}, nodeName=name))
        n = _gpu_node(name, rng, rng.choice(["gpu-4x", "gpu-8x"]), pods_=bound)
        if i < 5:
            n.update(candidate=True, disruptionCost=float(rng.choice([0, 1, 2])), creationTimestamp=float(i))
        nodes.append(n)
    nodes += [_mig_node(f"mig-{i}", rng, (7, 2, 1)) for i in range(2)]
    nodes[-1]["pods"] = [fx.pod({"cpu": "1", "memory": "4Gi", MIG[0]: "1"}, labels={"app": "infer"}, nodeName=nodes[-1]["name"])]
    nodes[-1].update(candidate=True, disruptionCost=0.0, creationTimestamp=9.0)
    return fx.problem([], instance_types=instance_types(), provisioners=pools(), nodes=nodes, daemonSetPods=daemonsets())


def after(seed):
    """cluster(seed) after the TTL: one more GPU pod is pending and a node has taken a MIG pod"""
    a = copy.deepcopy(cluster(seed))
    a["pods"] = _pods(1, {"cpu": "2", "memory": "8Gi", "nvidia.com/gpu": "1"}, labels={"app": "late"})
    n = a["nodes"][-2]
    n["pods"] = n["pods"] + [fx.pod({"cpu": "1", "memory": "4Gi", MIG[1]: "1"}, labels={"app": "mid"}, nodeName=n["name"])]
    return a


def corpus():
    """[(name, problem dict)]: every problem reads 9 to 32 resources"""
    out = [(f"fleet-{s}", fleet(s)) for s in range(3)]
    out.append(("fleet-32", fleet(3, extra=tuple(f"example.com/res-{i:02d}" for i in range(18)))))
    return out


def fresh_corpus():
    """[(name, problem dict)]: the fleet without existing nodes, ext and other classes mixed"""
    return [(f"fresh-{s}", fleet(s, existing=False)) for s in range(3)] + \
           [("fresh-32", fleet(3, extra=tuple(f"example.com/res-{i:02d}" for i in range(18)), existing=False))]


# slot membership of fleet(): the limit- and daemonset-named resources and the three most requested others take the 8 row
# slots; the MIG profiles, EFA, Neuron and FPGAs are ext resources
SLOTS = ("cpu", "memory", "pods", "nvidia.com/gpu", "hugepages-2Mi", "ephemeral-storage", "vpc.amazonaws.com/pod-eni", "hugepages-1Gi")
EXT_RESOURCES = MIG + ("vpc.amazonaws.com/efa", "aws.amazon.com/neuron", "example.com/fpga")


def too_many_resources():
    """33 read resources"""
    return fleet(4, extra=tuple(f"example.com/res-{i:02d}" for i in range(19)))


def too_many_slot_resources():
    """9 resources that need a row slot: cpu, memory, pods, the GPU limit, and five a daemonset requests"""
    p = fleet(5)
    p["daemonSetPods"] = [fx.pod({"cpu": "100m", "hugepages-2Mi": "1Mi", "hugepages-1Gi": "1Gi", "ephemeral-storage": "1Gi",
                                  "vpc.amazonaws.com/efa": "0", "vpc.amazonaws.com/pod-eni": "1"}, name="ds-wide", isDaemonSet=True)]
    return p


def read_resources(prob):
    """names some pending pod requests (containers or init containers), some daemonset requests or a limit names"""
    names = set()
    for p in prob["pods"] + prob.get("daemonSetPods", []):
        names |= set(p.get("requests", {}))
        for c in p.get("containers", []) + p.get("initContainers", []):
            names |= set(c.get("requests", {}))
    for pr in prob["provisioners"]:
        names |= set(pr.get("limits", {}))
    return names | {"pods"}


def pairs(n_pairs=2200):
    """n_pairs pairs of classes, each pair identical except for its Neuron amount (1 or 8; only nx-64 holds 8), listed pair by
    pair so that the two classes of a pair are neighbours in the class table. With more classes than K1 has warps, one warp
    evaluates both rows of a pair back to back, so its consecutive-row cache must tell them apart. Limits on five resources
    no pod requests fill the row slots, which makes Neuron an ext resource."""
    its = [fx.instance_type("nx-4", {"cpu": "64", "memory": "256Gi", "pods": "110", "aws.amazon.com/neuron": "4"}),
           fx.instance_type("nx-64", {"cpu": "64", "memory": "256Gi", "pods": "110", "aws.amazon.com/neuron": "64"})]
    pool = fx.provisioner("neuron", limits={f"example.com/quota-{i}": "1000000" for i in range(5)})
    pods = []
    for k in range(n_pairs):
        for amount in ("1", "8"):
            pods.append(fx.pod({"cpu": f"{10 + k}m", "memory": "64Mi", "aws.amazon.com/neuron": amount}, labels={"app": f"p{k}"}))
    return fx.problem(pods, instance_types=its, provisioners=[pool])
