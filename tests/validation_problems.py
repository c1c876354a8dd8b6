"""Seeded (before, after) pairs for consolidation validation: `before` is a cluster a consolidation pass computes on (fuzz
problems with topology, run-shaped zone-spread clusters, plain synthetic clusters); `after` is derived from it by seeded
mutations of what can change during the TTL - pods bound, new pending pods, a node removed / marked for deletion /
nominated / un-initialised, doNotConsolidate flipped, allocatable shrunk, new spread pods."""
import copy
import random

import fixtures as fx
import run_problems
import validation_answers as va
from fuzz_problems import random_problem


def _fuzz_cluster(seed):
    prob = random_problem(seed)
    rng = random.Random(seed * 31 + 7)
    offered = {(it["name"], o["capacityType"], o["zone"]) for it in prob["instanceTypes"] for o in it["offerings"]}
    n = 0
    for node in prob.get("nodes", []):
        lab = node["labels"]
        if lab.get(fx.PROVISIONER_NAME) and not node.get("markedForDeletion") and \
                (lab.get(fx.INSTANCE_TYPE), lab.get(fx.CAPACITY_TYPE), lab.get(fx.ZONE)) in offered:
            node["candidate"] = True
            node["disruptionCost"] = float(rng.choice([0, 1, 1, 2, 3]))
            n += 1
    return prob if n >= 2 else None


def _mutate(after, rng):
    nodes = after.setdefault("nodes", [])
    kinds = rng.sample(["bind", "pending", "remove", "delete", "nominate", "uninit", "dnc", "shrink", "spread"], rng.choice([1, 1, 2, 3]))
    for kind in kinds:
        if not nodes:
            break
        i = rng.randrange(len(nodes))
        n = nodes[i]
        if kind == "bind" and after.get("pods"):
            p = after["pods"].pop(rng.randrange(len(after["pods"])))
            p["nodeName"] = n["name"]
            n.setdefault("pods", []).append(p)
        elif kind == "pending":
            after.setdefault("pods", []).extend(fx.pod({"cpu": rng.choice(["100m", "1", "3", "12"]), "memory": rng.choice(["128Mi", "2Gi"])}) for _ in range(rng.choice([1, 2, 5])))
        elif kind == "remove":
            nodes.pop(i)
        elif kind == "delete":
            n["markedForDeletion"] = True
        elif kind == "nominate":
            n["nominated"] = True
        elif kind == "uninit":
            n["labels"].pop(fx.INITIALIZED, None)
        elif kind == "dnc":
            n["doNotConsolidate"] = "false" if n.get("doNotConsolidate") == "true" else "true"
        elif kind == "shrink":
            n["allocatable"] = dict(n.get("allocatable", {}), cpu=rng.choice(["500m", "1", "2"]))
        elif kind == "spread":
            lab = {"app": f"spread-{rng.randrange(1000)}"}
            after.setdefault("pods", []).extend(fx.pod({"cpu": "500m"}, labels=lab, topologySpreadConstraints=[fx.spread(fx.ZONE, lab)])
                                                for _ in range(rng.choice([2, 3])))
    return kinds


def pairs(count=72):
    """[(name, before, after)]: a third each from fuzz clusters, run-shaped clusters and synthetic ones"""
    out = []
    seed = 0
    while len([p for p in out if p[0].startswith("fuzz")]) < count // 3:
        b = _fuzz_cluster(seed)
        if b is not None:
            out.append((f"fuzz-{seed}", b))
        seed += 1
    for s in range(count // 3):
        out.append((f"run-{s}", run_problems.cluster(s + 1, (9, 16)[s % 2], s % 3 == 0)))
    for s in range(count - len(out)):
        b = va._cluster(2 + s % 5, ("1", "4", "12")[s % 3])
        out.append((f"synthetic-{s}", b))
    res = []
    for k, (name, before) in enumerate(out):
        rng = random.Random(1000 + k)
        after = copy.deepcopy(before)
        kinds = _mutate(after, rng) if k % 6 else []   # every sixth pair: the cluster did not change
        res.append((f"{name}:{'+'.join(kinds) or 'unchanged'}", before, after))
    return res
