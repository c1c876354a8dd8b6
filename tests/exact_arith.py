"""An independent restatement, in exact Python arithmetic, of the numeric parts of Scheduler.Solve and of the candidate
ranking, for the numeric-edge corpus (tests/numeric_problems.py). Quantities are exact integers of milli-units parsed
with `fractions` (resource.Quantity is exact decimal and never wraps); costs are IEEE float64 like Go's.

  RequestsForPods, allocatable, Fits        utils/resources/resources.go:25-33,62-89,138-145
  daemonset overhead                         scheduler.go:250-267 (the corpus's daemonsets select every node)
  provisioner remaining                      scheduler.go:221-248 (limits minus the owned nodes' capacity),
                                             scheduler.go:273-309 (each new node's max over its options)
  GetPodEvictionCost, calculateLifetimeRemaining, clamp, the disruption sort
                                             deprovisioning/helpers.go:125-165,275-287,317-325, consolidation.go:85-103

check_exact(problem, result) holds a Solve result to that arithmetic. It checks necessary conditions only: the result's
final options are a subset of the options a new node was charged for, so the remaining it computes is never below the
reference's."""
import math
from fractions import Fraction

import numpy as np

PROVISIONER_NAME = "karpenter.sh/provisioner-name"
SUFFIX = {"": 1, "m": Fraction(1, 1000), "k": 10 ** 3, "M": 10 ** 6, "G": 10 ** 9, "T": 10 ** 12, "P": 10 ** 15, "E": 10 ** 18,
          "Ki": 2 ** 10, "Mi": 2 ** 20, "Gi": 2 ** 30, "Ti": 2 ** 40, "Pi": 2 ** 50, "Ei": 2 ** 60}


def quantity_milli(s):
    """exact value of a quantity string in milli-units: an int, or a Fraction when it is not a whole number of milli"""
    s = str(s)
    i = 0
    while i < len(s) and (s[i].isdigit() or s[i] in "+-."):
        i += 1
    num, suf = s[:i], s[i:]
    return Fraction(num) * SUFFIX[suf] * 1000


def _resources(d):
    return {k: quantity_milli(v) for k, v in (d or {}).items()}


def _merge(a, b):
    r = dict(a)
    for k, v in b.items():
        r[k] = r.get(k, 0) + v
    return r


def _subtract(lhs, rhs):
    return {k: v - rhs.get(k, 0) for k, v in lhs.items()}


def _containers(pod):
    cs = list(pod.get("containers", []))
    if any(k in pod for k in ("requests", "limits", "ports")):
        cs.append(pod)
    return cs, pod.get("initContainers", [])


def _effective(c):
    r = _resources(c.get("requests"))
    for k, v in _resources(c.get("limits")).items():
        r.setdefault(k, v)
    return r


def pod_requests(pod):
    """RequestsForPods(pod): containers summed (limits standing in for missing requests), init containers' max, pods: 1"""
    cs, init = _containers(pod)
    r = {}
    for c in cs:
        r = _merge(r, _effective(c))
    for c in init:
        for k, v in _effective(c).items():
            if k not in r or v > r[k]:
                r[k] = v
    r["pods"] = 1000
    return r


def requests_for_pods(pods):
    r = {}
    for p in pods:
        r = _merge(r, pod_requests(p))
    r["pods"] = 1000 * len(pods)
    return r


def allocatable(it):
    ov = it.get("overhead") or {}
    overhead = _merge(_merge(_resources(ov.get("kubeReserved")), _resources(ov.get("systemReserved"))), _resources(ov.get("evictionThreshold")))
    return _subtract(_resources(it.get("capacity")), overhead)


def fits(candidate, total):
    return all(v <= total.get(k, 0) for k, v in candidate.items())


def _templates(problem):
    """provisioners in weight order (OrderByWeight, stable)"""
    provs = problem.get("provisioners", [])
    return sorted(range(len(provs)), key=lambda i: -provs[i].get("weight", 0))


def daemon_overhead(problem):
    return requests_for_pods(problem.get("daemonSetPods", []))


def remaining_after_existing(problem, prov, removed=()):
    """limits minus the capacity of every node the provisioner owns (nodes in `removed` are not charged)"""
    rem = _resources(prov["limits"])
    for i, n in enumerate(problem.get("nodes", [])):
        if i in removed or n.get("labels", {}).get(PROVISIONER_NAME) != prov["name"]:
            continue
        rem = _subtract(rem, _resources(n.get("capacity") or n.get("allocatable")))
    return rem


def check_exact(problem, result, answer=None):
    """Solve's result held to exact arithmetic: pods on existing nodes fit, every option of every new node holds its pods
    and the daemonset overhead, no provisioner opens a node its remaining limits exclude, and `answer` (a callable on the
    result, from the corpus) holds. Returns a list of failures, empty when the result passes."""
    bad = []
    pods = problem.get("pods", [])
    nodes = problem.get("nodes", [])
    its = problem["instanceTypes"]
    provs = problem["provisioners"]
    order = _templates(problem)
    existing = result["existing"]
    n_ex = len(existing)
    ds = problem.get("daemonSetPods", [])
    overhead = daemon_overhead(problem)
    for k, ex in enumerate(existing):  # ExistingNode.Add: remaining daemon requests + new pods <= allocatable - bound pods
        n = nodes[ex["node"]] if isinstance(ex, dict) and "node" in ex else None
        if n is None:
            continue
        mine = [pods[i] for i, a in enumerate(result["assign"]) if a == k]
        if not mine:
            continue
        bound = n.get("pods", [])
        rem_ds = {k2: max(v, 0) for k2, v in _subtract(overhead, requests_for_pods([p for p in bound if p.get("isDaemonSet")])).items()} if ds else {}
        need = _merge(rem_ds, requests_for_pods(mine))
        avail = _subtract(_resources(n.get("allocatable")), requests_for_pods(bound))
        if not fits(need, avail):
            bad.append(f"existing node {n['name']}: requests {need} do not fit {avail}")
    remaining = {}
    for v, pi in enumerate(order):
        if provs[pi].get("limits") is not None:
            remaining[v] = remaining_after_existing(problem, provs[pi])
    for j, nn in enumerate(result["newNodes"]):
        v = nn["provisioner"]
        req = _merge(overhead if ds else {}, requests_for_pods([pods[i] for i in nn["pods"]]))
        for t in nn["options"]:
            if not fits(req, allocatable(its[t])):
                bad.append(f"new node {j}: option {its[t]['name']} cannot hold {req}")
        if v in remaining:
            rem = remaining[v]
            for t in nn["options"]:
                cap = _resources(its[t]["capacity"])
                if any(cap.get(k, 0) > q for k, q in rem.items()):
                    bad.append(f"new node {j}: option {its[t]['name']} is beyond provisioner {provs[order[v]]['name']}'s remaining {rem}")
            mx = {}
            for t in nn["options"]:
                for k, q in _resources(its[t]["capacity"]).items():
                    mx[k] = max(mx.get(k, q), q)
            remaining[v] = _subtract(rem, mx)
    if answer is not None and not answer(result):
        bad.append("the result differs from the stated answer")
    return bad


# ---------------------------------------------------------------- candidate ranking (float64, as Go computes it)
def _div(a, b):
    with np.errstate(divide="ignore", invalid="ignore"):
        return float(np.float64(a) / np.float64(b))


def clamp(lo, val, hi):  # helpers.go:317-325: NaN passes through
    if val < lo:
        return lo
    if val > hi:
        return hi
    return val


def pod_eviction_cost(pod):  # helpers.go:125-146
    cost = 1.0
    if "deletionCost" in pod and pod["deletionCost"] is not None:
        cost += _div(float(pod["deletionCost"]), 2.0 ** 27)
    if "priority" in pod and pod["priority"] is not None:
        cost += _div(float(pod["priority"]), 2.0 ** 25)
    return clamp(-10.0, cost, 10.0)


def lifetime_remaining(problem, node, prov):  # helpers.go:275-287
    if prov.get("ttlSecondsUntilExpired") is None:
        return 1.0
    age = float(problem.get("now", 0.0)) - float(node.get("creationTimestamp", 0.0))
    total = float(prov["ttlSecondsUntilExpired"])
    return clamp(0.0, _div(total - age, total), 1.0)


def disruption_cost(problem, node):  # helpers.go:159-165: summed in pod order
    prov = next(p for p in problem["provisioners"] if p["name"] == node["labels"][PROVISIONER_NAME])
    c = 0.0
    for p in node.get("pods", []):
        c += pod_eviction_cost(p)
    return c * lifetime_remaining(problem, node, prov)


def ranked(problem, eligible):
    """sort.Slice by disruption cost over the eligible nodes, stable (R4), NaN after every number and stable among NaNs (R8)
    -> (node indices, costs)"""
    costs = {i: disruption_cost(problem, problem["nodes"][i]) for i in eligible}
    order = sorted(eligible, key=lambda i: (1, 0.0) if math.isnan(costs[i]) else (0, costs[i]))
    return order, [costs[i] for i in order]
