"""Seeded corpus of daemonsets whose node selector or node affinity names node.kubernetes.io/instance-type (DESIGN.md §3,
daemonset overhead). Device-plugin daemonsets pick their nodes this way: the Neuron plugin by inf2 / trn1 types, the EFA
plugin by a list of EFA-capable types. The catalog mixes general types with inf2 / trn1 / p4d-like ones.

 * neuron(seed): a tainted neuron pool with an instance-type requirement and a general pool with neither; the plugin
   tolerates only the neuron taint and is charged on both templates (the general one does not define the key);
 * efa(seed): an Exists toleration; pools whose type lists do and do not meet the plugin's list;
 * operators(seed): the beta alias key, NotIn, Exists, DoesNotExist, Gt and Lt against pools with In, NotIn, labelled and
   no instance-type requirement;
 * terms(seed): instance-type requirements in the node selector, in the heaviest preferred term (a lighter one is ignored)
   and in a second required term (ignored: NewPodRequirements reads the first);
 * existing(seed): existing nodes of selected and unselected types, of a type outside the catalog, without the label,
   already running the daemon pod, tainted and tolerated, and a hostname daemonset that tolerates no template;
 * miscount(seed): a daemon no template admits, selecting a type that existing node n-0 is not; an 800m pod fits n-0 only
   when that daemon is not charged there;
 * cluster(seed) / after(seed): a consolidation cluster of 60 nodes, and the same cluster after the TTL with a new plugin
   daemonset rolled out;
 * near_misses(): daemons with a hostname requirement that a template admits, alone and with an instance-type one.

template_overhead / existing_overhead / former_existing_overhead restate getDaemonOverhead and calculateExistingMachines
(scheduler.go:221-267) on strings, for the tests.
"""
import copy
import random

import exact_arith as ea
import fixtures as fx
from fixtures import CAPACITY_TYPE, HOSTNAME, INSTANCE_TYPE, PROVISIONER_NAME, ZONE, ZONES

BETA_INSTANCE_TYPE = "beta.kubernetes.io/instance-type"
NEURON, GPU, EFA = "aws.amazon.com/neuron", "nvidia.com/gpu", "vpc.amazonaws.com/efa"
NEURON_TAINT = {"key": NEURON, "value": "true", "effect": "NoSchedule"}
NEURON_TYPES = ["inf2.xlarge", "inf2.8xlarge", "trn1.2xlarge", "trn1.32xlarge"]
EFA_TYPES = ["p4d.24xlarge", "trn1.32xlarge", "c5n.18xlarge"]
SMALL_TYPES = ["t3.nano", "t3.micro"]


def catalog():
    """general types, then inf2 / trn1 / p4d-like ones carrying accelerator and EFA resources"""
    spec = [("t3.nano", "2", "512Mi", {}), ("t3.micro", "2", "1Gi", {}), ("m5.large", "2", "8Gi", {}), ("m5.xlarge", "4", "16Gi", {}),
            ("m5.2xlarge", "8", "32Gi", {}), ("c5.xlarge", "4", "8Gi", {}), ("c5.4xlarge", "16", "32Gi", {}),
            ("c5n.18xlarge", "72", "192Gi", {EFA: "1"}), ("inf2.xlarge", "4", "16Gi", {NEURON: "1"}),
            ("inf2.8xlarge", "32", "128Gi", {NEURON: "1"}), ("trn1.2xlarge", "8", "32Gi", {NEURON: "1"}),
            ("trn1.32xlarge", "128", "512Gi", {NEURON: "16", EFA: "8"}), ("p4d.24xlarge", "96", "1152Gi", {GPU: "8", EFA: "4"})]
    out = []
    for name, cpu, mem, extra in spec:
        cpus = int(cpu)
        out.append(fx.instance_type(name, dict({"cpu": cpu, "memory": mem, "pods": str(min(110, 8 + cpus * 4))}, **extra)))
    return out


TYPES = catalog()


def _it(op, values=(), key=INSTANCE_TYPE):
    r = {"key": key, "operator": op}
    if values:
        r["values"] = list(values)
    return r


def _daemon(cpu="100m", mem="128Mi", **kw):
    return fx.pod({"cpu": cpu, "memory": mem}, **kw)


def _pods(n, cpu="1", mem="1Gi", **kw):
    return [fx.pod({"cpu": cpu, "memory": mem}, **kw) for _ in range(n)]


def _node(name, itype, rng, cpu=8, pods=None, **kw):
    alloc = {"cpu": f"{cpu * 1000 - 100}m", "memory": f"{cpu * 4}Gi", "pods": str(cpu * 10)}
    return fx.state_node(name, itype, zone=rng.choice(ZONES), allocatable=alloc, capacity=dict(alloc, cpu=str(cpu)), pods_=pods or [], **kw)


def _problem(pods, daemons, nodes=(), provisioners=None, types=None, **kw):
    return fx.problem(pods, instance_types=types or TYPES, provisioners=provisioners, nodes=list(nodes), daemonSetPods=daemons, **kw)


def _on(prov):
    return {PROVISIONER_NAME: prov}


NEURON_TOL = [{"key": NEURON, "operator": "Exists", "effect": "NoSchedule"}]


# ---------------------------------------------------------------- templates
def neuron(seed):
    rng = random.Random(seed + 11)
    prov = [fx.provisioner("neuron", weight=10, taints=[NEURON_TAINT], requirements=[_it("In", NEURON_TYPES)]),
            fx.provisioner("general")]
    plugin = _daemon("250m", "512Mi", tolerations=NEURON_TOL, nodeAffinity={"required": [[_it("In", NEURON_TYPES)]]})
    proxy = _daemon("100m", "64Mi", tolerations=[{"operator": "Exists"}])
    pods = [fx.pod({"cpu": "3", "memory": "8Gi", NEURON: "1"}, tolerations=NEURON_TOL, nodeSelector=_on("neuron"))
            for _ in range(rng.randint(6, 10))]
    pods += _pods(rng.randint(8, 14), cpu=rng.choice(["1", "1500m", "3500m"]), mem="2Gi")
    return _problem(pods, [plugin, proxy], provisioners=prov)


def efa(seed):
    rng = random.Random(seed + 22)
    prov = [fx.provisioner("gpu", weight=30, requirements=[_it("In", ["p4d.24xlarge", "m5.2xlarge"])]),
            fx.provisioner("cpu", weight=20, requirements=[_it("In", ["m5.large", "m5.xlarge", "c5.xlarge"])]),
            fx.provisioner("not-efa", weight=10, requirements=[_it("NotIn", EFA_TYPES)]),
            fx.provisioner("not-small", requirements=[_it("NotIn", SMALL_TYPES)])]
    plugin = _daemon("500m", "1Gi", tolerations=[{"operator": "Exists"}], nodeAffinity={"required": [[_it("In", EFA_TYPES)]]})
    pods = []
    for name in ("gpu", "cpu", "not-efa", "not-small"):
        pods += _pods(rng.randint(3, 6), cpu=rng.choice(["1", "1700m", "3"]), mem=rng.choice(["1Gi", "6Gi"]), nodeSelector=_on(name))
    rng.shuffle(pods)
    return _problem(pods, [plugin], provisioners=prov)


def operators(seed):
    rng = random.Random(seed + 33)
    prov = [fx.provisioner("small", weight=40, requirements=[_it("In", SMALL_TYPES + ["m5.large"])]),
            fx.provisioner("big", weight=30, requirements=[_it("NotIn", SMALL_TYPES)]),
            fx.provisioner("labelled", weight=20, labels={INSTANCE_TYPE: "m5.xlarge"}),
            fx.provisioner("any")]
    daemons = [_daemon("110m", "32Mi", nodeSelector={BETA_INSTANCE_TYPE: "m5.xlarge"}),
               _daemon("120m", "64Mi", nodeAffinity={"required": [[_it("NotIn", SMALL_TYPES)]]}),
               _daemon("130m", "96Mi", nodeAffinity={"required": [[_it("Exists")]]}),
               _daemon("140m", "128Mi", nodeAffinity={"required": [[_it("DoesNotExist")]]}),
               _daemon("150m", "160Mi", nodeAffinity={"required": [[_it("Gt", ["3"])]]}),
               _daemon("160m", "192Mi", nodeAffinity={"required": [[_it("Lt", ["100"], key=BETA_INSTANCE_TYPE)]]}),
               _daemon("170m", "224Mi", nodeAffinity={"required": [[_it("In", ["t3.micro", "m5.xlarge"]), _it("NotIn", ["t3.micro"])]]})]
    pods = []
    for name in ("small", "big", "labelled", "any"):
        pods += _pods(rng.randint(3, 6), cpu=rng.choice(["500m", "1", "1500m"]), mem=rng.choice(["256Mi", "1Gi"]), nodeSelector=_on(name))
    rng.shuffle(pods)
    return _problem(pods, daemons, provisioners=prov)


def terms(seed):
    rng = random.Random(seed + 44)
    prov = [fx.provisioner("compute", weight=10, requirements=[_it("In", ["c5.xlarge", "c5.4xlarge"])]), fx.provisioner("general")]
    in_selector = _daemon("200m", "64Mi", nodeSelector={INSTANCE_TYPE: "c5.4xlarge"})
    preferred = _daemon("300m", "128Mi", nodeAffinity={"preferred": [{"weight": 10, "terms": [_it("In", ["c5.xlarge"])]},
                                                                     {"weight": 50, "terms": [_it("In", ["m5.large"])]}]})
    second_term = _daemon("400m", "256Mi", nodeAffinity={"required": [[_it("In", ZONES, key=ZONE)], [_it("In", ["no-such-type"])]]})
    first_term = _daemon("450m", "256Mi", nodeAffinity={"required": [[_it("In", ["no-such-type"])], [_it("In", ZONES, key=ZONE)]]})
    pods = _pods(rng.randint(4, 8), cpu=rng.choice(["1", "2500m"]), nodeSelector=_on("compute"))
    pods += _pods(rng.randint(4, 8), cpu=rng.choice(["700m", "1", "3"]), mem="3Gi")
    return _problem(pods, [in_selector, preferred, second_term, first_term], provisioners=prov)


# ---------------------------------------------------------------- existing nodes
def existing(seed):
    rng = random.Random(seed + 55)
    prov = [fx.provisioner("infra", taints=[{"key": "dedicated", "value": "infra", "effect": "NoSchedule"}]),
            fx.provisioner("neuron", taints=[NEURON_TAINT], requirements=[_it("In", NEURON_TYPES)])]
    plugin = _daemon("600m", "1Gi", tolerations=NEURON_TOL + [{"key": "dedicated", "operator": "Exists"}],
                     nodeAffinity={"required": [[_it("In", NEURON_TYPES + ["inf1.xlarge"])]]})
    hosts = ["e-01", "e-04", "e-07"]
    local = _daemon("700m", "512Mi", nodeAffinity={"required": [[_it("In", hosts, key=HOSTNAME)]]})
    gt = _daemon("300m", "256Mi", nodeAffinity={"required": [[_it("Gt", ["4"])]]})
    types = ["inf2.xlarge", "m5.xlarge", "trn1.2xlarge", "inf1.xlarge", "c5.xlarge", "inf2.8xlarge", "16", "m5.2xlarge", "inf2.xlarge"]
    nodes = []
    for i, t in enumerate(types):
        name = f"e-{i:02d}"
        n = _node(name, t, rng, cpu=4, provisioner_name="neuron" if t in NEURON_TYPES else "infra")
        n["pods"] = [fx.pod({"cpu": "500m", "memory": "512Mi"}, nodeName=name) for _ in range(rng.randint(0, 2))]
        nodes.append(n)
    del nodes[4]["labels"][INSTANCE_TYPE]  # no label: compatible with every instance-type requirement
    nodes[5]["pods"].append(dict(copy.deepcopy(plugin), nodeName="e-05", isDaemonSet=True, name="plugin-e-05", uid="uid-plugin-e-05"))
    nodes[8]["taints"] = [NEURON_TAINT]  # tolerated by the plugin only
    nodes[2]["taints"] = [{"key": "dedicated", "value": "infra", "effect": "NoSchedule"}]
    pods = _pods(rng.randint(10, 16), cpu=rng.choice(["600m", "900m", "1200m"]), mem="1Gi")
    pods += _pods(4, cpu="800m", mem="1Gi", tolerations=[{"operator": "Exists"}])
    return _problem(pods, [plugin, local, gt], nodes, provisioners=prov)


def miscount(seed):
    """the daemon selects single-pod-instance-type and tolerates no template; n-0 is a default-instance-type node of 1 cpu"""
    rng = random.Random(seed + 66)
    prov = [fx.provisioner("tainted", taints=[{"key": "team", "value": "a", "effect": "NoSchedule"}])]
    ds = fx.pod({"cpu": "500m"}, nodeAffinity={"required": [[_it("In", ["single-pod-instance-type"])]]})
    nodes = [fx.state_node("n-0", "default-instance-type", allocatable={"cpu": "1", "memory": "4Gi", "pods": "5"}),
             fx.state_node("n-1", "single-pod-instance-type", zone=rng.choice(ZONES), allocatable={"cpu": "1", "memory": "4Gi", "pods": "5"})]
    return _problem([fx.pod({"cpu": "800m"})], [ds], nodes, provisioners=prov, types=fx.default_instance_types())


# ---------------------------------------------------------------- consolidation
CLUSTER_TYPES = ["m5.large", "m5.xlarge", "m5.2xlarge", "c5.xlarge", "c5.4xlarge", "inf2.xlarge", "trn1.2xlarge", "p4d.24xlarge"]


def _cluster_daemons():
    neuron_plugin = _daemon("200m", "256Mi", tolerations=[{"operator": "Exists"}], nodeAffinity={"required": [[_it("In", NEURON_TYPES)]]})
    efa_plugin = _daemon("300m", "256Mi", tolerations=[{"operator": "Exists"}], nodeAffinity={"required": [[_it("In", EFA_TYPES)]]})
    return [neuron_plugin, efa_plugin]


def _sizes(t):
    it = next(x for x in TYPES if x["name"] == t)
    return int(it["capacity"]["cpu"])


def cluster(seed, n_nodes=60, candidates=24):
    """nodes of general, neuron and GPU types with web pods; the plugins' pods are bound on the nodes they select"""
    rng = random.Random(seed * 23 + 5)
    daemons = _cluster_daemons()
    prov = [fx.provisioner("default", limits={"cpu": "4000"})]
    nodes = []
    for i in range(n_nodes):
        x, t = f"c-{i:02d}", CLUSTER_TYPES[rng.randrange(len(CLUSTER_TYPES))] if i % 3 else CLUSTER_TYPES[i % 5]
        cpu = min(_sizes(t), 16)
        bound = [fx.pod({"cpu": rng.choice(["300m", "700m", "1"]), "memory": "512Mi"}, nodeName=x, labels={"app": "web"})
                 for _ in range(rng.randint(1, max(1, cpu // 2)))]
        for d, sel in zip(daemons, (NEURON_TYPES, EFA_TYPES)):
            if t in sel:
                bound.append(dict(copy.deepcopy(d), nodeName=x, isDaemonSet=True, name=f"ds-{x}-{len(bound)}", uid=f"uid-ds-{x}-{len(bound)}"))
        nodes.append(_node(x, t, rng, cpu=cpu, pods=bound))
    for k in range(candidates):
        nodes[k].update(candidate=True, disruptionCost=float(rng.choice([0, 1, 2])), creationTimestamp=float(k))
    return _problem([], daemons, nodes, provisioners=prov)


def after(seed):
    """cluster(seed) after the TTL: a new plugin daemonset (general types only) rolled out and bound where it runs, a few
    web pods moved, and a pending pod"""
    a = copy.deepcopy(cluster(seed))
    rng = random.Random(seed + 77)
    monitor = _daemon("250m", "256Mi", nodeAffinity={"required": [[_it("NotIn", NEURON_TYPES + ["p4d.24xlarge"])]]})
    a["daemonSetPods"].append(monitor)
    for n in a["nodes"]:
        if n["labels"][INSTANCE_TYPE] not in NEURON_TYPES + ["p4d.24xlarge"] and rng.random() < 0.7:
            n["pods"].append(dict(copy.deepcopy(monitor), nodeName=n["name"], isDaemonSet=True, name=f"mon-{n['name']}", uid=f"uid-mon-{n['name']}"))
    for _ in range(6):
        src, dst = rng.sample(a["nodes"], 2)
        movable = [p for p in src["pods"] if p.get("labels", {}).get("app") == "web"]
        if movable:
            p = rng.choice(movable)
            src["pods"].remove(p)
            p["nodeName"] = dst["name"]
            dst["pods"].append(p)
    a["pods"] = _pods(1, cpu="300m", mem="256Mi")
    return a


# ---------------------------------------------------------------- refused
def near_misses():
    rng = random.Random(5)
    nodes = [_node(f"m-{i}", "m5.xlarge", rng) for i in range(3)]
    host = _daemon(nodeAffinity={"required": [[_it("In", ["m-0", "m-1"], key=HOSTNAME)]]})
    both = _daemon(nodeAffinity={"required": [[_it("In", ["m-0"], key=HOSTNAME), _it("In", ["m5.xlarge"])]]})
    return [("hostname", _problem(_pods(2), [host], nodes)), ("hostname-and-instance-type", _problem(_pods(2), [both], nodes))]


def known_answers():
    """provisioning/suite_test.go:475-530 ("Daemonsets and Node Overhead") and instance-type cases in their style:
    [(name, problem dict, (cpu, memory) capacity of the type launched for the one pod)]. The daemon requests 1 cpu / 1Gi,
    so it is charged exactly where the answer is the 4-cpu default type rather than the 2-cpu small one."""
    req = {"cpu": "1", "memory": "1Gi"}
    two = ["small-instance-type", "default-instance-type"]
    cases = [("invalid-selector", {"nodeSelector": {"node": "invalid"}}, None, ("2", "2Gi")),
             ("notin-unspecified-key", {"nodeAffinity": {"required": [[_it("NotIn", ["bar"], key="foo")]]}}, None, ("4", "4Gi")),
             ("itype-in-template-without-key", {"nodeSelector": {INSTANCE_TYPE: "small-instance-type"}}, None, ("4", "4Gi")),
             ("itype-in-disjoint", {"nodeAffinity": {"required": [[_it("In", ["arm-instance-type"])]]}}, [_it("In", two)], ("2", "2Gi")),
             ("itype-notin-overlap", {"nodeAffinity": {"required": [[_it("NotIn", ["small-instance-type"])]]}}, [_it("In", two)], ("4", "4Gi")),
             ("itype-notin-both", {"nodeAffinity": {"required": [[_it("NotIn", ["gpu-vendor-instance-type"], key=BETA_INSTANCE_TYPE)]]}},
              [_it("NotIn", ["arm-instance-type"])], ("4", "4Gi")),
             ("itype-gt-names", {"nodeAffinity": {"required": [[_it("Gt", ["1"])]]}}, [_it("In", two)], ("2", "2Gi")),
             ("itype-dne-vs-in", {"nodeAffinity": {"required": [[_it("DoesNotExist")]]}}, [_it("In", two)], ("2", "2Gi"))]
    out = []
    for name, ds_kw, prov_reqs, want in cases:
        pod_kw = {"nodeAffinity": {"required": [[_it("In", ["test-zone-2"], key=ZONE)]]}} if name == "notin-unspecified-key" else {}
        prov = [fx.provisioner(requirements=prov_reqs)] if prov_reqs else None
        out.append((name, fx.problem([fx.pod(req, **pod_kw)], provisioners=prov, daemonSetPods=[fx.pod(req, **ds_kw)]), want))
    return out


def corpus():
    """[(name, problem dict)]"""
    return [("neuron", neuron(0)), ("neuron-1", neuron(1)), ("efa", efa(0)), ("operators", operators(0)), ("terms", terms(0)),
            ("existing", existing(0)), ("existing-1", existing(1)), ("miscount", miscount(0)), ("cluster-after", after(0))]


# ---------------------------------------------------------------- the reference's rules, restated on strings
def normalize(key):  # v1alpha5.NormalizedLabels (labels.go:103-109)
    return {"failure-domain.beta.kubernetes.io/zone": ZONE, "beta.kubernetes.io/arch": "kubernetes.io/arch",
            "beta.kubernetes.io/os": "kubernetes.io/os", BETA_INSTANCE_TYPE: INSTANCE_TYPE,
            "failure-domain.beta.kubernetes.io/region": "topology.kubernetes.io/region"}.get(key, key)


def _int(v):
    try:
        return int(v)
    except ValueError:
        return None


class Req:
    """scheduling.Requirement on strings (requirement.go:44-197)"""

    def __init__(self, comp, values, gt=None, lt=None):
        self.comp, self.values, self.gt, self.lt = comp, set(values), gt, lt

    @staticmethod
    def new(op, values=()):
        if op == "In":
            return Req(False, values)
        if op == "NotIn":
            return Req(True, values)
        if op == "Exists":
            return Req(True, ())
        if op == "DoesNotExist":
            return Req(False, ())
        return Req(True, (), gt=int(values[0])) if op == "Gt" else Req(True, (), lt=int(values[0]))

    def _within(self, v, gt, lt):
        if gt is None and lt is None:
            return True
        x = _int(v)
        return x is not None and (gt is None or x > gt) and (lt is None or x < lt)

    def intersection(self, o):
        gt = max((x for x in (self.gt, o.gt) if x is not None), default=None)
        lt = min((x for x in (self.lt, o.lt) if x is not None), default=None)
        if gt is not None and lt is not None and gt >= lt:
            return Req(False, ())
        comp = self.comp and o.comp
        if self.comp and o.comp:
            vals = self.values | o.values
        elif self.comp:
            vals = o.values - self.values
        elif o.comp:
            vals = self.values - o.values
        else:
            vals = self.values & o.values
        vals = {v for v in vals if self._within(v, gt, lt)}
        return Req(comp, vals, gt, lt) if comp else Req(False, vals)

    def empty(self):  # Len() == 0
        return not self.comp and not self.values

    def negative(self):  # Operator() is NotIn or DoesNotExist
        return bool(self.values) if self.comp else not self.values


def requirements(reqs):
    """Requirements.Add of a list of NodeSelectorRequirements"""
    out = {}
    for r in reqs:
        k, q = normalize(r["key"]), Req.new(r["operator"], r.get("values", ()))
        out[k] = q.intersection(out[k]) if k in out else q
    return out


def label_requirements(labels):
    return requirements([{"key": k, "operator": "In", "values": [v]} for k, v in labels.items()])


def pod_requirements(pod):
    """NewPodRequirements (requirements.go:61-78): node selector, the heaviest preferred term, the first required term"""
    reqs = [{"key": k, "operator": "In", "values": [v]} for k, v in (pod.get("nodeSelector") or {}).items()]
    na = pod.get("nodeAffinity") or {}
    pref = sorted(na.get("preferred") or [], key=lambda t: -t["weight"])
    if pref:
        reqs += pref[0]["terms"]
    if na.get("required"):
        reqs += na["required"][0]
    return requirements(reqs)


def well_known(problem):
    return {PROVISIONER_NAME, ZONE, "topology.kubernetes.io/region", INSTANCE_TYPE, "kubernetes.io/arch", "kubernetes.io/os",
            CAPACITY_TYPE} | set(problem.get("wellKnownLabels", []))


def compatible(node, inc, wk):
    """Requirements.Compatible (requirements.go:123-133, Intersects :189-206), `node` the receiver"""
    for k, q in inc.items():
        if k not in wk and k not in node and not q.negative():
            return False
    for k in node.keys() & inc.keys():
        if node[k].intersection(inc[k]).empty() and not (inc[k].negative() and node[k].negative()):
            return False
    return True


def _tolerates(taints, pod):
    def one(t, taint):
        if t.get("effect") and t["effect"] != taint.get("effect"):
            return False
        if t.get("key") and t["key"] != taint["key"]:
            return False
        if t.get("operator", "Equal") in ("", "Equal"):
            return t.get("value", "") == taint.get("value", "")
        return t["operator"] == "Exists"
    return all(any(one(t, taint) for t in pod.get("tolerations", [])) for taint in taints)


def template_requirements(prov):
    """NewMachineTemplate (machinetemplate.go:46-62): the provisioner's requirements, its labels and its name label"""
    labels = dict(prov.get("labels") or {}, **{PROVISIONER_NAME: prov["name"]})
    return requirements(list(prov.get("requirements") or []) + [{"key": k, "operator": "In", "values": [v]} for k, v in labels.items()])


def template_overhead(problem):
    """getDaemonOverhead (scheduler.go:250-267): per template, in weight order, the requests of the daemons it runs"""
    wk = well_known(problem)
    provs = problem["provisioners"]
    out = []
    for pi in ea._templates(problem):
        tr = template_requirements(provs[pi])
        ds = [d for d in problem.get("daemonSetPods", []) if _tolerates(provs[pi].get("taints", []), d) and compatible(tr, pod_requirements(d), wk)]
        out.append(ea.requests_for_pods(ds))
    return out


def _owned(problem, candidates, superset):
    cand = set(candidates)
    return [i for i, n in enumerate(problem.get("nodes", [])) if (superset or i not in cand) and not n.get("markedForDeletion")
            and n.get("labels", {}).get(PROVISIONER_NAME)]


def _existing(problem, candidates, superset, keep):
    wk = well_known(problem)
    out = []
    for i in _owned(problem, candidates, superset):
        n = problem["nodes"][i]
        ds = [d for d in problem.get("daemonSetPods", []) if _tolerates(n.get("taints", []), d) and keep(n, d, wk)]
        bound = ea.requests_for_pods([p for p in n.get("pods", []) if p.get("isDaemonSet")])
        out.append((i, {k: max(v, 0) for k, v in ea._subtract(ea.requests_for_pods(ds), bound).items()}))
    return out


def existing_overhead(problem, candidates=(), superset=False):
    """calculateExistingMachines (scheduler.go:221-248): [(node index, remaining daemon requests)] of the existing nodes"""
    return _existing(problem, candidates, superset, lambda n, d, wk: compatible(label_requirements(n["labels"]), pod_requirements(d), wk))


def former_existing_overhead(problem, candidates=(), superset=False):
    """the rule the encoder used before: the node's and the daemon's hostname and instance-type requirements were not read"""
    def keep(n, d, wk):
        strip = lambda rs: {k: q for k, q in rs.items() if k not in (HOSTNAME, INSTANCE_TYPE)}
        return compatible(strip(label_requirements(n["labels"])), strip(pod_requirements(d)), wk)
    return _existing(problem, candidates, superset, keep)
