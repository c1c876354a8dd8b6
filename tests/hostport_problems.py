"""Seeded corpus of clusters whose pods name more than 64 distinct host-port entries (DESIGN.md §3, host ports beyond the
word). hostNetwork pods get hostPort = containerPort for every declared port, so node agents, ingress controllers and game
servers add up entries quickly, whether or not the batch uses a host port.

 * daemonsets(n_nodes, seed, batch): bound hostNetwork-style daemonset pods name 80-200 entries (one entry shared by every
   node, TCP and UDP on one port, node-specific IPs next to 0.0.0.0 and ::). batch "none" declares no port, "few" a handful
   that match some entries. The encoder's pruning leaves these under 64 entries, with no table;
 * games(n, seed): n deployments of 2-6 game servers with one port each from 7000-7999, some ports already held on existing
   nodes, mixed with zone spread, hostname anti-affinity and a preferred term that relaxes. More than 64 entries survive;
 * traps(seed): a specific IP against 0.0.0.0 on one port, two specific IPs that both match one wildcard but not each other,
   the same port in the other protocol, one pod with two containers on one port, and a class whose only entries have ids of
   64 and above (its row words are zero). Filler nodes first: they are full, and their entries take ids 0-69;
 * boundary(kind): exactly 64 entries ("fit64"), 65 entries that prune to 64 ("prune65"), 65 that prune to 65 ("keep65");
 * cluster(seed) / after(seed): game-server nodes for the consolidation session, and the same cluster after the TTL with some
   host-port pods moved;
 * kept_entries / node_conflicts: the encoder's entry table and HostPortUsage's rule restated on the problem's strings.
"""
import copy
import random

import fixtures as fx
from fixtures import HOSTNAME, ZONE, ZONES


def port(p, ip="", proto="TCP"):
    return {"hostPort": p, "hostIP": ip, "protocol": proto}


def _node(name, rng, pods, full=False, **kw):
    it = rng.choice(["fake-it-7", "fake-it-11", "fake-it-15"])
    cpu = int(it.split("-")[-1]) + 1
    alloc = {"cpu": "50m" if full else f"{cpu * 1000 - 100}m", "memory": f"{cpu * 2 - 1}Gi", "pods": str(cpu * 10)}
    return fx.state_node(name, it, zone=rng.choice(ZONES), capacity_type=rng.choice(["on-demand", "spot"]), allocatable=alloc,
                         capacity=dict(alloc, cpu=f"{cpu}"), pods_=pods, **kw)


def _bound(name, app, ports, ds=True, cpu="10m"):
    return fx.pod({"cpu": cpu, "memory": "16Mi"}, nodeName=name, isDaemonSet=ds, labels={"app": app}, ports=list(ports))


def _pods(n, requests, ports=(), **kw):
    return [fx.pod(dict(requests), **(dict(kw, ports=list(ports)) if ports else kw)) for _ in range(n)]


def _problem(pods, nodes):
    return fx.problem(pods, instance_types=fx.fake_instance_types(16), nodes=nodes)


# ---------------------------------------------------------------- daemonset ports
def _agents(name, i):
    ip = f"10.1.{i // 200}.{i % 200 + 1}"
    out = [_bound(name, "node-exporter", [port(9100)]),
           _bound(name, "dns-cache", [port(53, "169.254.20.10"), port(53, "169.254.20.10", "UDP")]),
           _bound(name, "cni", [port(9099, "::")])]
    if i % 2 == 0:
        out.append(_bound(name, "ingress", [port(80, ip), port(443, ip)]))
    if i % 3 == 0:
        out.append(_bound(name, "log-shipper", [port(24224, ip), port(24224, ip, "UDP")]))
    return out


def daemonsets(n_nodes, seed, batch):
    rng = random.Random(seed * 31 + n_nodes)
    nodes = [_node(f"n-{i:03d}", rng, _agents(f"n-{i:03d}", i)) for i in range(n_nodes)]
    pods = _pods(40, {"cpu": "1", "memory": "1Gi"}, labels={"app": "web"})
    pods += _pods(9, {"cpu": "500m", "memory": "512Mi"}, labels={"app": "spread"}, topologySpreadConstraints=[fx.spread(ZONE, {"app": "spread"})])
    if batch == "few":
        pods += _pods(3, {"cpu": "250m"}, [port(9100)], labels={"app": "exporter-2"})          # every node's exporter entry
        pods += _pods(2, {"cpu": "250m"}, [port(53, "169.254.20.10", "UDP")], labels={"app": "dns-2"})  # the UDP entry only
        pods += _pods(2, {"cpu": "250m"}, [port(80, "10.1.0.5")], labels={"app": "ingress-5"})  # one node's ingress entry
        pods += _pods(2, {"cpu": "250m"}, [port(8080)], labels={"app": "fresh-port"})           # a port no node holds
    rng.shuffle(pods)
    return _problem(pods, nodes)


# ---------------------------------------------------------------- game servers
def games(n, seed, n_nodes=30):
    rng = random.Random(seed * 7 + n)
    gports = rng.sample(range(7000, 8000), n)
    held = rng.sample(gports, n // 5)  # ports of the batch already taken on some existing nodes
    nodes = []
    for i in range(n_nodes):
        name = f"g-{i:02d}"
        bound = [_bound(name, "node-exporter", [port(9100)])]
        for p in rng.sample(held, rng.choice([0, 1, 2])):
            bound.append(_bound(name, f"old-{p}", [port(p, proto="UDP" if p % 5 == 0 else "TCP")], ds=False, cpu="250m"))
        nodes.append(_node(name, rng, bound))
    pods = []
    for d, p in enumerate(gports):
        lab = {"app": f"gs-{d}"}
        kw = {"labels": lab}
        kind = d % 6
        if kind == 1:
            kw["topologySpreadConstraints"] = [fx.spread(ZONE, lab)]
        elif kind == 3:
            kw["podAntiAffinity"] = {"required": [fx.affinity_term(HOSTNAME, lab)]}
        elif kind == 4:
            kw["nodeAffinity"] = {"preferred": [{"weight": 10, "terms": [{"key": ZONE, "operator": "In", "values": ["nowhere"]}]}]}
        pods += _pods(rng.randint(2, 6), {"cpu": rng.choice(["250m", "500m", "1"]), "memory": "256Mi"},
                      [port(p, proto="UDP" if p % 5 == 0 else "TCP")], **kw)
    pods += _pods(30, {"cpu": "500m", "memory": "512Mi"}, labels={"app": "lobby"})
    rng.shuffle(pods)
    return _problem(pods, nodes)


# ---------------------------------------------------------------- wildcard and identity traps
def traps(seed):
    rng = random.Random(seed + 4242)
    # 70 full nodes first: their ports are entries 0-69 (a two-replica scanner deployment matches every one of them)
    nodes = [_node(f"f-{i:02d}", rng, [_bound(f"f-{i:02d}", "filler", [port(7000 + i)])], full=True) for i in range(70)]
    nodes.append(_node("x-wild", rng, [_bound("x-wild", "wild", [port(8080)])]))               # 0.0.0.0:8080
    nodes.append(_node("y-udp", rng, [_bound("y-udp", "udp", [port(8082, proto="UDP")])]))     # 8082 UDP only
    nodes += [_node(f"free-{i}", rng, []) for i in range(4)]
    pods = _pods(2, {"cpu": "100m"}, [port(7000 + i) for i in range(70)], labels={"app": "scanner"})
    pods += _pods(2, {"cpu": "100m"}, [port(8080, "10.9.0.1")], labels={"app": "specific"})      # not on x-wild
    pods += _pods(1, {"cpu": "100m"}, [port(8081, "10.9.0.1")], labels={"app": "b1"})           # b1 and b2 may share a node,
    pods += _pods(1, {"cpu": "100m"}, [port(8081, "10.9.0.2")], labels={"app": "b2"})           # neither with c
    pods += _pods(1, {"cpu": "100m"}, [port(8081)], labels={"app": "c"})
    pods += _pods(2, {"cpu": "100m"}, [port(8082)], labels={"app": "tcp"})                      # y-udp takes one
    pods += [fx.pod(labels={"app": "two-containers"}, containers=[{"requests": {"cpu": "100m"}, "ports": [port(9000)]},
                                                                  {"requests": {"cpu": "100m"}, "ports": [port(9000)]}])
             for _ in range(2)]
    pods += _pods(4, {"cpu": "100m"}, [port(9500)], labels={"app": "high-only"})  # entry id >= 64, no other: zero row words
    pods += _pods(6, {"cpu": "100m"}, labels={"app": "plain"})
    return _problem(pods, nodes)


# ---------------------------------------------------------------- boundaries
def boundary(kind):
    """bound pods hold 10.0.0.k:8080 (63 or 64 of them); two pending replicas declare 0.0.0.0:8080, which matches every one"""
    rng = random.Random({"fit64": 1, "prune65": 2, "keep65": 3}[kind])
    n = 64 if kind == "keep65" else 63
    nodes = [_node(f"free-{i}", rng, []) for i in range(2)]  # first in slice order: the replicas try them first
    nodes += [_node(f"b-{k:02d}", rng, [_bound(f"b-{k:02d}", "agent", [port(8080, f"10.0.0.{k + 1}")])]) for k in range(n)]
    if kind == "prune65":  # an entry no pending pod matches
        nodes.append(_node("b-9999", rng, [_bound("b-9999", "lonely", [port(9999, "10.0.0.1")])]))
    pods = _pods(2, {"cpu": "100m"}, [port(8080)], labels={"app": "wild"}) + _pods(4, {"cpu": "100m"}, labels={"app": "plain"})
    return _problem(pods, nodes)


# ---------------------------------------------------------------- consolidation
def cluster(seed, n_nodes=40, n_deploy=110, candidates=22):
    """game servers spread over the nodes, two replicas of each on different nodes; the first `candidates` nodes are
    consolidation candidates, whose pods hold more than 64 entries that another pod matches"""
    rng = random.Random(seed * 17 + 3)
    names = [f"c-{i:02d}" for i in range(n_nodes)]
    bound = {n: [_bound(n, "node-exporter", [port(9100)])] for n in names}
    for d, p in enumerate(rng.sample(range(7000, 8000), n_deploy)):
        for n in rng.sample(names, 2):
            bound[n].append(_bound(n, f"gs-{d}", [port(p)], ds=False, cpu="200m"))
    nodes = [_node(n, rng, bound[n]) for n in names]
    for k in range(candidates):
        nodes[k].update(candidate=True, disruptionCost=float(rng.choice([0, 1, 2])), creationTimestamp=float(k))
    return _problem([], nodes)


def after(seed):
    """cluster(seed) after the TTL: a dozen game servers moved to other nodes, and a new pending one"""
    a = copy.deepcopy(cluster(seed))
    rng = random.Random(seed + 77)
    for _ in range(12):
        src, dst = rng.sample(a["nodes"], 2)
        movable = [p for p in src["pods"] if not p.get("isDaemonSet")]
        if not movable:
            continue
        p = rng.choice(movable)
        src["pods"].remove(p)
        p["nodeName"] = dst["name"]
        dst["pods"].append(p)
    a["pods"] = _pods(1, {"cpu": "200m"}, [port(7999)], labels={"app": "late"})
    return a


def corpus():
    """[(name, problem dict, expects a table)]"""
    return [("ds-none-60", daemonsets(60, 0, "none"), False), ("ds-few-60", daemonsets(60, 0, "few"), False),
            ("ds-few-120", daemonsets(120, 1, "few"), False),
            ("games-100", games(100, 0), True), ("games-300", games(300, 1), True), ("traps", traps(0), True),
            ("fit64", boundary("fit64"), False), ("prune65", boundary("prune65"), False), ("keep65", boundary("keep65"), True)]


# ---------------------------------------------------------------- the reference's rules, restated
def pod_ports(p):
    """getHostPorts (hostportusage.go:118-144) in the loader's container order: `containers`, then the pod-level one"""
    decl = [hp for c in p.get("containers", []) for hp in c.get("ports", [])]
    if any(k in p for k in ("requests", "limits", "ports")):
        decl += p.get("ports", [])
    return [(hp.get("hostIP") or "0.0.0.0", hp["hostPort"], hp.get("protocol", "TCP")) for hp in decl if hp.get("hostPort")]


def matches(a, b):
    """HostPort.matches (hostportusage.go:45-57)"""
    wild = ("0.0.0.0", "::")
    return a[2] == b[2] and a[1] == b[1] and (a[0] == b[0] or a[0] in wild or b[0] in wild)


def kept_entries(prob, candidates=()):
    """(every entry in id order, the entries the encoder keeps in id order): first appearance over the owned state nodes'
    bound pods, then the batch; with more than 64, an entry stays iff a pod holds it and a DIFFERENT pod of the batch has a
    port that matches it"""
    cand = set(candidates)
    stay = [n for i, n in enumerate(prob["nodes"]) if i not in cand and n["labels"].get(fx.PROVISIONER_NAME)]
    batch = list(prob["pods"]) + [p for i in candidates for p in prob["nodes"][i]["pods"]
                                  if not p.get("isDaemonSet") and not p.get("terminal") and not p.get("terminating")]
    holders = [(id(p), pod_ports(p)) for n in stay for p in n["pods"]] + [(id(p), pod_ports(p)) for p in batch]
    seen = list(dict.fromkeys(e for _, ports in holders for e in ports))
    if len(seen) <= 64:
        return seen, seen
    held = {e: {h for h, ports in holders if e in ports} for e in seen}
    matched = {e: {id(p) for p in batch if any(matches(a, e) for a in pod_ports(p))} for e in seen}
    return seen, [e for e in seen if any(q != p for q in held[e] for p in matched[e])]


def node_conflicts(prob, res):
    """pods of the result that share a node with a different pod holding an entry one of their ports matches"""
    bad = []
    members = [[(("bound", j), pod_ports(q)) for j, q in enumerate(prob["nodes"][e["node"]]["pods"])] +
               [(("pod", i), pod_ports(prob["pods"][i])) for i in e["pods"]] for e in res["existing"]]
    members += [[(("pod", i), pod_ports(prob["pods"][i])) for i in n["pods"]] for n in res["newNodes"]]
    for m in members:
        for who, ports in m:
            if who[0] != "pod":
                continue
            for other, held in m:
                if other != who and any(matches(a, e) for a in ports for e in held):
                    bad.append((who, other))
    return bad
