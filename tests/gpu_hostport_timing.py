"""Timing of consolidation on a C5-shaped cluster (5 000 nodes, 50 000 bound pods) whose bound pods hold a few hundred
host-port entries, not part of bench.py. Every node runs a node-exporter daemonset pod (0.0.0.0:9100) and one game server
with a port of its own among --ports (each port held on several nodes, so consolidation moves pods that conflict with
entries kept on other nodes: host-port entry ids from 64 on, read from the entry tables). Run twice: with the ports and with
every port stripped. Times the multi-node search and the single-node sweep over every candidate, medians of --reps, and
prints one JSON line per run with the card name and power limit read in the same run.

    python tests/gpu_hostport_timing.py [--reps R] [--ports N] [--out FILE]
"""
import argparse

import fixtures as fx
import hostport_problems as hp
from timing_lib import card, emit, load_pkg, need_device, sweep_singles, timed


def c5_dict(ports, nodes=5000, pods_per_node=10, types=1000):
    its = fx.fake_instance_types(types)
    big = its[-1]
    provs = [fx.provisioner("default", consolidationEnabled=True, limits=None)]
    ns = []
    for i in range(nodes):
        name = f"n{i}"
        pods_ = [fx.pod({"cpu": "100m", "memory": "128Mi"}, nodeName=name, labels={"app": f"a{j % 50}"}) for j in range(pods_per_node - 2)]
        exporter = fx.pod({"cpu": "10m", "memory": "16Mi"}, nodeName=name, isDaemonSet=True, labels={"app": "node-exporter"})
        game = fx.pod({"cpu": "250m", "memory": "256Mi"}, nodeName=name, labels={"app": f"gs-{i % max(ports, 1)}"})
        if ports:
            exporter["ports"] = [hp.port(9100)]
            game["ports"] = [hp.port(7000 + i % ports)]
        ns.append(fx.state_node(name, big["name"], zone=fx.ZONES[i % 3], allocatable=big["capacity"], pods_=pods_ + [exporter, game]))
    return fx.problem([], instance_types=its, provisioners=provs, nodes=ns, deriveCandidates=True)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--ports", type=int, default=300)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    pkg = load_pkg()
    need_device(pkg)
    gpu = card()
    lines = []
    for ports in (a.ports, 0):
        d = c5_dict(ports)
        problem = pkg.Problem.from_dict(d)
        line = {"card": gpu, "nodes": len(d["nodes"]), "bound_pods": sum(len(n["pods"]) for n in d["nodes"]),
                "host_port_entries": len({e for n in d["nodes"] for p in n["pods"] for e in hp.pod_ports(p)})}
        multi = pkg.MultiNodeConsolidation(problem)
        line["multi_node_search_ms"], r = timed(multi.first_n_node_consolidation_option, a.reps)
        line["multi_node_action"], line["multi_node_removed"] = r["action"], r["nodes_removed"]

        line["single_node_sweep_ms"], acts = timed(lambda: sweep_singles(pkg, problem), a.reps)
        line["single_node_candidates"] = len(acts)
        line["single_node_actionable"] = sum(1 for x in acts if x in (1, 2))
        lines.append(line)
    emit(lines, a.out)


if __name__ == "__main__":
    main()
