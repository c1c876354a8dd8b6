"""Problems at the numeric limits of the int64 milli-unit arithmetic, the queue's packed sort key and the float64 candidate
ranking (tests/exact_arith.py restates what the answers must be):

  limits      provisioner limits against owned nodes whose capacities sum past 2^63 (4Ti x 2 090 / 2 100, 4Pi x 3), two
              provisioners one over and one under, a wrapped memory sum under a cpu-only limit, and a consolidation cluster
              whose remaining is over the limit until the candidates' capacity is given back
  quantities  milli values around 2^62 and INT64_MAX, negatives, mantissas of 39+ digits; container sums, init containers
              and daemonset overhead plus a request crossing 2^62
  queue       timestamps 0, 1.7e9, year 1 and year 9999 (and beyond metav1.Time), enough classes and pods that the packed
              queue key is wider than 64 bits before the timestamps are ranked, ties only the timestamp or the UID decides
  ranking     priority -2^31 and 1e9, deletion cost +-(2^31 - 1), +-Inf and NaN, costs exactly +-10, TTL 0 at age 0 and
              after it, a negative age, 256 and 257 equal costs across the ranking kernel's 256-node tile

Each scheduling entry is (name, problem, answer): answer is None or a predicate on the result dict that the reference's
exact arithmetic decides."""
import consolidation_answers as ca
import fixtures as fx
import ranking_answers as ra

INT64_MAX = 2 ** 63 - 1
B62 = 2 ** 62


def _it(name, res, price):
    """fx.instance_type with capacities it cannot read as floats (Pi, m): its labels are those of a small type"""
    it = fx.instance_type(name, {"cpu": "4", "memory": "4Gi"}, offerings=[{"capacityType": "on-demand", "zone": fx.ZONES[0], "price": price, "available": True}])
    it["capacity"] = dict(res)
    return it


def _owned(name, it, cap, pods_, provisioner="default", **kw):
    return fx.state_node(name, it, allocatable=dict(cap), capacity=dict(cap), pods_=pods_, provisioner_name=provisioner, **kw)


def _no_new_node(r):
    return not r["newNodes"]


# ---------------------------------------------------------------- quantity strings: (text, exact milli or None = must refuse)
QUANTITIES = [
    ("4611686018427387903m", B62 - 1), ("-4611686018427387903m", -(B62 - 1)), ("4611686018427387904m", None), ("-4611686018427387904m", None),
    ("9223372036854775807m", None), ("9223372036854775808m", None), ("4Pi", 4 * 2 ** 50 * 1000), ("4.1Pi", None), ("5Pi", None),
    ("-1", -1000), ("-0.5", -500), ("0.001", 1), ("1Ti", 2 ** 40 * 1000),
    ("123456789012345678901234567890123456789", None),                # 39 digits
    ("340282366920938463463374607431768211456m", None),               # 2^128: an __int128 mantissa wraps to 0
    ("170141183460469231731687303715884105728m", None),               # 2^127
    ("340282366920938463463374607431768211457m", None),               # 2^128 + 1 wraps to 1
    ("0.000000000000000000000000000000000000001", None),              # 39 fractional digits
    ("1.000000000000000000000000000000000000000", 1000),             # exact, or refused for its length
    ("00000000000000000000000000000000000000001", 1000),             # leading zeros
]


# ---------------------------------------------------------------- limits
def limit_wrap(n_nodes, cap_mem="4Ti", limits=None):
    """n owned nodes of 4 cpu / cap_mem, each holding a 3 900m pod, and one pending 1-cpu pod the nodes cannot take"""
    cap = {"cpu": "4", "memory": cap_mem, "pods": "110"}
    its = [_it("big", cap, 10.0), _it("small", {"cpu": "2", "memory": "4Gi", "pods": "110"}, 1.0)]
    nodes = [_owned(f"n{i}", "big", cap, [fx.pod({"cpu": "3900m"}, nodeName=f"n{i}")]) for i in range(n_nodes)]
    prov = {"name": "default", "limits": limits or {"memory": "1Ti"}}
    return fx.problem([fx.pod({"cpu": "1"})], instance_types=its, provisioners=[prov], nodes=nodes)


def two_provisioners():
    """'heavy' (weight 10) owns 3 x 4Pi of memory against a 1Ti limit, 'light' owns nothing: the pod goes to 'light'"""
    prob = limit_wrap(3, "4Pi")
    for n in prob["nodes"]:
        n["labels"][fx.PROVISIONER_NAME] = "heavy"
    prob["provisioners"] = [{"name": "light", "limits": {"memory": "1Ti"}}, {"name": "heavy", "weight": 10, "limits": {"memory": "1Ti"}}]
    return prob


def limits_corpus():
    # the weight order puts 'heavy' first: template 0 is heavy, template 1 light
    return [
        ("limit-4Ti-x2090", limit_wrap(2090), _no_new_node),
        ("limit-4Ti-x2100", limit_wrap(2100), _no_new_node),
        ("limit-4Pi-x3", limit_wrap(3, "4Pi"), _no_new_node),
        ("limit-two-provisioners", two_provisioners(), lambda r: [n["provisioner"] for n in r["newNodes"]] == [1]),
        ("limit-cpu-only-wrapped-memory", limit_wrap(3, "4Pi", {"cpu": "1000"}), lambda r: len(r["newNodes"]) == 1),
    ]


def limit_cluster(kept):
    """Three consolidatable nodes of 4Pi memory (one 1-cpu pod each) and `kept` full ones marked do-not-consolidate, under
    a 4Pi memory limit. With kept == 0 removing all three candidates gives the whole limit back and removing two leaves 0;
    with kept == 2 the exact remaining stays below zero whatever is removed, while the capacity given back to a remaining
    held at a floor would be far above it."""
    cap = {"cpu": "4", "memory": "4Pi", "pods": "110"}
    its = [_it("huge", cap, 10.0), _it("small", {"cpu": "4", "memory": "4Gi", "pods": "110"}, 1.0)]
    nodes = [_owned(f"c{i}", "huge", cap, [fx.pod({"cpu": "1"}, nodeName=f"c{i}")]) for i in range(3)]
    nodes += [_owned(f"k{i}", "huge", cap, [fx.pod({"cpu": "4"}, nodeName=f"k{i}")], doNotConsolidate="true") for i in range(kept)]
    prov = fx.provisioner(consolidationEnabled=True, limits={"memory": "4Pi"})
    return fx.problem([], instance_types=its, provisioners=[prov], nodes=nodes, deriveCandidates=True)


# ---------------------------------------------------------------- quantities inside problems
def _one_type_problem(pods_, mem="4Pi", **kw):
    its = [_it("big", {"cpu": "100", "memory": mem, "pods": "110"}, 10.0)]
    return fx.problem(pods_, instance_types=its, provisioners=[{"name": "default"}], **kw)


def quantity_corpus():
    """(name, problem, answer); answer None where the problem must be refused (a sum crosses 2^62)"""
    two = lambda q: {"containers": [{"requests": {"cpu": "1", "memory": q}}, {"requests": {"cpu": "1", "memory": q}}]}
    return [
        ("containers-sum-over", _one_type_problem([fx.pod(**{"containers": [{"requests": {"cpu": "1", "memory": "3.5Pi"}}] * 3})]), None),
        ("containers-sum-at-2^62", _one_type_problem([fx.pod(**two(f"{2 ** 61}m"))]), None),
        ("containers-sum-under", _one_type_problem([fx.pod(**two("1Pi"))]), lambda r: len(r["newNodes"]) == 1),
        ("init-container-max", _one_type_problem([fx.pod(**{"containers": [{"requests": {"cpu": "1", "memory": "1Pi"}}] * 3,
                                                             "initContainers": [{"requests": {"memory": "3.5Pi"}}]})]),
         lambda r: len(r["newNodes"]) == 1 and r["newNodes"][0]["requests"]["memory"] == 3.5 * 2 ** 50 * 1000),
        ("init-container-over-type", _one_type_problem([fx.pod(**{"containers": [{"requests": {"cpu": "1"}}],
                                                                   "initContainers": [{"requests": {"memory": "4Pi"}}]})], mem="3Pi"),
         lambda r: r["assign"] == [-1]),
        ("daemon-plus-request-over-2^62", _one_type_problem([fx.pod({"cpu": "1", "memory": "3Pi"})],
                                                             daemonSetPods=[fx.pod({"cpu": "1", "memory": "3Pi"})]),
         lambda r: r["assign"] == [-1]),
        ("daemons-sum-over", _one_type_problem([fx.pod({"cpu": "1"})], daemonSetPods=[fx.pod({"memory": "3.5Pi"}), fx.pod({"memory": "3.5Pi"})]), None),
        ("bound-pods-sum-over", _one_type_problem([fx.pod({"cpu": "1"})], nodes=[_owned("n0", "big", {"cpu": "100", "memory": "4Pi", "pods": "110"},
                                                                                        [fx.pod({"memory": "3.5Pi"}, nodeName="n0")] * 3)]), None),
        ("limits-stand-in-for-requests", _one_type_problem([fx.pod(**{"containers": [{"limits": {"cpu": "1", "memory": "3.5Pi"}}] * 2})]), None),
    ]


# ---------------------------------------------------------------- queue order
YEAR1, YEAR9999 = -62135596800, 253402300799
TIMESTAMPS = (0, 1_700_000_000, YEAR1, YEAR9999)


def queue_ties(n_classes, extreme=False):
    """`n_classes` pods of distinct cpu (one class each, so the class rank takes bits(n_classes - 1) bits) and, at the
    largest request, 8 pods of one class whose order only the timestamp decides (4 timestamps) or, at equal timestamps, the
    UID. One new node holds them all, in queue order. extreme: timestamps +-4e18 (accepted by the loader, beyond
    metav1.Time) so that the span alone is wider than 2^62."""
    ts = (-4 * 10 ** 18, 0, 4 * 10 ** 18, 1024) if extreme else TIMESTAMPS
    pods_ = [fx.pod({"cpu": f"{i + 1}m"}, creationTimestamp=ts[i % 4]) for i in range(n_classes)]
    tied = []
    for j, t in enumerate((ts[3], ts[2], ts[1], ts[0], ts[3], ts[0])):
        tied.append(fx.pod({"cpu": "500"}, creationTimestamp=t, uid=f"tie-{5 - j}"))
    tied += [fx.pod({"cpu": "500"}, creationTimestamp=ts[1], uid=u) for u in ("uid-b", "uid-a")]
    its = [_it("wide", {"cpu": "100000", "memory": "1Ti", "pods": "100000"}, 10.0)]
    return fx.problem(tied + pods_, instance_types=its, provisioners=[{"name": "default"}])


def queue_order(problem):
    """queue.go:82-108 restated on the problem: cpu desc, memory desc, timestamp asc, UID asc -> pod indices"""
    import exact_arith as ea
    pods_ = problem["pods"]

    def key(i):
        r = ea.pod_requests(pods_[i])
        return (-r.get("cpu", 0), -r.get("memory", 0), pods_[i].get("creationTimestamp", 0), pods_[i]["uid"])
    return sorted(range(len(pods_)), key=key)


def queue_corpus():
    in_queue_order = lambda prob: (lambda r: len(r["newNodes"]) == 1 and r["newNodes"][0]["pods"] == queue_order(prob))
    out = []
    for name, prob in (("queue-ties-small", queue_ties(8)), ("queue-extreme-span", queue_ties(8, extreme=True)),
                       ("queue-key-over-64-bits", queue_ties(4200))):
        out.append((name, prob, in_queue_order(prob)))
    return out


# ---------------------------------------------------------------- ranking
def _rank_problem(pods_per_node, ttl=None, now=0.0, created=None):
    its = ca.assorted()
    nodes = [ra._node(f"n{i}", [fx.pod({"cpu": "1"}, nodeName=f"n{i}", **kw) for kw in pods], its=its,
                      **({"creationTimestamp": created[i]} if created else {}))
             for i, pods in enumerate(pods_per_node)]
    return ra._problem(nodes, its, provisioner={"ttlSecondsUntilExpired": ttl} if ttl is not None else {}, now=now)


NAN, INF = float("nan"), float("inf")


def ranking_corpus():
    """(name, problem): every node is a consolidation candidate"""
    to10 = 9 * 2 ** 27          # 1 + 9 = 10 exactly
    return [
        ("rank-nan-between", _rank_problem([[{}], [{"deletionCost": NAN}], [{"priority": -2 ** 25}]])),  # costs 1, NaN, 0
        ("rank-nans-first-and-last", _rank_problem([[{"deletionCost": NAN}], [{}], [{"deletionCost": NAN}, {}], [{"priority": -2 ** 25}],
                                                    [{"deletionCost": NAN}]])),
        ("rank-extremes", _rank_problem([[{"priority": -2147483648}], [{"priority": 1000000000}], [{"deletionCost": 2147483647}],
                                         [{"deletionCost": -2147483647}], [{"deletionCost": INF}], [{"deletionCost": -INF}],
                                         [{"deletionCost": to10}], [{"deletionCost": -11 * 2 ** 27}], [{"deletionCost": to10, "priority": 1}],
                                         [{"deletionCost": 2147483647, "priority": 1000000000}, {"deletionCost": -INF}]])),
        ("rank-ttl0-age0", _rank_problem([[{}], [{}, {}], [{"priority": -2 ** 25}]], ttl=0, now=100.0, created=[100.0, 100.0, 100.0])),
        ("rank-ttl0-age-positive", _rank_problem([[{}], [{}, {}], [{}]], ttl=0, now=100.0, created=[100.0, 50.0, 100.0])),
        ("rank-negative-age", _rank_problem([[{}], [{}, {}], [{}]], ttl=30, now=100.0, created=[130.0, 90.0, 100.0])),
        ("rank-256-equal", _rank_problem([[{}]] * 256)),
        ("rank-257-equal", _rank_problem([[{}]] * 257)),
        ("rank-257-nan-across-tiles", _rank_problem([[{"deletionCost": NAN}] if i % 7 == 3 else [{}] for i in range(257)])),
    ]


def corpus():
    """every scheduling entry: (name, problem, answer)"""
    return limits_corpus() + quantity_corpus() + queue_corpus()
