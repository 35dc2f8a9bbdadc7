"""Scheduling problems that fill one fixed-width table of the solver to its last lane or bit (tests/test_table_widths.py).

The solver keeps one warp lane per label key (32), one 64-bit instance-type word per lane (32 words = 2 048 types), one
lane per resource (8), one bit of a 64-bit word per NodePool, per value of a key, per reservation and per host port, one
lane per distinct offering requirement set (32), and 32- / 64-bit words over the existing nodes.  Each generator here
reaches one of those widths with a problem whose answer depends on the last lane or bit, and takes an `edge` flag that
removes that last element, so a test can check that the answer changes without it.  The generators have their own
random streams; tests/fuzz.py is not touched.
"""
from __future__ import annotations

import random

import numpy as np

from karpenter_b200 import kwok
from karpenter_b200.model import (CAPACITY_TYPE_LABEL, HOSTNAME_LABEL, INSTANCE_TYPE_LABEL, NODEPOOL_LABEL, OS_LABEL,
                                  RESERVATION_ID_LABEL, ZONE_LABEL, ARCH_LABEL, LabelSelector, NodePool,
                                  NodeSelectorRequirement, Offering, Pod, PodAffinityTerm, StateNode, Taint, Toleration,
                                  TopologySpreadConstraint, quantity_units)
from karpenter_b200.scheduler import Scheduler

AWS = 1724  # types in the AWS catalog (kwok.aws_instance_types)
RACK = "example.com/rack"
EDGE_KEYS = ["zz.example.com/e0", "zz.example.com/e1", "zz.example.com/e2"]  # sort last: keys 29, 30, 31 at K = 32
FPGA = "example.com/fpga"
BOTH = ("on-demand", "spot")


def req(key, op, *values, min_values=None):
    return NodeSelectorRequirement(key, op, tuple(values), min_values)


class _Uid:
    def __init__(self, seed):
        self.rng = random.Random(seed)
        self.n = 0

    def pods(self, n, **kw):
        out = []
        for _ in range(n):
            self.n += 1
            out.append(Pod(name=f"p{self.n}", uid=self.rng.getrandbits(100), **kw))
        return out


def encode(sched: Scheduler, pods):
    """Scheduler.encode that also returns the ProblemBuilder (its interned host-port bits)"""
    b = sched._builder()
    idx = {n.name: b.add_node(n) for n in sched.state_nodes}
    for n in sched.state_nodes:
        for p in n.running_pods:
            b.add_running(p, idx[n.name])
    for p in pods:
        b.add_pod(p)
    return b.build(), b


def node(name, it, pool="default", labels=None, frac=0.5, running=(), taints=(), host_ports=(), zone=None):
    """an existing node of instance type `it` with `frac` of its allocatable left"""
    arch = [x for x in it.requirements if x.key == ARCH_LABEL][0].values[0]
    zone = zone or [x for x in it.offerings[0].requirements if x.key == ZONE_LABEL][0].values[0]
    lab = {HOSTNAME_LABEL: name, ZONE_LABEL: zone, CAPACITY_TYPE_LABEL: "on-demand", OS_LABEL: "linux", ARCH_LABEL: arch,
           NODEPOOL_LABEL: pool, INSTANCE_TYPE_LABEL: it.name}
    lab.update(labels or {})
    avail = {}
    for r in ("cpu", "memory", "pods"):
        a = quantity_units(r, it.capacity[r]) - quantity_units(r, it.overhead.get(r, 0))
        v = int(a * frac)
        avail[r] = f"{v}m" if r == "cpu" else v
    cap = dict(it.capacity)
    return StateNode(name=name, labels=lab, taints=list(taints), available=avail, capacity=cap, nodepool=pool,
                     instance_type=it.name, running_pods=list(running), host_ports=list(host_ports))


# ---- instance types: T in {1 985, 2 047, 2 048} ----------------------------------------------------------------------
def catalog(n_types):
    """The AWS catalog plus n_types - 1 724 synthetic types.  Synthetic type i copies the offerings (so the prices) of AWS
    type 7 i mod 1 724, so price-order ties cross words 26 - 31.  Their names (family "lastw" in word 31, index >= 1 984,
    "edge" before it) are instance-type values no AWS type carries."""
    aws = kwok.aws_instance_types()
    assert len(aws) == AWS
    out = list(aws)
    for t in range(AWS, n_types):
        src = aws[(7 * (t - AWS)) % AWS]
        fam = "lastw" if t >= 1984 else "edge"
        offs = [([r for r in o.requirements if r.key == CAPACITY_TYPE_LABEL][0].values[0],
                 [r for r in o.requirements if r.key == ZONE_LABEL][0].values[0], o.price) for o in src.offerings]
        cpu = 2 + (t % 5) * 2
        out.append(kwok.new_instance_type(f"{fam}-{t}", "amd64", ["linux"], {"cpu": str(cpu), "memory": f"{cpu * 4}Gi",
                                                                             "pods": "30", "ephemeral-storage": "20Gi"}, offs))
    return out


def types_problem(n_types=2048, max_instance_types=0, edge=True, min_values=True, n_fill=0, seed=1):
    """T instance types on two NodePools: `default`, and `mv` with Strict minValues 64 on the instance-type key (so a
    truncation to 63 types drops its claims).  Pods: generic ones (claims with hundreds of types, cut inside price ties),
    ones that fit only a few synthetic types before word 31, ones that fit only types of word 31, and ones pinned to `mv`.
    edge=False drops the types of word 31 (and the word-31 pods then stay pending).  n_fill NodePool labels add as many
    label keys (26 make K = 32)."""
    its = catalog(n_types)
    if not edge:
        its = its[:1984]
    fill = {f"example.com/f{i:02d}": "v" for i in range(n_fill)}
    pools = [NodePool(name="default", weight=10, labels=fill, requirements=[req(CAPACITY_TYPE_LABEL, "In", *BOTH)])]
    if min_values:
        pools.append(NodePool(name="mv", requirements=[req(CAPACITY_TYPE_LABEL, "In", *BOTH),
                                                       req(INSTANCE_TYPE_LABEL, "Exists", min_values=64)]))
    names = [it.name for it in its]
    lastw = [names[t] for t in (1984, 1985, 2046, 2047) if t < len(names)]
    u = _Uid(seed)
    pods = (u.pods(60, requests={"cpu": "1", "memory": "2Gi"}, labels={"app": "generic"})
            + u.pods(20, requests={"cpu": "3", "memory": "1Gi"}, labels={"app": "edge"},
                     node_affinity_required=[[req(INSTANCE_TYPE_LABEL, "In", *[names[t] for t in (1724, 1800, 1983)])]])
            + u.pods(12, requests={"cpu": "1500m", "memory": "1Gi"}, labels={"app": "lastw"},
                     node_affinity_required=[[req(INSTANCE_TYPE_LABEL, "In", *lastw)]] if lastw else [])
            + u.pods(8, requests={"cpu": "40", "memory": "64Gi"}, labels={"app": "big"}))
    if min_values:
        pods += u.pods(10, requests={"cpu": "2", "memory": "4Gi"}, labels={"app": "mv"}, node_selector={NODEPOOL_LABEL: "mv"})
    s = Scheduler(pools, {p.name: its for p in pools}, max_instance_types=max_instance_types)
    return s.encode(pods)


# ---- label keys: K == 32 ---------------------------------------------------------------------------------------------
def keys_problem(bounds=True, edge=True, n_fill=24, seed=2):
    """32 active label keys: hostname, capacity type, zone, nodepool, node class, 24 NodePool label keys example.com/fNN and
    the three keys zz.example.com/e0 - e2 that sort last (29, 30, 31).  Pods use In / NotIn / Exists / DoesNotExist on e0,
    Gt / Lt on the integer key e1 (bounds=True), In on e2 and spread on e2, the highest-numbered key.  edge=False drops the
    pods' requirement on e2 (the spread keeps the key).  n_fill = 25 makes 33 keys."""
    e0, e1, e2 = EDGE_KEYS
    fill = {f"example.com/f{i:02d}": "v" for i in range(n_fill)}
    a = NodePool(name="a", weight=10, labels=dict(fill, **{e0: "x"}),
                 requirements=[req(CAPACITY_TYPE_LABEL, "In", *BOTH), req(e1, "In", "2", "4", "8", "16"), req(e2, "In", "a", "b", "c")])
    b = NodePool(name="b", labels=dict(fill),
                 requirements=[req(CAPACITY_TYPE_LABEL, "In", *BOTH), req(e1, "In", "2", "4"), req(e2, "In", "a", "b", "c")])
    its = kwok.aws_instance_types(80)
    u = _Uid(seed)
    r = {"cpu": "1", "memory": "1Gi"}
    spread = [TopologySpreadConstraint(1, e2, LabelSelector.of({"app": "spread"}))]
    pods = (u.pods(15, requests=r, labels={"app": "in"}, node_affinity_required=[[req(e0, "In", "x")]])
            + u.pods(15, requests=r, labels={"app": "notin"}, node_affinity_required=[[req(e0, "NotIn", "x")]])
            + u.pods(10, requests=r, labels={"app": "exists"}, node_affinity_required=[[req(e0, "Exists")]])
            + u.pods(10, requests=r, labels={"app": "dne"}, node_affinity_required=[[req(e0, "DoesNotExist")]])
            + u.pods(20, requests={"cpu": "2", "memory": "1Gi"}, labels={"app": "c"},
                     node_affinity_required=[[req(e2, "In", "c")]] if edge else [])
            + u.pods(30, requests={"cpu": "500m", "memory": "1Gi"}, labels={"app": "spread"}, topology_spread_constraints=spread))
    if bounds:
        pods += (u.pods(10, requests=r, labels={"app": "gt"}, node_affinity_required=[[req(e1, "Gt", "3")]])
                 + u.pods(10, requests=r, labels={"app": "lt"}, node_affinity_required=[[req(e1, "Lt", "3"), req(e0, "Exists")]]))
    else:
        pods += u.pods(10, requests=r, labels={"app": "e1"}, node_affinity_required=[[req(e1, "In", "8")]])
    return Scheduler([a, b], {"a": its, "b": its}).encode(pods)


# ---- values of a key: 64 on a topology key ---------------------------------------------------------------------------
def values_problem(edge=True, n_values=64, seed=3):
    """The rack key takes exactly 64 values r00 - r63 (a spread on it keeps it out of value compaction): the NodePool
    requires rack In all 64 (edge=False: all but r63), two existing nodes carry r63, pods use In [r63] and NotIn [r63], and
    an app spreads over the racks.  n_values = 65 adds r64 (the key cannot be compacted: it is a topology key)."""
    racks = [f"r{i:02d}" for i in range(n_values)]
    pool = NodePool(name="default", requirements=[req(CAPACITY_TYPE_LABEL, "In", *BOTH),
                                                  req(RACK, "In", *(racks if edge else [r for r in racks if r != "r63"]))])
    its = kwok.aws_instance_types(60)
    small = [it for it in its if quantity_units("cpu", it.capacity["cpu"]) >= 8000][0]
    nodes = [node(f"node-{i}", small, labels={RACK: "r63"}, frac=4500 / quantity_units("cpu", small.capacity["cpu"]))
             for i in range(2)]  # four pods each
    u = _Uid(seed)
    sel = LabelSelector.of({"app": "spread"})
    pods = (u.pods(30, requests={"cpu": "1", "memory": "1Gi"}, labels={"app": "in63"}, node_affinity_required=[[req(RACK, "In", "r63")]])
            + u.pods(20, requests={"cpu": "1", "memory": "1Gi"}, labels={"app": "notin63"},
                     node_affinity_required=[[req(RACK, "NotIn", "r63")]])
            + u.pods(70, requests={"cpu": "250m", "memory": "256Mi"}, labels={"app": "spread"},
                     topology_spread_constraints=[TopologySpreadConstraint(1, RACK, sel)],
                     pod_anti_affinity=[PodAffinityTerm(sel, HOSTNAME_LABEL)]))
    return Scheduler([pool], {"default": its}, nodes).encode(pods)


# ---- resources: R == 8 -----------------------------------------------------------------------------------------------
RESOURCES = ["cpu", "memory", "pods", "ephemeral-storage", "nvidia.com/gpu", "hugepages-2Mi", "hugepages-1Gi", FPGA]


def resources_problem(edge=True, extra=False, seed=4):
    """Eight resources: the four defaults, nvidia.com/gpu, two hugepages sizes (subtracted from allocatable memory) and
    example.com/fpga on lane 7.  Some pods request the fpga (edge=False: they do not), some a GPU, some nearly all the
    memory of a type whose hugepages leave too little of it.  extra=True adds a ninth resource, example.com/asic."""
    its = kwok.aws_instance_types(80)
    for i in range(16):
        res = {"cpu": "16", "memory": "64Gi", "pods": "30", "ephemeral-storage": "20Gi", "nvidia.com/gpu": str(i % 3),
               "hugepages-2Mi": f"{(i % 4) * 2}Gi", "hugepages-1Gi": f"{(i % 2) * 8}Gi", FPGA: str(i % 4)}
        if extra:
            res["example.com/asic"] = "1"
        its.append(kwok.new_instance_type(f"accel-{i}", "amd64", ["linux"], res,
                                          [("on-demand", z, 1.5 + 0.05 * (i % 5)) for z in kwok.AWS_ZONES]))
    pool = NodePool(name="default", requirements=[req(CAPACITY_TYPE_LABEL, "In", *BOTH)])
    u = _Uid(seed)
    pods = (u.pods(30, requests={"cpu": "1", "memory": "2Gi"}, labels={"app": "plain"})
            + u.pods(12, requests={"cpu": "2", "memory": "4Gi", FPGA: "1" if edge else "0"}, labels={"app": "fpga"})
            + u.pods(8, requests={"cpu": "2", "memory": "4Gi", "nvidia.com/gpu": "1"}, labels={"app": "gpu"})
            + u.pods(6, requests={"cpu": "2", "memory": "50Gi", "hugepages-2Mi": "1Gi"}, labels={"app": "huge"}))
    return Scheduler([pool], {"default": its}).encode(pods)


# ---- NodePools: N == 64 ----------------------------------------------------------------------------------------------
def pools_problem(n_pools=64, limits=True, edge=True, seed=5, n_its=60):
    """n_pools NodePools, tainted pool=<name>, in groups of eight of equal weight (weights fall with the template index, and
    names fall within a group, so template i is NodePool np-(63 - i)).  Classes tolerate only template 31, 32 or 63 (the
    low / high word of the template mask and bit 63) or every pool; template 63 has a cpu limit (limits=True).  edge=False
    drops template 63."""
    n = n_pools if edge else n_pools - 1
    names = [f"np-{99 - i:02d}" for i in range(n)]
    pools = []
    for i, name in enumerate(names):
        lim = {"cpu": "6"} if limits and i == 63 else {}
        pools.append(NodePool(name=name, weight=(n_pools - i) // 8 * 10, requirements=[req(CAPACITY_TYPE_LABEL, "In", *BOTH)],
                              taints=[Taint("pool", name, "NoSchedule")], limits=lim))
    its = kwok.aws_instance_types(n_its)
    u = _Uid(seed)

    def only(i):
        return [Toleration("pool", "Equal", f"np-{99 - i:02d}", "NoSchedule")]
    pods = (u.pods(10, requests={"cpu": "1", "memory": "1Gi"}, labels={"app": "any"}, tolerations=[Toleration("pool", "Exists")])
            + u.pods(8, requests={"cpu": "1", "memory": "1Gi"}, labels={"app": "t31"}, tolerations=only(31))
            + u.pods(8, requests={"cpu": "1", "memory": "1Gi"}, labels={"app": "t32"}, tolerations=only(32))
            + u.pods(12, requests={"cpu": "1", "memory": "1Gi"}, labels={"app": "t63"}, tolerations=only(63))
            + u.pods(6, requests={"cpu": "1", "memory": "1Gi"}, labels={"app": "t31_63"}, tolerations=only(31) + only(63)))
    return Scheduler(pools, {p.name: its for p in pools}).encode(pods), names


# ---- offering requirement sets: 32 -----------------------------------------------------------------------------------
OFF_ZONES = [f"wz-{i:02d}" for i in range(17)]


def offerings_problem(n_sets=32, edge=True, seed=6):
    """Instance types offered in zones wz-00 ... times spot / on-demand: n_sets distinct offering requirement sets, set 31
    being (wz-15, on-demand).  Some pods require wz-15 and on-demand, which leaves only set 31; edge=False removes that
    offering from every type."""
    sets = [(ct, z) for z in OFF_ZONES for ct in ("spot", "on-demand")][:n_sets]
    if not edge:
        sets = [s for s in sets if s != ("on-demand", "wz-15")]
    its = []
    for i, it in enumerate(kwok.aws_instance_types(50)):
        res = {k: it.capacity[k] for k in ("cpu", "memory", "pods", "ephemeral-storage")}
        base = it.offerings[1].price
        its.append(kwok.new_instance_type(it.name, "amd64", ["linux"], res,
                                          [(ct, z, base * (0.7 if ct == "spot" else 1.0) * (1 + 0.001 * j)) for j, (ct, z) in enumerate(sets)]))
    pool = NodePool(name="default", requirements=[req(CAPACITY_TYPE_LABEL, "In", *BOTH)])
    u = _Uid(seed)
    pods = (u.pods(20, requests={"cpu": "1", "memory": "1Gi"}, labels={"app": "plain"})
            + u.pods(15, requests={"cpu": "1", "memory": "1Gi"}, labels={"app": "set31"},
                     node_selector={ZONE_LABEL: "wz-15", CAPACITY_TYPE_LABEL: "on-demand"})
            + u.pods(10, requests={"cpu": "2", "memory": "1Gi"}, labels={"app": "wz15"}, node_selector={ZONE_LABEL: "wz-15"}))
    return Scheduler([pool], {"default": its}).encode(pods)


def offering_sets(problem):
    """distinct offering requirement sets of an encoded problem: (requirement set, reservation id) pairs"""
    rsv = problem.get("off_reserved")
    rid = problem.get("off_reservation_id") if problem.n_reservations else None
    return len({(int(rs), int(rid[o]) if rid is not None and rsv[o] else -1) for o, rs in enumerate(problem.get("off_reqset"))})


# ---- reservations: 64 ids, id 63 in use ------------------------------------------------------------------------------
def reservations_problem(strict=True, edge=True, n_reservations=64, seed=7):
    """Reserved offerings of two reservations, r-00 and r-63, on a few types; the encoded problem then declares
    n_reservations ids with r-63 as the last one (ids in between are declared and unused: every reserved offering set is a
    distinct offering requirement set, and those are 32 at most).  edge=False leaves reservation 63 without offerings."""
    its = kwok.aws_instance_types(40)
    zones = kwok.AWS_ZONES
    for i, it in enumerate(its[:12]):
        for r in it.requirements:
            if r.key == CAPACITY_TYPE_LABEL:
                object.__setattr__(r, "values", tuple(r.values) + ("reserved",))
        rids = ["r-00"] if (i % 2 == 0 or not edge) else ["r-63"]
        if i == 0 and edge:
            rids.append("r-63")
        for rid in rids:
            it.offerings = list(it.offerings) + [Offering([req(CAPACITY_TYPE_LABEL, "In", "reserved"), req(ZONE_LABEL, "In", zones[i % 4]),
                                                           req(RESERVATION_ID_LABEL, "In", rid)], 0.0001, True, reservation_capacity=2 + i % 3)]
    pool = NodePool(name="default", requirements=[req(CAPACITY_TYPE_LABEL, "In", "reserved", *BOTH)])
    u = _Uid(seed)
    pods = (u.pods(30, requests={"cpu": "1", "memory": "1Gi"}, labels={"app": "plain"})
            + u.pods(10, requests={"cpu": "500m", "memory": "512Mi"}, labels={"app": "rsv"},
                     node_selector={CAPACITY_TYPE_LABEL: "reserved"}))

    class S(Scheduler):
        def _builder(self):
            b = super()._builder()
            b.reserved_offering_strict = strict
            return b
    enc = S([pool], {"default": its}).encode(pods)
    p = enc.problem
    names = enc.reservation_names
    rid = p.get("off_reservation_id").copy()
    last = n_reservations - 1
    remap = {names.index(n): (0 if n == "r-00" else last) for n in names}
    rsv = p.get("off_reserved")
    for o in range(len(rid)):
        if rsv[o]:
            rid[o] = remap[int(rid[o])]
    vals = np.full(n_reservations, enc.value_id(RESERVATION_ID_LABEL, "r-00"), np.int32)
    if "r-63" in names:
        vals[last] = enc.value_id(RESERVATION_ID_LABEL, "r-63")
    p.set("off_reservation_id", rid)
    p.set("n_reservations", n_reservations)
    p.set("reservation_value", vals)
    return enc


# ---- host ports: 64 --------------------------------------------------------------------------------------------------
PORTS = [("", 10_000 + i, "TCP") for i in range(64)]


def ports_problem(edge=True, seed=8):
    """64 distinct host ports: NodePool `d` runs a daemon on port 0, node-0 holds ports 0 - 62 (bits 0 - 62), node-1 port 63
    (bit 63); pods use port 63, port 10, port 62 or port 0.  edge=False takes port 63 off node-1 (64 ports stay: a pod
    still uses it)."""
    its = kwok.aws_instance_types(60)
    big = [it for it in its if quantity_units("cpu", it.capacity["cpu"]) >= 16000][0]
    nodes = [node("node-0", big, frac=0.9, host_ports=PORTS[:63]),
             node("node-1", big, frac=0.9, host_ports=PORTS[63:] if edge else [])]
    pools = [NodePool(name="d", weight=10, requirements=[req(CAPACITY_TYPE_LABEL, "In", *BOTH)]),
             NodePool(name="default", requirements=[req(CAPACITY_TYPE_LABEL, "In", *BOTH)])]
    u = _Uid(seed)
    pods = (u.pods(6, requests={"cpu": "1", "memory": "1Gi"}, labels={"app": "p63"}, host_ports=[PORTS[63]])
            + u.pods(5, requests={"cpu": "1", "memory": "1Gi"}, labels={"app": "p10"}, host_ports=[PORTS[10]])
            + u.pods(5, requests={"cpu": "1", "memory": "1Gi"}, labels={"app": "p62"}, host_ports=[PORTS[62]])
            + u.pods(5, requests={"cpu": "1", "memory": "1Gi"}, labels={"app": "p0"}, host_ports=[PORTS[0]])
            + u.pods(10, requests={"cpu": "1", "memory": "1Gi"}, labels={"app": "plain"}))
    s = Scheduler(pools, {p.name: its for p in pools}, nodes, daemon_host_ports={"d": [PORTS[0]]})
    return encode(s, pods)


# ---- existing nodes: E across 32 and 64 ------------------------------------------------------------------------------
def named_nodes(E):
    """indices of the existing nodes the hostname rules name: 0, 31, 32, 63, 64 and E - 1, those below E"""
    return sorted({i for i in (0, 31, 32, 63, 64, E - 1) if i < E})


def nodes_problem(E, edge=True, seed=9):
    """E existing nodes node-000 ... (all initialized: node i is index i).  Pods use hostname In / NotIn on the nodes of
    named_nodes(E), an app is anti-affine on the hostname to pods running on nodes >= 64 (and on node E - 1), and another
    spreads over the hostname.  edge=False drops node E - 1 from the In rule."""
    its = kwok.aws_instance_types(40)
    mid = [it for it in its if quantity_units("cpu", it.capacity["cpu"]) >= 4000][:4]
    anti = LabelSelector.of({"app": "anti"})
    u = _Uid(seed)
    running = {i: u.pods(1, labels={"app": "anti"}, requests={"cpu": "100m"}) for i in range(E) if i >= 64 or i == E - 1}
    # about 1.2 cpu left on every node: one pod of the In rule each
    nodes = [node(f"node-{i:03d}", mid[i % len(mid)], frac=1200 / quantity_units("cpu", mid[i % len(mid)].capacity["cpu"]),
                  running=running.get(i, ())) for i in range(E)]
    named = named_nodes(E)
    host_in = [f"node-{i:03d}" for i in named if edge or i != E - 1]
    pool = NodePool(name="default", requirements=[req(CAPACITY_TYPE_LABEL, "In", *BOTH)])
    r = {"cpu": "500m", "memory": "512Mi"}
    pods = (u.pods(len(named) + 2, requests={"cpu": "1", "memory": "512Mi"}, labels={"app": "in"}, node_affinity_required=[[req(HOSTNAME_LABEL, "In", *host_in)]])
            + u.pods(20, requests=r, labels={"app": "notin"},
                     node_affinity_required=[[req(HOSTNAME_LABEL, "NotIn", *[f"node-{i:03d}" for i in named])]])
            + u.pods(min(E, 40), requests={"cpu": "100m", "memory": "128Mi"}, labels={"app": "anti"},
                     pod_anti_affinity=[PodAffinityTerm(anti, HOSTNAME_LABEL)])
            + u.pods(30, requests={"cpu": "100m", "memory": "128Mi"}, labels={"app": "spread"},
                     topology_spread_constraints=[TopologySpreadConstraint(1, HOSTNAME_LABEL, LabelSelector.of({"app": "spread"}))]))
    return Scheduler([pool], {"default": its}, nodes).encode(pods)


# ---- consolidation at width ------------------------------------------------------------------------------------------
def consolidation_case(E, n_types=2048, n_pools=64, seed=10):
    """E existing nodes, n_pools NodePools of equal and differing weights over n_types types.  Nodes 31, 32, 63, 64 and
    E - 1 (the "edge" nodes) run the most expensive type of the catalog with two 1 500m pods and one free cpu; every other
    node is a small type nearly full with one or two 300m pods.  An edge pod fits no other node, so removing an edge node
    means a new, much cheaper NodeClaim whose options are most of the catalog (more than 600 types, ties included).  The
    pods of node 5 are pinned by hostname to node 31, those of node 6 to node E - 1, and one pod of node 63 to node 63
    itself.  Candidate sets contain nodes 31, 32, 63, 64 and E - 1.
    -> (pools, instance types per pool, nodes, candidate sets)"""
    its = catalog(n_types)
    small = [it for it in its[:200] if 2000 <= quantity_units("cpu", it.capacity["cpu"]) <= 8000][:6]
    price = lambda it: max(o.price for o in it.offerings)
    dear = max((it for it in its[:AWS] if quantity_units("cpu", it.capacity["cpu"]) >= 8000 and OS_of(it) == "linux"), key=price)
    names = [f"np-{99 - i:02d}" for i in range(n_pools)]
    pools = [NodePool(name=n, weight=(n_pools - i) // 8 * 10, requirements=[req(CAPACITY_TYPE_LABEL, "In", *BOTH)])
             for i, n in enumerate(names)]
    u = _Uid(seed)
    last = E - 1
    edge = {31, 32, 63, 64, last}
    pinned = {5: 31, 6: last}
    nodes = []
    for i in range(E):
        pool = names[i % n_pools]
        if i in edge:
            n = node(f"node-{i:03d}", dear, pool=pool, frac=1000 / quantity_units("cpu", dear.capacity["cpu"]))  # 1 cpu left
            n.pods = u.pods(2, requests={"cpu": "1500m", "memory": "1Gi"}, labels={"app": "edge"})
            if i == 63:
                n.pods[1].node_affinity_required = [[req(HOSTNAME_LABEL, "In", "node-063")]]
        else:
            n = node(f"node-{i:03d}", small[i % len(small)], pool=pool, frac=0.1)
            rule = [[req(HOSTNAME_LABEL, "In", f"node-{pinned[i]:03d}")]] if i in pinned else []
            n.pods = u.pods(1 + i % 2, requests={"cpu": "300m", "memory": "256Mi"}, labels={"app": f"a{i % 3}"},
                            node_affinity_required=rule)
        nodes.append(n)
    sets = [[i] for i in (5, 6, 31, 32, 63, 64, last)] + [[31, 32], [63, 64], [5, 31], [0, last], [1, 2, last]]
    sets = [[f"node-{i:03d}" for i in s] for s in sets if all(i < E for i in s)]
    return pools, {p.name: its for p in pools}, nodes, sets


def OS_of(it):
    return [x for x in it.requirements if x.key == OS_LABEL][0].values[0]
