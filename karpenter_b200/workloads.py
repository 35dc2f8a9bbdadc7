"""Synthetic KWOK workloads C1..C5 of BASELINE.json / SURVEY.md section 8(d).

Deterministic: every random draw comes from splitmix64 seeded with 42 (mirroring the reference benchmark's
`rand.New(rand.NewSource(42))`, scheduling_benchmark_test.go:62) and the pod request mix is the reference's
randomCPU / randomMemory (scheduling_benchmark_test.go:446-454).
"""
from __future__ import annotations

from typing import Dict, List, Tuple

import numpy as np

from . import kwok
from .encode import EncodedProblem, ProblemBuilder
from .model import (ARCH_LABEL, CAPACITY_TYPE_LABEL, HOSTNAME_LABEL, NODEPOOL_LABEL, OS_LABEL, ZONE_LABEL, LabelSelector,
                    NodePool, NodeSelectorRequirement, Pod, PodAffinityTerm, StateNode, Taint, Toleration,
                    TopologySpreadConstraint)

SEED = 42
CPU_MILLI = [100, 250, 500, 1000, 1500]
MEM_MI = [100, 256, 512, 1024, 2048, 4096]
_G = np.uint64(0x9E3779B97F4A7C15)


def splitmix64(seed: int, idx: np.ndarray) -> np.ndarray:
    """splitmix64 output number `idx` (0-based) of the stream started at `seed`."""
    with np.errstate(over="ignore"):
        z = np.uint64(seed) + (idx.astype(np.uint64) + np.uint64(1)) * _G
        z = (z ^ (z >> np.uint64(30))) * np.uint64(0xBF58476D1CE4E5B9)
        z = (z ^ (z >> np.uint64(27))) * np.uint64(0x94D049BB133111EB)
        return z ^ (z >> np.uint64(31))


def draws(n: int, width: int, seed: int = SEED) -> np.ndarray:
    """[n, width] table of uint64 draws; row i uses stream positions i*width .. i*width+width-1."""
    idx = np.arange(n * width, dtype=np.uint64)
    return splitmix64(seed, idx).reshape(n, width)


def default_nodepool(name="default", taints=(), zones=None, limits=None, weight=0) -> NodePool:
    """test/pkg/environment/common/default_nodepool.yaml (os In [linux], capacity-type In [on-demand])."""
    reqs = [NodeSelectorRequirement(OS_LABEL, "In", ("linux",)),
            NodeSelectorRequirement(CAPACITY_TYPE_LABEL, "In", ("on-demand",))]
    if zones:
        reqs.append(NodeSelectorRequirement(ZONE_LABEL, "In", tuple(zones)))
    return NodePool(name=name, weight=weight, requirements=reqs, taints=list(taints), limits=dict(limits or {}))


def _requests(ci: int, mi: int) -> Dict[str, str]:
    return {"cpu": f"{CPU_MILLI[ci]}m", "memory": f"{MEM_MI[mi]}Mi"}


def config_c1(n_pods=1000, n_its=50) -> EncodedProblem:
    """C1: cpu/mem-only pods, first 50 generic KWOK types, one NodePool."""
    b = ProblemBuilder()
    its = kwok.generic_instance_types()[:n_its]
    for it in its:
        b.add_instance_type(it)
    b.add_nodepool(default_nodepool(), list(range(len(its))))
    d = draws(n_pods, 4)
    ci, mi = (d[:, 0] % np.uint64(5)).astype(int), (d[:, 1] % np.uint64(6)).astype(int)
    table = np.zeros((5, 6), np.int32)
    for c in range(5):
        for m in range(6):
            table[c, m] = b.pod_class(Pod(requests=_requests(c, m)))
    b.set_pod_arrays(table[ci, mi], np.zeros(n_pods, np.int64), d[:, 2], d[:, 3])
    return b.build()


def config_c2(n_pods=100_000, n_its=500, nodepool="default") -> EncodedProblem:
    """C2: zone / arch node selectors + tolerations against a tainted NodePool, first 500 AWS-KWOK types."""
    b = ProblemBuilder()
    its = kwok.aws_instance_types(n_its)
    for it in its:
        b.add_instance_type(it)
    taint = Taint("bench/dedicated", "true", "NoSchedule")
    b.add_nodepool(default_nodepool(nodepool, taints=[taint]), list(range(len(its))))
    cls, uid_hi, _ = _c2_pods(b, n_pods, None)
    uid_lo = splitmix64(SEED + 2, np.arange(n_pods, dtype=np.uint64))
    b.set_pod_arrays(cls, np.zeros(n_pods, np.int64), uid_hi, uid_lo)
    return b.build()


def _c2_pods(b: ProblemBuilder, n_pods: int, nodepool_pin, seed=SEED, pools=None):
    zones = kwok.AWS_ZONES
    archs = ["x86_64", "arm64"]
    d = draws(n_pods, 8, seed)
    ci, mi = (d[:, 0] % np.uint64(5)).astype(int), (d[:, 1] % np.uint64(6)).astype(int)
    zsel = np.where(d[:, 2] % np.uint64(2) == 0, (d[:, 3] % np.uint64(4)).astype(int), -1)  # 50 % pick a zone
    asel = np.where(d[:, 4] % np.uint64(4) == 0, (d[:, 5] % np.uint64(2)).astype(int), -1)  # 25 % pick an arch
    t = (d[:, 6] % np.uint64(40)).astype(int)
    tol = np.where(t < 2, 0, np.where(t % 2 == 0, 1, 2))  # 5 % none, else half Equal / half Exists
    npools = 1 if pools is None else len(pools)
    pool = np.arange(n_pods) % npools
    table = np.zeros((5, 6, 5, 3, 3, npools), np.int32)
    for c in range(5):
        for m in range(6):
            for z in range(-1, 4):
                for a in range(-1, 2):
                    for k in range(3):
                        for pl in range(npools):
                            sel = {}
                            if z >= 0:
                                sel[ZONE_LABEL] = zones[z]
                            if a >= 0:
                                sel[ARCH_LABEL] = archs[a]
                            tols = []
                            key = "bench/dedicated" if pools is None else f"bench/{pools[pl]}"
                            if pools is not None:
                                sel[NODEPOOL_LABEL] = pools[pl]
                            if k == 1:
                                tols = [Toleration(key, "Equal", "true", "NoSchedule")]
                            elif k == 2:
                                tols = [Toleration(key, "Exists", "", "")]
                            table[c, m, z + 1, a + 1, k, pl] = b.pod_class(
                                Pod(requests=_requests(c, m), node_selector=sel, tolerations=tols))
    return table[ci, mi, zsel + 1, asel + 1, tol, pool], d[:, 7], pool


def config_c3(n_apps=1000, replicas=1000, n_its=1000, zones=3) -> EncodedProblem:
    """C3: apps x replicas, zonal topology spread (maxSkew 1) + hostname anti-affinity per app."""
    b = ProblemBuilder()
    its = kwok.aws_instance_types(n_its)
    for it in its:
        b.add_instance_type(it)
    b.add_nodepool(default_nodepool(zones=kwok.AWS_ZONES[:zones]), list(range(len(its))))
    n_pods = n_apps * replicas
    d = draws(n_pods, 4)
    ci, mi = (d[:, 0] % np.uint64(5)).astype(int), (d[:, 1] % np.uint64(6)).astype(int)
    app = np.arange(n_pods) // replicas
    table = _app_classes(b, n_apps)
    b.set_pod_arrays(table[app, ci, mi], np.zeros(n_pods, np.int64), d[:, 2], d[:, 3])
    return b.build()


def config_deployments(n_deployments=1000, replicas=1000, n_its=1000, zones=3, topology=True, seed=SEED) -> EncodedProblem:
    """Deployment-shaped variant of C3 / C2 (not a BASELINE configuration): `n_deployments` Deployments of `replicas`
    IDENTICAL pods each, every Deployment with its own CPU request, so byCPUAndMemoryDescending keeps a Deployment's pods
    together in the queue -- what a scale-up of real Deployments looks like, and what the solver's cohort commits are for.
    topology=True: zonal spread (maxSkew 1) + hostname anti-affinity per Deployment (C3's constraints); False: C2's
    zone / arch selectors and tolerations against a tainted NodePool."""
    b = ProblemBuilder()
    its = kwok.aws_instance_types(n_its)
    for it in its:
        b.add_instance_type(it)
    zones_l = kwok.AWS_ZONES
    if topology:
        b.add_nodepool(default_nodepool(zones=zones_l[:zones]), list(range(len(its))))
    else:
        b.add_nodepool(default_nodepool("default", taints=[Taint("bench/dedicated", "true", "NoSchedule")]), list(range(len(its))))
    d = draws(n_deployments, 8, seed)
    cls = np.zeros(n_deployments, np.int32)
    for a in range(n_deployments):
        c, m = int(d[a, 0] % np.uint64(5)), int(d[a, 1] % np.uint64(6))
        req = {"cpu": f"{CPU_MILLI[c] + a % 97}m", "memory": f"{MEM_MI[m] + a // 97}Mi"}  # unique (cpu, memory) per Deployment
        if topology:
            labels = {"app": f"dep-{a:05d}"}
            sel = LabelSelector.of(labels)
            pod = Pod(labels=labels, requests=req, topology_spread_constraints=[TopologySpreadConstraint(1, ZONE_LABEL, sel)],
                      pod_anti_affinity=[PodAffinityTerm(sel, HOSTNAME_LABEL)])
        else:
            nsel = {}
            if int(d[a, 2] % np.uint64(2)) == 0:
                nsel[ZONE_LABEL] = zones_l[int(d[a, 3] % np.uint64(4))]
            if int(d[a, 4] % np.uint64(4)) == 0:
                nsel[ARCH_LABEL] = ["x86_64", "arm64"][int(d[a, 5] % np.uint64(2))]
            t = int(d[a, 6] % np.uint64(40))
            tols = [] if t < 2 else ([Toleration("bench/dedicated", "Equal", "true", "NoSchedule")] if t % 2 == 0
                                     else [Toleration("bench/dedicated", "Exists", "", "")])
            pod = Pod(requests=req, node_selector=nsel, tolerations=tols)
        cls[a] = b.pod_class(pod)
    n_pods = n_deployments * replicas
    u = draws(n_pods, 2, seed + 5)
    b.set_pod_arrays(np.repeat(cls, replicas), np.zeros(n_pods, np.int64), u[:, 0], u[:, 1])
    return b.build()


def _app_classes(b: ProblemBuilder, n_apps: int, extra_selector=None, tolerations=(), prefix="app"):
    table = np.zeros((n_apps, 5, 6), np.int32)
    for a in range(n_apps):
        labels = {"app": f"{prefix}-{a:05d}"}
        sel = LabelSelector.of(labels)
        tsc = [TopologySpreadConstraint(1, ZONE_LABEL, sel)]
        anti = [PodAffinityTerm(sel, HOSTNAME_LABEL)]
        for c in range(5):
            for m in range(6):
                table[a, c, m] = b.pod_class(Pod(labels=labels, requests=_requests(c, m),
                                                 node_selector=dict(extra_selector or {}),
                                                 tolerations=list(tolerations), topology_spread_constraints=tsc,
                                                 pod_anti_affinity=anti))
    return table


def config_c5(n_pods=10_000_000, n_pools=8, n_its=1000, app_replicas=1000, pools_subset=None) -> EncodedProblem:
    """C5: pods pinned to one of `n_pools` NodePools (selector + toleration of the pool's taint); half the pods carry
    the C2 constraint mix, half the C3 mix (apps never span pools).  `pools_subset` keeps only the pods (and pools) of
    the given pool indices -- the shard one rank owns when the job is split by NodePool."""
    keep = list(range(n_pools)) if pools_subset is None else list(pools_subset)
    return config_c5_shards(n_pods, n_pools, n_its, app_replicas, [keep])[0]


def config_c5_shards(n_pods=10_000_000, n_pools=8, n_its=1000, app_replicas=1000, pool_groups=None) -> List[EncodedProblem]:
    """Several shards of C5 at once (one EncodedProblem per entry of `pool_groups`, default: one per pool): the pod
    draws are computed once and shared, so building all 8 shards of the 10 M-pod job costs little more than one."""
    pools = [f"pool-{i}" for i in range(n_pools)]
    groups = [[i] for i in range(n_pools)] if pool_groups is None else [list(g) for g in pool_groups]
    its = kwok.aws_instance_types(n_its)
    zones = kwok.AWS_ZONES
    archs = ["x86_64", "arm64"]
    half = n_pods // 2
    # ---- C2 half: draws shared by every shard
    d2 = draws(half, 8, SEED)
    ci2, mi2 = (d2[:, 0] % np.uint64(5)).astype(np.int8), (d2[:, 1] % np.uint64(6)).astype(np.int8)
    zsel = np.where(d2[:, 2] % np.uint64(2) == 0, (d2[:, 3] % np.uint64(4)).astype(np.int8), -1).astype(np.int8)
    asel = np.where(d2[:, 4] % np.uint64(4) == 0, (d2[:, 5] % np.uint64(2)).astype(np.int8), -1).astype(np.int8)
    t = (d2[:, 6] % np.uint64(40)).astype(np.int8)
    tol = np.where(t < 2, 0, np.where(t % 2 == 0, 1, 2)).astype(np.int8)
    pool_a = (np.arange(half) % n_pools).astype(np.int16)
    uid_a_hi = d2[:, 7].copy()
    uid_a_lo = splitmix64(SEED + 2, np.arange(half, dtype=np.uint64))
    del d2
    # ---- C3 half
    n_b = n_pods - half
    per_pool = n_b // n_pools
    n_apps_pool = max(1, per_pool // app_replicas)
    d3 = draws(n_b, 4, SEED + 1)
    ci3, mi3 = (d3[:, 0] % np.uint64(5)).astype(np.int8), (d3[:, 1] % np.uint64(6)).astype(np.int8)
    pool_b = (np.arange(n_b) % n_pools).astype(np.int16)
    app_b = np.minimum((np.arange(n_b) // n_pools) // app_replicas, n_apps_pool - 1)
    out = []
    for keep in groups:
        b = ProblemBuilder()
        for it in its:
            b.add_instance_type(it)
        for i in keep:
            b.add_nodepool(default_nodepool(pools[i], taints=[Taint(f"bench/{pools[i]}", "true", "NoSchedule")],
                                            zones=kwok.AWS_ZONES[:3]), list(range(len(its))))
        # class tables of the kept pools only
        table2 = np.zeros((5, 6, 5, 3, 3, n_pools), np.int32)
        for pl in keep:
            key = f"bench/{pools[pl]}"
            for c in range(5):
                for m in range(6):
                    for z in range(-1, 4):
                        for a in range(-1, 2):
                            for k in range(3):
                                sel = {NODEPOOL_LABEL: pools[pl]}
                                if z >= 0:
                                    sel[ZONE_LABEL] = zones[z]
                                if a >= 0:
                                    sel[ARCH_LABEL] = archs[a]
                                tols = []
                                if k == 1:
                                    tols = [Toleration(key, "Equal", "true", "NoSchedule")]
                                elif k == 2:
                                    tols = [Toleration(key, "Exists", "", "")]
                                table2[c, m, z + 1, a + 1, k, pl] = b.pod_class(
                                    Pod(requests=_requests(c, m), node_selector=sel, tolerations=tols))
        ma = np.isin(pool_a, keep)
        cls_a = table2[ci2[ma], mi2[ma], zsel[ma] + 1, asel[ma] + 1, tol[ma], pool_a[ma]]
        mb = np.isin(pool_b, keep)
        cls_b = np.zeros(int(mb.sum()), np.int32)
        pb, ab, cb, mmb = pool_b[mb], app_b[mb], ci3[mb], mi3[mb]
        for pl in keep:
            tbl = _app_classes(b, n_apps_pool, {NODEPOOL_LABEL: pools[pl]},
                               [Toleration(f"bench/{pools[pl]}", "Exists", "", "")], prefix=f"p{pl}-app")
            m = pb == pl
            cls_b[m] = tbl[ab[m], cb[m], mmb[m]]
        cls = np.concatenate([cls_a, cls_b])
        b.set_pod_arrays(cls, np.zeros(len(cls), np.int64), np.concatenate([uid_a_hi[ma], d3[mb, 2]]),
                         np.concatenate([uid_a_lo[ma], d3[mb, 3]]))
        out.append(b.build())
    return out


def config_c4(n_nodes=10_000, n_pods=200_000, n_candidates=100, max_subset=3, n_its=144, catalog="generic",
              spot_fraction=0.0, spot_to_spot=False, node_cpus=(8, 16), window=4, slack_pods=20, pin_own=0, vol_alts=0):
    """C4: a cluster of existing KWOK nodes holding `n_pods` running pods + the removal subsets to evaluate.

    Returns (EncodedProblem, ConsolInput-kwargs dict).  BASELINE configs[3]: 10 000 nodes, 200 000 running pods, i.e.
    20 pods per node on average.  C1's 50 smallest generic types cannot hold that (4.7 vCPU per node on average against
    13.4 vCPU of requests), so the catalog is the whole generic KWOK table (144 types).  The cluster is what a bin-packing
    provisioner leaves behind: the pod stream (reference request mix, seed 42) is dealt first-fit into the last
    `window` nodes opened; when a pod fits none of them the next node is opened, with a size class from `node_cpus`
    chosen by a feedback rule (pods left / nodes left against the expected pods per full node of each class) and,
    inside the class, a uniformly drawn linux type (family c / s / m, amd64 / arm64) and zone.  With the defaults all
    10 000 nodes are used, 99 % of the allocatable vCPU are requested, nodes hold 7 .. 41 pods -- and EVERY pod is
    placed (asserted; nothing is dropped).  `slack_pods` extra pods are packed with the rest and have terminated since,
    so exactly `n_pods` run and the cluster has a dozen pod-sized holes: the freed pods of a candidate set fit into
    them only partly, which is what makes delete, replace and no-op all occur (one half-empty node anywhere would turn
    every <=3-node set into a delete).
    Candidates are the `n_candidates` non-empty nodes with the lowest DisruptionCost (multinodeconsolidation.go:87,
    utils/disruption/disruption.go:71-77: with default pod deletion costs and no expiry the cost of a node is its pod
    count; ties by node index), and every subset of size 1..max_subset of them is one computeConsolidation call
    (100 + 4950 + 161700 = 166750).  A cluster with fewer pods than nodes x pods-per-node simply leaves the tail nodes
    partly filled (the small test instances).

    `catalog="aws"` draws the nodes from the AWS-KWOK catalog instead (size classes by vCPU) and lets the NodePool launch
    any OS and capacity type, so a replacement NodeClaim can carry more than 600 instance types (the price-ordered
    truncation of scheduler.go:361-379); `spot_fraction` of the nodes run on spot capacity (spot-to-spot rules,
    consolidation.go:236-316).

    `pin_own` > 0: on that many nodes one running pod selects its own node by hostname (every tenth candidate, then
    nodes evenly spread over the rest), so removing such a node leaves that pod nowhere to go.

    `vol_alts` > 0: on that many nodes (picked the same way) the last running pod has two volume-topology alternatives,
    each a zone (a StorageClass whose allowedTopologies lists two zones, volumetopology.go:44-125).  On every other such
    node the first alternative is the node's own zone and the second the next zone; on the rest the first is a zone no
    node and no offering has, and the second the node's own zone, which is then what places the pod and what pins a
    replacement NodeClaim.
    """
    from .model import quantity_units
    b = ProblemBuilder()
    aws = catalog == "aws"
    its = kwok.aws_instance_types(n_its) if aws else kwok.generic_instance_types()[:n_its]
    for it in its:
        b.add_instance_type(it)
    if aws:
        b.add_nodepool(NodePool(name="default", requirements=[
            NodeSelectorRequirement(CAPACITY_TYPE_LABEL, "In", ("on-demand", "spot"))]), list(range(len(its))))
    else:
        b.add_nodepool(default_nodepool(), list(range(len(its))))

    def _os(it):
        return [r.values[0] for r in it.requirements if r.key == OS_LABEL][0]

    def _arch(it):
        return [r.values[0] for r in it.requirements if r.key == ARCH_LABEL][0]
    classes = [[i for i, it in enumerate(its) if _os(it) == "linux" and int(it.capacity["cpu"]) == c] for c in node_cpus]
    classes = [c for c in classes if c]
    if not classes:
        raise ValueError(f"no linux instance type with cpu in {node_cpus} among the first {n_its} of the {catalog} catalog")
    zones = kwok.AWS_ZONES if aws else kwok.KWOK_ZONES
    dn = draws(n_nodes, 2, SEED + 10)
    node_zone = (dn[:, 1] % np.uint64(4)).astype(int)
    node_spot = (draws(n_nodes, 1, SEED + 12)[:, 0] % np.uint64(1000)).astype(int) < int(1000 * spot_fraction)
    R = ["cpu", "memory", "pods", "ephemeral-storage"]
    alloc_t = np.array([[quantity_units(name, it.capacity[name]) - quantity_units(name, it.overhead.get(name, 0))
                         for name in R] for it in its], np.int64)
    n_keep = n_pods
    n_pods = n_keep + int(slack_pods)  # packed first, then `slack_pods` of them leave again (see below)
    dp = draws(n_pods, 5, SEED + 11)
    ci, mi = (dp[:, 0] % np.uint64(5)).astype(int), (dp[:, 1] % np.uint64(6)).astype(int)
    req = np.stack([np.array(CPU_MILLI)[ci], np.array(MEM_MI)[mi] * (1 << 20), np.ones(n_pods, np.int64),
                    np.zeros(n_pods, np.int64)], axis=1).astype(np.int64)
    per = [alloc_t[c[0], 0] / req[:, 0].mean() for c in classes]  # expected pods of a full node, per size class
    node_it = np.zeros(n_nodes, np.int64)
    alloc = np.zeros((n_nodes, 4), np.int64)
    used = np.zeros((n_nodes, 4), np.int64)
    pod_node = np.full(n_pods, -1, np.int64)
    nn = 0
    for i in range(n_pods):
        r = req[i]
        n = -1
        for m in range(max(0, nn - window), nn):
            if used[m, 0] + r[0] <= alloc[m, 0] and used[m, 1] + r[1] <= alloc[m, 1] and used[m, 2] + 1 <= alloc[m, 2]:
                n = m
                break
        if n < 0:
            if nn >= n_nodes:  # every node is open: the stragglers go first-fit into whatever crack holds them
                ok = np.nonzero(np.all(used + r <= alloc, axis=1))[0]
                if ok.size:
                    used[ok[0]] += r
                    pod_node[i] = ok[0]
                continue
            want = (n_pods - i) / (n_nodes - nn)
            k = 0
            for kk in range(len(classes) - 1):
                if want > 0.5 * (per[kk] + per[kk + 1]):
                    k = kk + 1
            node_it[nn] = classes[k][int(dn[nn, 0] % np.uint64(len(classes[k])))]
            alloc[nn] = alloc_t[node_it[nn]]
            n = nn
            nn += 1
        used[n] += r
        pod_node[i] = n
    for n in range(nn, n_nodes):  # nodes the stream never reached stay empty (small test instances only)
        node_it[n] = classes[0][int(dn[n, 0] % np.uint64(len(classes[0])))]
        alloc[n] = alloc_t[node_it[n]]
    # scale-down since the nodes were provisioned: `slack_pods` pods (lowest draw first; a pod the full cluster had no
    # room for counts as gone already) have left again, which leaves exactly the requested number of running pods and
    # a handful of holes scattered over the cluster
    stay = pod_node >= 0
    if stay.sum() < n_keep:
        raise ValueError(f"C4: {n_nodes} nodes of {node_cpus} vCPU cannot hold {n_keep} pods ({stay.sum()} placed)")
    placed = np.nonzero(stay)[0]
    gone = placed[np.argsort(dp[placed, 4], kind="stable")[:len(placed) - n_keep]]
    np.subtract.at(used, pod_node[gone], req[gone])
    stay[gone] = False
    assert stay.sum() == n_keep and (used <= alloc).all() and (used >= 0).all()
    pod_node, ci, mi, dp, req, n_pods = pod_node[stay], ci[stay], mi[stay], dp[stay], req[stay], n_keep
    table = np.zeros((5, 6), np.int32)
    for c in range(5):
        for m in range(6):
            table[c, m] = b.pod_class(Pod(requests=_requests(c, m)))
    for n in range(n_nodes):
        it = its[node_it[n]]
        zone = zones[node_zone[n]]
        labels = {HOSTNAME_LABEL: f"node-{n:05d}", ZONE_LABEL: zone,
                  CAPACITY_TYPE_LABEL: "spot" if node_spot[n] else "on-demand",
                  OS_LABEL: "linux", ARCH_LABEL: _arch(it), NODEPOOL_LABEL: "default",
                  "node.kubernetes.io/instance-type": it.name}
        avail = {name: int(alloc[n, r] - used[n, r]) for r, name in enumerate(R)}
        avail["cpu"] = f"{avail['cpu']}m"
        cap = dict(it.capacity)
        cap["nodes"] = 1
        b.add_node(StateNode(name=f"node-{n:05d}", labels=labels, available=avail, capacity=cap, nodepool="default",
                             instance_type=it.name))
    # pod rows grouped by node (kp_consol_input.node_pod_off); node order == name order == index order here
    order = np.argsort(pod_node, kind="stable")
    rows_cls = table[ci, mi][order]
    rows_node = pod_node[order]
    counts = np.bincount(rows_node, minlength=n_nodes)
    node_pod_off = np.concatenate([[0], np.cumsum(counts)]).astype(np.int32)
    # candidates: non-empty nodes sorted by disruption cost (== pod count), ties by index (stable canon)
    nonempty = np.nonzero(counts > 0)[0]
    cand = nonempty[np.argsort(counts[nonempty], kind="stable")][:n_candidates]
    if pin_own > 0:
        rest = np.setdiff1d(nonempty, cand)
        pick = list(cand[::10]) + list(rest[::max(1, len(rest) // pin_own)])
        for n in pick[:pin_own]:
            i = node_pod_off[n]  # the node's first pod row
            rows_cls[i] = b.pod_class(Pod(requests=_requests(ci[order][i], mi[order][i]),
                                          node_selector={HOSTNAME_LABEL: f"node-{n:05d}"}))
    if vol_alts > 0:
        rest = np.setdiff1d(nonempty, cand)
        pick = list(cand[::10]) + list(rest[::max(1, len(rest) // vol_alts)])
        for j, n in enumerate(pick[:vol_alts]):
            i = node_pod_off[n + 1] - 1  # the node's last pod row
            own = zones[node_zone[n]]
            alts = [own, zones[(node_zone[n] + 1) % len(zones)]] if j % 2 == 0 else ["no-such-zone", own]
            rows_cls[i] = b.pod_class(Pod(requests=_requests(ci[order][i], mi[order][i]),
                                          volume_requirements=[[NodeSelectorRequirement(ZONE_LABEL, "In", (z,))]
                                                               for z in alts]))
    b.set_pod_arrays(rows_cls, np.zeros(len(rows_cls), np.int64), dp[order, 2], dp[order, 3])
    enc = b.build()
    subsets: List[Tuple[int, ...]] = []
    k = len(cand)
    for i in range(k):
        subsets.append((i,))
    if max_subset >= 2:
        for i in range(k):
            for j in range(i + 1, k):
                subsets.append((i, j))
    if max_subset >= 3:
        for i in range(k):
            for j in range(i + 1, k):
                for l in range(j + 1, k):
                    subsets.append((i, j, l))
    sub_off = np.concatenate([[0], np.cumsum([len(s) for s in subsets])]).astype(np.int32)
    sub_nodes = np.array([cand[i] for s in subsets for i in s], np.int32)
    consol = dict(node_pod_off=node_pod_off, node_it=node_it.astype(np.int32), node_is_spot=node_spot.astype(np.uint8),
                  n_subsets=len(subsets), subset_off=sub_off, subset_nodes=sub_nodes,
                  spot_to_spot_enabled=int(spot_to_spot),
                  capacity_type_key=enc.key_id(CAPACITY_TYPE_LABEL),
                  ct_reserved=enc.value_id(CAPACITY_TYPE_LABEL, "reserved"),
                  ct_spot=enc.value_id(CAPACITY_TYPE_LABEL, "spot"),
                  ct_on_demand=enc.value_id(CAPACITY_TYPE_LABEL, "on-demand"))
    return enc, consol


def config_existing(n_nodes=200, n_pods=3000, n_its=50, fill=0.6, limits=None, pin_in=0.0, pin_not_in=0.0) -> EncodedProblem:
    """Provisioning against a live cluster: `n_nodes` existing KWOK nodes (zone / arch / capacity-type labels, a third
    of them tainted, `fill` of their allocatable already used) + pending pods with zone / arch selectors and
    tolerations.  Exercises addToExistingNode (scheduler.go:520-555) before the NodeClaim stages.  `pin_in` of the pods
    select one of the first 500 nodes by hostname, `pin_not_in` keep off three nodes (NotIn on the hostname)."""
    from .model import quantity_units
    b = ProblemBuilder()
    its = kwok.generic_instance_types()[:n_its]
    for it in its:
        b.add_instance_type(it)
    b.add_nodepool(default_nodepool(limits=limits), list(range(len(its))))
    linux = [i for i, it in enumerate(its) if it.name.endswith("-linux")]
    dn = draws(n_nodes, 4, SEED + 20)
    node_it = np.array(linux)[(dn[:, 0] % np.uint64(len(linux))).astype(int)]
    R = ["cpu", "memory", "pods", "ephemeral-storage"]
    taint = Taint("bench/dedicated", "true", "NoSchedule")
    for n in range(n_nodes):
        it = its[node_it[n]]
        zone = kwok.KWOK_ZONES[int(dn[n, 1] % np.uint64(4))]
        labels = {HOSTNAME_LABEL: f"node-{n:05d}", ZONE_LABEL: zone, CAPACITY_TYPE_LABEL: "on-demand",
                  OS_LABEL: "linux", ARCH_LABEL: it.name.split("-")[2], NODEPOOL_LABEL: "default",
                  "node.kubernetes.io/instance-type": it.name}
        avail = {}
        for name in R:
            a = quantity_units(name, it.capacity[name]) - quantity_units(name, it.overhead.get(name, 0))
            frac = 1.0 - fill * (int(dn[n, 2] % np.uint64(100)) / 100.0)
            avail[name] = int(a * frac)
        avail["cpu"] = f"{avail['cpu']}m"
        cap = dict(it.capacity)
        cap["nodes"] = 1
        b.add_node(StateNode(name=f"node-{n:05d}", labels=labels, available=avail, capacity=cap, nodepool="default",
                             instance_type=it.name, taints=[taint] if int(dn[n, 3] % np.uint64(3)) == 0 else []))
    d = draws(n_pods, 8, SEED + 21)
    ci, mi = (d[:, 0] % np.uint64(5)).astype(int), (d[:, 1] % np.uint64(6)).astype(int)
    zsel = np.where(d[:, 2] % np.uint64(2) == 0, (d[:, 3] % np.uint64(4)).astype(int), -1)
    asel = np.where(d[:, 4] % np.uint64(4) == 0, (d[:, 5] % np.uint64(2)).astype(int), -1)
    tol = (d[:, 6] % np.uint64(2)).astype(int)
    archs = ["amd64", "arm64"]
    table = np.zeros((5, 6, 5, 3, 2), np.int32)
    for c in range(5):
        for m in range(6):
            for z in range(-1, 4):
                for a in range(-1, 2):
                    for k in range(2):
                        sel = {}
                        if z >= 0:
                            sel[ZONE_LABEL] = kwok.KWOK_ZONES[z]
                        if a >= 0:
                            sel[ARCH_LABEL] = archs[a]
                        tols = [Toleration("bench/dedicated", "Exists", "", "")] if k else []
                        table[c, m, z + 1, a + 1, k] = b.pod_class(
                            Pod(requests=_requests(c, m), node_selector=sel, tolerations=tols))
    cls = table[ci, mi, zsel + 1, asel + 1, tol]
    if pin_in or pin_not_in:
        h = draws(n_pods, 4, SEED + 23)
        u = (h[:, 0] % np.uint64(10_000)).astype(int)
        for i in np.flatnonzero(u < int((pin_in + pin_not_in) * 10_000)):
            sel = {}
            if zsel[i] >= 0:
                sel[ZONE_LABEL] = kwok.KWOK_ZONES[zsel[i]]
            if asel[i] >= 0:
                sel[ARCH_LABEL] = archs[asel[i]]
            aff = []
            if u[i] < int(pin_in * 10_000):
                sel[HOSTNAME_LABEL] = f"node-{int(h[i, 1] % np.uint64(min(500, n_nodes))):05d}"
            else:
                hosts = tuple(f"node-{int(h[i, k] % np.uint64(n_nodes)):05d}" for k in (1, 2, 3))
                aff = [[NodeSelectorRequirement(HOSTNAME_LABEL, "NotIn", hosts)]]
            tols = [Toleration("bench/dedicated", "Exists", "", "")] if tol[i] else []
            cls[i] = b.pod_class(Pod(requests=_requests(ci[i], mi[i]), node_selector=sel, node_affinity_required=aff,
                                     tolerations=tols))
    b.set_pod_arrays(cls, np.zeros(n_pods, np.int64), d[:, 7], splitmix64(SEED + 22, np.arange(n_pods, dtype=np.uint64)))
    return b.build()
