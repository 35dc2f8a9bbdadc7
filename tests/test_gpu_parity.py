"""-m gpu: the CUDA path (through the C ABI) against the CPU oracle on the same seeded inputs."""
import numpy as np
import pytest

from karpenter_b200 import _native, workloads
from tests import oracle_lib
from tests.parity import assert_same

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def handle():
    h = _native.Handle()
    yield h
    h.close()


@pytest.mark.parametrize("n_pods", [1, 13, 60, 200, 1000])
def test_c1_parity(handle, n_pods):
    enc = workloads.config_c1(n_pods=n_pods)
    assert_same(handle.solve(enc.problem), oracle_lib.solve(enc.problem), f"C1[{n_pods}] ")


def test_c1_stable_order(handle):
    enc = workloads.config_c1(n_pods=500)
    enc.problem.set("claim_order_mode", 1)
    assert_same(handle.solve(enc.problem), oracle_lib.solve(enc.problem), "C1 stable ")


def test_feasibility_parity(handle):
    enc = workloads.config_c2(n_pods=2000, n_its=500)
    assert np.array_equal(handle.feasibility(enc.problem), oracle_lib.feasibility(enc.problem))


@pytest.mark.parametrize("n_pods", [300, 3000])
def test_c2_parity(handle, n_pods):
    enc = workloads.config_c2(n_pods=n_pods, n_its=500)
    assert_same(handle.solve(enc.problem), oracle_lib.solve(enc.problem), f"C2[{n_pods}] ")


@pytest.mark.parametrize("apps,replicas", [(3, 5), (10, 30), (40, 50)])
def test_c3_parity(handle, apps, replicas):
    enc = workloads.config_c3(n_apps=apps, replicas=replicas, n_its=300)
    assert_same(handle.solve(enc.problem), oracle_lib.solve(enc.problem), f"C3[{apps}x{replicas}] ")


def test_c2_full_size_parity(handle):
    """BASELINE configs[1] at full size: 100k pods x 500 instance types, bit-identical to the oracle."""
    enc = workloads.config_c2()
    assert_same(handle.solve(enc.problem), oracle_lib.solve(enc.problem), "C2[100k] ")


def test_c3_medium_parity(handle):
    enc = workloads.config_c3(n_apps=200, replicas=200, n_its=1000)
    assert_same(handle.solve(enc.problem), oracle_lib.solve(enc.problem), "C3[200x200] ")


@pytest.mark.parametrize("kw", [dict(), dict(n_nodes=50, n_pods=1500), dict(n_nodes=400, n_pods=2500, fill=0.9),
                                dict(limits={"cpu": "3000"}), dict(limits={"cpu": "200"})])
def test_existing_nodes_parity(handle, kw):
    """addToExistingNode through the candidate bitmaps (k_node_cand) + exact re-check, then claims, with limits."""
    enc = workloads.config_existing(**kw)
    assert_same(handle.solve(enc.problem), oracle_lib.solve(enc.problem), f"existing{kw} ")


def _consol_same(gpu, orc, what):
    from karpenter_b200 import _abi
    for k in _abi.CONSOL_PARITY_KEYS:
        assert np.array_equal(gpu[k], orc[k]), f"{what}{k}: {np.argwhere(gpu[k] != orc[k])[:5].tolist()}"


@pytest.mark.parametrize("n_nodes,n_pods,n_cand", [(300, 1500, 12), (200, 2500, 10), (1000, 12000, 14)])
def test_c4_consolidation_parity(handle, n_nodes, n_pods, n_cand):
    """Every <=3-node removal subset: decision, replacement instance types, claim / unscheduled counts."""
    from karpenter_b200 import _abi
    enc, consol = workloads.config_c4(n_nodes=n_nodes, n_pods=n_pods, n_candidates=n_cand, max_subset=3)
    ci = _abi.ConsolInput(**consol)
    _consol_same(handle.consolidate(enc.problem, ci), oracle_lib.consolidate(enc.problem, ci), f"C4[{n_nodes}] ")


def test_c4_consolidation_uninitialized_and_price(handle):
    """Uninitialized targets count as unscheduled (helpers.go:121-140); a candidate without a known instance type
    zeroes the candidate price (consolidation.go:323-326)."""
    from karpenter_b200 import _abi
    enc, consol = workloads.config_c4(n_nodes=300, n_pods=1500, n_candidates=12, max_subset=2)
    flags = enc.problem.get("node_flags").copy()
    flags[::7] &= ~np.uint8(2)  # clear KP_NODE_INITIALIZED on every 7th node
    enc.problem.set("node_flags", flags)
    node_it = consol["node_it"].copy()
    node_it[consol["subset_nodes"][0]] = -1
    consol["node_it"] = node_it
    ci = _abi.ConsolInput(**consol)
    _consol_same(handle.consolidate(enc.problem, ci), oracle_lib.consolidate(enc.problem, ci), "C4 uninit ")


def test_c4_full_size_sampled_parity(handle):
    """BASELINE configs[3] at full size (10 000 nodes holding 200 000 running pods, all 166 750 <=3-node subsets of the
    100 cheapest candidates) on the GPU; the oracle re-simulates a seeded sample of 5 400 subsets stratified over subset
    size AND over the GPU's decisions (every delete / no-op the GPU reports, up to 1 800 each, the rest replaces), and
    every one must agree bit for bit.  Size-independent properties checked on all subsets: a delete decision has no
    new claim, a replace exactly one, nothing is left unscheduled in either."""
    from karpenter_b200 import _abi
    enc, consol = workloads.config_c4()
    assert enc.problem.n_nodes == 10000 and enc.problem.n_pods == 200000
    gpu = handle.consolidate(enc.problem, _abi.ConsolInput(**consol))
    S = consol["n_subsets"]
    assert S == 166750 and len(gpu["decision"]) == S
    dec, nnew, uns = gpu["decision"], gpu["n_new_claims"], gpu["n_unscheduled"]
    assert np.all(nnew[dec == 1] == 0) and np.all(nnew[dec == 2] == 1) and np.all(uns[dec != 0] == 0)
    assert np.all(gpu["replacement_its"][dec != 2] == 0) and np.all(gpu["replacement_its"][dec == 2].any(axis=1))
    assert len(set(dec.tolist())) == 3, "the full-size instance exercises delete, replace and no-op"
    rng = np.random.default_rng(7)
    off, nodes = consol["subset_off"], consol["subset_nodes"]
    size = off[1:] - off[:-1]
    pick = [np.nonzero(size == 1)[0]]
    for k in (0, 1, 2):
        idx = np.nonzero((dec == k) & (size > 1))[0]
        pick.append(rng.choice(idx, min(len(idx), 1800), replace=False))
    pick = np.unique(np.concatenate(pick))
    rest = np.setdiff1d(np.arange(S), pick)
    pick = np.unique(np.concatenate([pick, rng.choice(rest, max(0, 5400 - len(pick)), replace=False)]))
    assert len(pick) >= 5400 and set(dec[pick].tolist()) == {0, 1, 2}
    sizes = size[pick]
    smp = dict(consol, n_subsets=len(pick), subset_off=np.concatenate([[0], np.cumsum(sizes)]).astype(np.int32),
               subset_nodes=np.concatenate([nodes[off[i]:off[i + 1]] for i in pick]).astype(np.int32))
    orc = oracle_lib.consolidate(enc.problem, _abi.ConsolInput(**smp), threads=8)
    for k in ("decision", "n_new_claims", "n_unscheduled", "replacement_its"):
        assert np.array_equal(gpu[k][pick], orc[k]), k


def _topology_cluster(n_nodes, pods_per_node, seed=3):
    """Existing nodes whose pods carry a zonal spread + hostname anti-affinity per app: candidate sets of such a cluster
    take kp_consolidate's general path (one Scheduler instance per set)."""
    import random
    from karpenter_b200 import kwok
    from karpenter_b200.model import (ARCH_LABEL, CAPACITY_TYPE_LABEL, HOSTNAME_LABEL, INSTANCE_TYPE_LABEL, NODEPOOL_LABEL,
                                      OS_LABEL, ZONE_LABEL, LabelSelector, Pod, PodAffinityTerm, StateNode,
                                      TopologySpreadConstraint, quantity_units)
    rng = random.Random(seed)
    its = kwok.generic_instance_types()[:60]
    linux = [it for it in its if it.name.endswith("-linux") and int(it.capacity["cpu"]) >= 4]
    pool = workloads.default_nodepool()
    nodes, uid = [], 1
    for n in range(n_nodes):
        it = rng.choice(linux)
        pl = []
        full = int((int(it.capacity["cpu"]) * 1000 - 100) // 250)
        fill = max(1, int(full * rng.choice([0.15, 0.5, 0.9, 1.0, 1.0])))  # a mix of full and half-empty nodes
        for _ in range(min(fill, pods_per_node)):
            app = {"app": f"a{rng.randrange(6)}"}
            sel = LabelSelector.of(app)
            pl.append(Pod(name=f"p{uid}", uid=uid, labels=app, requests={"cpu": "250m", "memory": "128Mi"},
                          topology_spread_constraints=[TopologySpreadConstraint(2, ZONE_LABEL, sel)],
                          pod_anti_affinity=[PodAffinityTerm(sel, HOSTNAME_LABEL)] if rng.random() < 0.3 else []))
            uid += 1
        used = {"cpu": 250 * len(pl), "memory": (128 << 20) * len(pl), "pods": len(pl)}
        avail = {r: quantity_units(r, it.capacity[r]) - quantity_units(r, it.overhead.get(r, 0)) - used[r]
                 for r in ("cpu", "memory", "pods")}
        avail["cpu"] = f"{avail['cpu']}m"
        cap = dict(it.capacity)
        cap["nodes"] = 1
        labels = {HOSTNAME_LABEL: f"node-{n:03d}", ZONE_LABEL: kwok.KWOK_ZONES[n % 4], CAPACITY_TYPE_LABEL: "on-demand",
                  OS_LABEL: "linux", ARCH_LABEL: it.name.split("-")[2], NODEPOOL_LABEL: "default", INSTANCE_TYPE_LABEL: it.name}
        nodes.append(StateNode(name=f"node-{n:03d}", labels=labels, available=avail, capacity=cap, nodepool="default",
                               instance_type=it.name, pods=pl))
    return pool, its, nodes


def test_general_consolidation_is_one_batch_launch():
    """120 candidate sets whose pods carry topology constraints: every set is its own Scheduler instance (fresh
    NewTopology), all of them solved by ONE k_wsolve_batch launch per chunk instead of one launch + sync per set."""
    import random
    from karpenter_b200 import _abi
    from karpenter_b200.disruption import Consolidation
    pool, its, nodes = _topology_cluster(40, 40)
    rng = random.Random(11)
    names = [n.name for n in nodes]
    sets = [rng.sample(names, rng.randint(1, 3)) for _ in range(120)]
    orc = Consolidation([pool], {"default": its}, nodes, backend=oracle_lib.consolidate, filter_same_instance_type=True)
    want = orc.compute(sets)
    gpu = Consolidation([pool], {"default": its}, nodes, filter_same_instance_type=True)
    try:
        got = gpu.compute(sets)
        st = gpu._handle.stats()
    finally:
        gpu.close()
    for k in _abi.CONSOL_PARITY_KEYS:
        assert np.array_equal(gpu.raw[k], orc.raw[k]), k
    assert got == want and len({c.decision for c in want}) >= 2
    assert st["kernel_launches"] < 20 * len(sets)  # prep kernels per instance, ONE solver launch for the chunk


def test_consolidate_deadline_keeps_finished_subsets(handle):
    """kp_consolidate honours the deadline: KP_DEADLINE, finished subsets identical to the full run, the rest UNKNOWN."""
    from karpenter_b200 import _abi
    enc, consol = workloads.config_c4(n_nodes=3000, n_pods=60000, n_candidates=60, max_subset=3)
    ci = _abi.ConsolInput(**consol)
    full = handle.consolidate(enc.problem, ci)
    assert not full["deadline"] and 255 not in set(full["decision"].tolist())
    part = handle.consolidate(enc.problem, ci, deadline_ms=1)
    if part["deadline"]:
        done = part["decision"] != 255
        assert done.sum() < len(done)
        for k in ("decision", "n_new_claims", "n_unscheduled", "replacement_its"):
            assert np.array_equal(part[k][done], full[k][done]), k


def test_malformed_problem_is_refused_not_dereferenced(handle):
    """Input validation (kp_prep.cpp validate_problem): ids outside their tables come back as KP_ERR_INVALID."""
    for field, bad in (("pod_class", 10 ** 6), ("class_reqset", -3), ("tmpl_its", 99999), ("req_vals", 1 << 20),
                       ("it_reqset", 1 << 20)):
        enc = workloads.config_c2(n_pods=200, n_its=50)
        arr = enc.problem.get(field).copy()
        arr[len(arr) // 2] = bad
        enc.problem.set(field, arr)
        with pytest.raises(_native.SolverError) as e:
            handle.solve(enc.problem)
        assert e.value.code == 2 and "invalid problem" in str(e.value), (field, str(e.value))
    enc = workloads.config_c2(n_pods=200, n_its=50)   # and the handle still works afterwards
    assert_same(handle.solve(enc.problem), oracle_lib.solve(enc.problem), "after invalid ")


def test_solve_batch_matches_single_solves(handle):
    """kp_solve_batch: one CTA per Scheduler instance, instances of different shapes in one launch; every result is
    bit-identical to the oracle on that problem (and so to kp_solve)."""
    encs = [workloads.config_c1(n_pods=300), workloads.config_c2(n_pods=4000, n_its=500),
            workloads.config_c3(n_apps=12, replicas=40, n_its=300), workloads.config_existing(n_nodes=200, n_pods=1500),
            workloads.config_c2(n_pods=1, n_its=50)]
    outs = handle.solve_batch([e.problem for e in encs])
    assert len(outs) == len(encs)
    for i, (e, o) in enumerate(zip(encs, outs)):
        assert_same(o, oracle_lib.solve(e.problem), f"batch[{i}] ")
    # resident variant, twice (state restored between runs), and a single solve on the same handle afterwards
    handle.upload_batch([e.problem for e in encs[:3]])
    for _ in range(2):
        outs = handle.solve_batch_resident()
        for i, (e, o) in enumerate(zip(encs[:3], outs)):
            assert_same(o, oracle_lib.solve(e.problem), f"batch resident[{i}] ")
    assert_same(handle.solve(encs[1].problem), oracle_lib.solve(encs[1].problem), "single after batch ")
    assert handle.solve_batch([]) == []


def test_solve_batch_more_instances_than_sms(handle):
    """200 instances > 132 SMs: the launch runs in waves; results are per-instance exact."""
    encs = [workloads.config_c1(n_pods=20 + 3 * i) for i in range(200)]
    outs = handle.solve_batch([e.problem for e in encs])
    for i in (0, 57, 148, 199):
        assert_same(outs[i], oracle_lib.solve(encs[i].problem), f"wave batch[{i}] ")


def test_c5_pool_shards_as_one_batch(handle):
    """BASELINE configs[4] shape, scaled down: 8 NodePools, C2 + C3 constraint mix, pods pinned to their pool.  The 8
    pool shards solved as ONE batch on one GPU equal the 8 oracle solves of the shards."""
    n_pods, pools = 24000, 8
    shards = [workloads.config_c5(n_pods=n_pods, n_pools=pools, n_its=300, app_replicas=100, pools_subset=[r])
              for r in range(pools)]
    outs = handle.solve_batch([e.problem for e in shards])
    for r, (e, o) in enumerate(zip(shards, outs)):
        assert_same(o, oracle_lib.solve(e.problem), f"C5 shard {r} ")
        assert len(o["domain_counts"]) > 0 and o["domain_counts"].sum() > 0  # the table a multi-GPU run all-reduces


def test_library_counter_table_single_gpu(handle):
    """kp_comm_set_counter_layout without a communicator: after a resident (batch) solve the device-resident global
    table is the concatenation of the instances' domain counters -- what the NCCL all-reduce of a multi-GPU run sums."""
    from karpenter_b200 import sharding
    shards = [workloads.config_c5(n_pods=6000, n_pools=3, n_its=200, app_replicas=50, pools_subset=[r]) for r in range(3)]
    handle.upload_batch([e.problem for e in shards])
    slots = [handle.counter_slots(i) for i in range(3)]
    offs, total = sharding.instance_offsets(slots, 0, 1)
    handle.set_counter_layout(total, offs)
    outs = handle.solve_batch_resident()
    want = np.concatenate([o["domain_counts"] for o in outs])
    assert total == len(want) and want.sum() > 0
    assert np.array_equal(handle.global_counts(), want)
    assert handle.last_allreduce_ms() >= 0.0
    # the single-instance variant
    handle.upload(shards[1].problem)
    handle.set_counter_layout(handle.counter_slots(), [0])
    res = handle.solve_resident()
    assert np.array_equal(handle.global_counts(), res["domain_counts"])


def test_shared_to_global_migration(monkeypatch):
    """Claims outgrow the shared-memory copies of the claim order / failure bitmaps (forced early with KP_SMEM_CAP: at
    most 64 claims' small arrays and 32 claims' rows on chip): the solver migrates them to HBM mid-run and the result
    must not change."""
    monkeypatch.setenv("KP_SMEM_CAP", "64,32,,")
    h = _native.Handle()
    try:
        for enc, what in ((workloads.config_c2(n_pods=30000, n_its=500), "C2 migrate "),
                          (workloads.config_c3(n_apps=40, replicas=120, n_its=300), "C3 migrate ")):
            res = h.solve(enc.problem)
            assert res["n_claims"] > 64
            assert_same(res, oracle_lib.solve(enc.problem), what)
    finally:
        h.close()


def test_c3_100k_parity(handle):
    """C3 shape at 100 000 pods (100 apps x 1000 replicas, 1000 instance types): zonal spread + hostname anti-affinity,
    1000 NodeClaims, bit-identical to the oracle."""
    enc = workloads.config_c3(n_apps=100, replicas=1000, n_its=1000)
    res = handle.solve(enc.problem)
    assert_same(res, oracle_lib.solve(enc.problem), "C3[100x1000] ")
    # size-independent properties of the domain: one pod of an app per NodeClaim, zonal skew <= 1 per app
    tgt = res["pod_target"]
    assert np.all(tgt <= -2)
    claim = -2 - tgt
    app = np.arange(len(tgt)) // 1000
    assert len(set(zip(app.tolist(), claim.tolist()))) == len(tgt)


def test_deadline_returns_partial_results(handle):
    """KP_DEADLINE: the solve stops early, what was placed so far is exactly what the full solve places."""
    enc = workloads.config_c2(n_pods=60000, n_its=500)
    full = handle.solve(enc.problem)
    assert not full["deadline"]
    part = handle.solve(enc.problem, deadline_ms=20)
    assert part["deadline"]
    placed = part["pod_target"] != -1
    assert 0 < placed.sum() < (full["pod_target"] != -1).sum()
    assert np.array_equal(part["pod_target"][placed], full["pod_target"][placed])


def _expensive_cluster(spot: bool):
    """Three full, expensive nodes of the AWS-KWOK catalog, one tiny pod each, a NodePool that may launch any of the
    1000 catalog rows: the single replacement NodeClaim starts with > 600 instance types, so SimulateScheduling's
    TruncateInstanceTypes (scheduler.go:361-379) cuts it to the 600 cheapest -- with price ties between the linux and
    windows rows of the same type right at the cut."""
    from karpenter_b200 import kwok
    from karpenter_b200.disruption import Consolidation
    from karpenter_b200.model import (ARCH_LABEL, CAPACITY_TYPE_LABEL, HOSTNAME_LABEL, INSTANCE_TYPE_LABEL, NODEPOOL_LABEL,
                                      OS_LABEL, ZONE_LABEL, NodePool, NodeSelectorRequirement, Pod, StateNode)
    its = kwok.aws_instance_types(1000)
    big = sorted((it for it in its if [r.values[0] for r in it.requirements if r.key == OS_LABEL][0] == "linux"),
                 key=lambda it: -int(it.capacity["cpu"]))[:3]
    pool = NodePool(name="default", requirements=[NodeSelectorRequirement(CAPACITY_TYPE_LABEL, "In", ("on-demand", "spot"))])
    nodes = []
    for i, it in enumerate(big):
        arch = [r.values[0] for r in it.requirements if r.key == ARCH_LABEL][0]
        labels = {HOSTNAME_LABEL: f"node-{i}", ZONE_LABEL: kwok.AWS_ZONES[i % 4], OS_LABEL: "linux", ARCH_LABEL: arch,
                  CAPACITY_TYPE_LABEL: "spot" if spot else "on-demand", NODEPOOL_LABEL: "default",
                  INSTANCE_TYPE_LABEL: it.name}
        cap = dict(it.capacity)
        cap["nodes"] = 1
        nodes.append(StateNode(name=f"node-{i}", labels=labels, available={"cpu": "0", "memory": 0, "pods": 0},
                               capacity=cap, nodepool="default", instance_type=it.name,
                               pods=[Pod(name=f"p{i}", uid=i + 1, requests={"cpu": "100m", "memory": "64Mi"})]))
    sets = [["node-0"], ["node-1"], ["node-0", "node-1"], ["node-0", "node-1", "node-2"]]
    return pool, its, nodes, sets, Consolidation


@pytest.mark.parametrize("spot,enabled", [(False, False), (True, True), (True, False)])
def test_consolidation_truncates_to_600_cheapest_types(spot, enabled):
    pool, its, nodes, sets, Consolidation = _expensive_cluster(spot)
    orc = Consolidation([pool], {"default": its}, nodes, spot_to_spot=enabled, backend=oracle_lib.consolidate)
    want = orc.compute(sets)
    gpu = Consolidation([pool], {"default": its}, nodes, spot_to_spot=enabled)
    try:
        got = gpu.compute(sets)
    finally:
        gpu.close()
    for k in ("decision", "n_new_claims", "n_unscheduled", "replacement_its"):
        assert np.array_equal(gpu.raw[k], orc.raw[k]), k
    assert got == want
    if not spot:
        assert any(len(c.replacement_instance_types) == 600 for c in want)  # the cut really happened
    elif enabled:
        assert len(want[0].replacement_instance_types) == 15                # single-node spot-to-spot: 15 cheapest


def test_more_than_64_requirement_signatures_and_request_vectors(handle):
    """The failure / acceptance masks cache 64 requirement signatures and 64 request vectors; classes beyond that run
    uncached.  144 distinct node-affinity terms x 80 distinct request vectors must still match the oracle."""
    import itertools
    import random
    from karpenter_b200 import kwok
    from karpenter_b200.model import (ARCH_LABEL, CAPACITY_TYPE_LABEL, ZONE_LABEL, NodePool, NodeSelectorRequirement, Pod)
    from karpenter_b200.scheduler import Scheduler
    rng = random.Random(5)
    its = kwok.aws_instance_types(300)
    zones = kwok.AWS_ZONES
    terms = []
    for k in range(0, 4):
        for zs in itertools.combinations(zones, k):
            for arch in (None, "x86_64", "arm64"):
                for ct in (None, "spot", "on-demand"):
                    t = []
                    if zs:
                        t.append(NodeSelectorRequirement(ZONE_LABEL, "NotIn", zs))
                    if arch:
                        t.append(NodeSelectorRequirement(ARCH_LABEL, "In", (arch,)))
                    if ct:
                        t.append(NodeSelectorRequirement(CAPACITY_TYPE_LABEL, "In", (ct,)))
                    terms.append(t)
    assert len(terms) > 64
    reqs = [{"cpu": f"{100 + 50 * i}m", "memory": f"{128 + 64 * (i % 7)}Mi"} for i in range(80)]
    pods = [Pod(name=f"p{i}", uid=rng.getrandbits(100), requests=rng.choice(reqs),
                node_affinity_required=[t] if (t := rng.choice(terms)) else []) for i in range(6000)]
    pool = NodePool(name="default", requirements=[NodeSelectorRequirement(CAPACITY_TYPE_LABEL, "In", ("spot", "on-demand"))])
    enc = Scheduler([pool], {"default": its}).encode(pods)
    assert_same(handle.solve(enc.problem), oracle_lib.solve(enc.problem), "many signatures ")


# ---- cohort commits (kp_wsolve.cuh cohort_try): Deployment-shaped queues, where a Deployment's identical pods stand together
@pytest.mark.parametrize("deps,replicas,topology,order", [(40, 300, True, 0), (40, 300, True, 1), (150, 200, True, 0),
                                                          (60, 500, False, 0), (300, 100, False, 1), (8, 2500, False, 0)])
def test_deployment_cohorts_parity(handle, deps, replicas, topology, order):
    enc = workloads.config_deployments(deps, replicas, n_its=300, topology=topology)
    enc.problem.set("claim_order_mode", order)
    gpu = handle.solve(enc.problem)
    st = handle.stats()
    assert st["cohort_pods"] > deps * replicas // 4, st      # the cohort instantiation ran and committed runs
    assert_same(gpu, oracle_lib.solve(enc.problem, threads=8), f"deployments {deps}x{replicas} ")


def test_cohorts_are_the_same_solve_at_scale(handle, monkeypatch):
    """100 Deployments x 1 000 replicas (C3's constraints, 1 000 types): cohorts on and off give the same bits; the oracle
    checks a 200-replica version of the same shape above."""
    enc = workloads.config_deployments(100, 1000, n_its=1000, topology=True)
    on = handle.solve(enc.problem)
    assert handle.stats()["cohort_pods"] > 50_000
    monkeypatch.setenv("KP_NO_COHORT", "1")
    h2 = _native.Handle()
    try:
        off = h2.solve(enc.problem)
        assert h2.stats()["cohort_pods"] == 0
    finally:
        h2.close()
    assert_same(on, off, "cohorts on/off ")
