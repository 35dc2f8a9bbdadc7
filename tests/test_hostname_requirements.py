"""Pod requirements on kubernetes.io/hostname: node selectors, required and preferred node affinity, volume requirements
and topology-spread node filters that name hosts.  Every NodeClaim carries hostname In{placeholder} with a placeholder
no pod can name (nodeclaim.go:92-96), every existing node hostname In{its hostname} (existingnode.go:62), so such a
requirement only admits or rejects candidates: In / DoesNotExist admit no NodeClaim, NotIn / Exists every one.
CPU tier: the oracle; GPU tier: the CUDA path, bit-identical to the oracle (solve, batch and consolidation)."""
import collections
import random

import numpy as np
import pytest

from karpenter_b200 import _abi, _native, fake
from karpenter_b200.disruption import Consolidation, SingleNodeConsolidation
from karpenter_b200.model import (ARCH_LABEL, CAPACITY_TYPE_LABEL, HOSTNAME_LABEL, INSTANCE_TYPE_LABEL, NODEPOOL_LABEL,
                                  OS_LABEL, ZONE_LABEL, LabelSelector, NodePool, NodeSelectorRequirement, Pod,
                                  PodAffinityTerm, PreferredSchedulingTerm, StateNode, TopologySpreadConstraint,
                                  WeightedPodAffinityTerm, quantity_units)
from karpenter_b200.scheduler import Scheduler
from tests import fuzz, oracle_lib
from tests.parity import assert_same

BACKENDS = [pytest.param("oracle", id="oracle"), pytest.param("gpu", id="gpu", marks=pytest.mark.gpu)]


def req(key, op, *values):
    return NodeSelectorRequirement(key, op, tuple(values))


def host(op, *names):
    return req(HOSTNAME_LABEL, op, *names)


def pool(name="default"):
    return NodePool(name=name, requirements=[req(CAPACITY_TYPE_LABEL, "In", "on-demand")])


def node(name, zone="test-zone-1", cpu="4", pods_=10, **kw):
    it = fake.default_instance_types()[0]
    return StateNode(name=name, labels={HOSTNAME_LABEL: name, ZONE_LABEL: zone, CAPACITY_TYPE_LABEL: "on-demand"},
                     available={"cpu": cpu, "memory": "8Gi", "pods": pods_}, capacity=dict(it.capacity), managed=False, **kw)


def pod(name, uid, cpu="100m", **kw):
    return Pod(name=name, uid=uid, requests={"cpu": cpu}, **kw)


def solve(which, pods, state_nodes=(), pools=None, **kw):
    pools = pools or [pool()]
    its = {p.name: fake.default_instance_types() for p in pools}

    def run(backend):
        s = Scheduler(pools, its, state_nodes=state_nodes, backend=backend, **kw)
        try:
            return s.solve(pods)
        finally:
            s.close()
    r = run(oracle_lib.solve)
    if which == "gpu":
        g = run(None)
        assert_same(g.raw, r.raw, "hostname requirements ")
        r = g
    return r


def placed(r, p):
    """'claim', the existing node's name, or None"""
    for name, ps in r.existing_nodes.items():
        if any(q is p for q in ps):
            return name
    return "claim" if any(q is p for c in r.new_node_claims for q in c.pods) else None


# ---- restated reference cases --------------------------------------------------------------------------------------
@pytest.mark.parametrize("which", BACKENDS)
def test_should_not_schedule_nodes_with_a_hostname_selector(which):  # scheduling/suite_test.go:224-231, :698-705
    p = pod("p", 1, node_selector={HOSTNAME_LABEL: "red-node"})
    r = solve(which, [p])
    assert not r.new_node_claims and id(p) in r.pod_errors
    p = pod("p", 1, node_affinity_required=[[host("In", "red-node")]])
    r = solve(which, [p])
    assert not r.new_node_claims and id(p) in r.pod_errors


@pytest.mark.parametrize("which", BACKENDS)
def test_should_not_ignore_hostname_affinity_with_non_local_volumes(which):  # provisioning/suite_test.go:2155-2181
    p = pod("p", 1, volume_requirements=[[host("In", "random-host-name")]])
    r = solve(which, [p])
    assert not r.new_node_claims and id(p) in r.pod_errors


# ---- scenarios ------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("which", BACKENDS)
def test_selector_naming_an_existing_node_wins_over_an_inflight_claim(which):
    # the big pod fits no node and opens a NodeClaim with room to spare; the pinned pod still goes to n2, the unpinned
    # one to n1 (first in line)
    first = pod("a", 1, cpu="2")
    pinned = pod("b", 2, node_selector={HOSTNAME_LABEL: "n2"})
    other = pod("c", 3)
    r = solve(which, [first, pinned, other], state_nodes=[node("n1", cpu="500m"), node("n2", cpu="500m")])
    assert placed(r, first) == "claim" and len(r.new_node_claims) == 1
    assert placed(r, pinned) == "n2" and placed(r, other) == "n1"


@pytest.mark.parametrize("which", BACKENDS)
def test_in_two_hosts_with_the_first_full(which):
    p = pod("p", 1, cpu="1", node_affinity_required=[[host("In", "a", "b")]])
    r = solve(which, [p], state_nodes=[node("a", cpu="500m"), node("b"), node("c")])
    assert placed(r, p) == "b"


@pytest.mark.parametrize("which", BACKENDS)
def test_not_in_skips_a_node_that_would_take_the_pod(which):
    p = pod("p", 1, node_affinity_required=[[host("NotIn", "a")]])
    r = solve(which, [p], state_nodes=[node("a"), node("b")])
    assert placed(r, p) == "b"
    r = solve(which, [p], state_nodes=[node("a")])
    assert placed(r, p) == "claim"


@pytest.mark.parametrize("which", BACKENDS)
def test_exists_and_does_not_exist(which):
    p = pod("p", 1, node_affinity_required=[[host("Exists")]])
    assert placed(solve(which, [p], state_nodes=[node("a", cpu="10m")]), p) == "claim"
    assert placed(solve(which, [p], state_nodes=[node("a")]), p) == "a"
    p = pod("p", 1, node_affinity_required=[[host("DoesNotExist")]])
    r = solve(which, [p], state_nodes=[node("a")])
    assert placed(r, p) is None and id(p) in r.pod_errors


@pytest.mark.parametrize("which", BACKENDS)
def test_in_and_not_in_folded_in_one_term(which):
    p = pod("p", 1, node_affinity_required=[[host("In", "a", "b"), host("NotIn", "a")]])
    assert placed(solve(which, [p], state_nodes=[node("a"), node("b")]), p) == "b"
    p = pod("p", 1, node_affinity_required=[[host("In", "a"), host("NotIn", "a")]])
    assert placed(solve(which, [p], state_nodes=[node("a"), node("b")]), p) is None


@pytest.mark.parametrize("which", BACKENDS)
def test_two_required_terms_relax_past_a_missing_host(which):
    p = pod("p", 1, node_affinity_required=[[host("In", "gone")], [host("In", "b")]])
    assert placed(solve(which, [p], state_nodes=[node("a"), node("b")]), p) == "b"
    p = pod("p", 1, node_affinity_required=[[host("In", "gone")], [req(ZONE_LABEL, "In", "test-zone-2")]])
    assert placed(solve(which, [p], state_nodes=[node("a")]), p) == "claim"


@pytest.mark.parametrize("which", BACKENDS)
@pytest.mark.parametrize("policy", ["Respect", "Ignore"])
def test_preferred_host_honoured_and_relaxed(which, policy):
    pref = [PreferredSchedulingTerm(10, (host("In", "b"),))]
    p = pod("p", 1, node_affinity_preferred=pref)
    r = solve(which, [p], state_nodes=[node("a"), node("b")], preference_policy=policy)
    assert placed(r, p) == ("b" if policy == "Respect" else "a")
    p = pod("p", 1, cpu="1", node_affinity_preferred=pref)  # b is full: the preference is dropped
    r = solve(which, [p], state_nodes=[node("a", cpu="100m"), node("b", cpu="100m")], preference_policy=policy)
    assert placed(r, p) == "claim"


@pytest.mark.parametrize("which", BACKENDS)
@pytest.mark.parametrize("affinity_policy", ["Honor", "Ignore"])
def test_zone_spread_whose_pods_name_hosts(which, affinity_policy):
    sel = LabelSelector.of({"app": "web"})
    tsc = [TopologySpreadConstraint(1, ZONE_LABEL, sel, node_affinity_policy=affinity_policy)]
    nodes = [node("a", "test-zone-1", running_pods=[pod("r1", 100, labels={"app": "web"})]),
             node("b", "test-zone-2", running_pods=[pod("r2", 101, labels={"app": "web"}), pod("r3", 102, labels={"app": "web"})]),
             node("c", "test-zone-3")]
    pods = [pod(f"w{i}", i + 1, labels={"app": "web"}, topology_spread_constraints=tsc,
                node_affinity_required=[[host("In", "a", "c")]]) for i in range(4)]
    pods += [pod(f"v{i}", i + 10, labels={"app": "web"}, topology_spread_constraints=tsc) for i in range(3)]
    r = solve(which, pods, state_nodes=nodes)
    # two groups (the filters differ), three zones each.  Honor: the hosted group's filter leaves node b, its two pods and
    # the zone out of the counts and the domain choice; Ignore: both groups count every node.
    want = {"Honor": [3, 0, 2, 3, 2, 2], "Ignore": [4, 3, 3, 4, 3, 3]}[affinity_policy]
    assert r.raw["n_groups"] == 2 and r.raw["domain_counts"].tolist() == want


@pytest.mark.parametrize("which", BACKENDS)
def test_hostname_anti_affinity_with_not_in(which):
    sel = LabelSelector.of({"app": "solo"})
    pods = [pod(f"s{i}", i + 1, labels={"app": "solo"}, pod_anti_affinity=[PodAffinityTerm(sel, HOSTNAME_LABEL)],
                node_affinity_required=[[host("NotIn", "a")]]) for i in range(3)]
    r = solve(which, pods, state_nodes=[node("a"), node("b")])
    assert [placed(r, p) for p in pods].count("b") == 1 and not r.existing_nodes.get("a")
    assert len(r.new_node_claims) == 2


# ---- consolidation --------------------------------------------------------------------------------------------------
def cnode(name, it, pod_list, zone="test-zone-1"):
    used = {"cpu": 0, "memory": 0, "pods": len(pod_list)}
    for p in pod_list:
        used["cpu"] += quantity_units("cpu", p.requests.get("cpu", 0))
    avail = {}
    for r in ("cpu", "memory", "pods"):
        a = quantity_units(r, it.capacity[r]) - quantity_units(r, it.overhead.get(r, 0)) - used[r]
        avail[r] = f"{a}m" if r == "cpu" else a
    arch = [x for x in it.requirements if x.key == ARCH_LABEL][0].values[0]
    labels = {HOSTNAME_LABEL: name, ZONE_LABEL: zone, CAPACITY_TYPE_LABEL: "on-demand", OS_LABEL: "linux",
              ARCH_LABEL: arch, NODEPOOL_LABEL: "default", INSTANCE_TYPE_LABEL: it.name}
    cap = dict(it.capacity)
    cap["nodes"] = 1
    return StateNode(name=name, labels=labels, available=avail, capacity=cap, nodepool="default", instance_type=it.name,
                     pods=list(pod_list))


def consolidate(which, nodes, sets):
    its = fake.default_instance_types()
    kw = dict(backend=oracle_lib.consolidate, solve_backend=oracle_lib.solve) if which == "oracle" else {}
    eng = Consolidation([pool()], {"default": its}, nodes, **kw)
    try:
        cmds = eng.compute(sets)
        if which == "gpu":
            orc = Consolidation([pool()], {"default": its}, nodes, backend=oracle_lib.consolidate)
            orc.compute(sets)
            for k in _abi.CONSOL_PARITY_KEYS:
                assert np.array_equal(eng.raw[k], orc.raw[k]), k
        return cmds
    finally:
        eng.close()


def two_nodes(selector_of):
    """two half-empty default nodes; the pod on node-0 carries selector_of(its own name, the other name)"""
    by = {it.name: it for it in fake.default_instance_types()}
    it = by["arm-instance-type"]
    p0 = pod("p0", 1, **selector_of("node-0", "node-1"))
    p1 = pod("p1", 2)
    return [cnode("node-0", it, [p0]), cnode("node-1", it, [p1])]


@pytest.mark.parametrize("which", BACKENDS)
def test_consolidation_pod_pinned_to_its_own_node_blocks_it(which):
    nodes = two_nodes(lambda own, other: dict(node_selector={HOSTNAME_LABEL: own}))
    c = consolidate(which, nodes, [["node-0"]])[0]
    assert c.decision == "noop" and c.n_unscheduled == 1


@pytest.mark.parametrize("which", BACKENDS)
def test_consolidation_pod_pinned_to_the_other_node_moves(which):
    nodes = two_nodes(lambda own, other: dict(node_selector={HOSTNAME_LABEL: other}))
    assert consolidate(which, nodes, [["node-0"]])[0].decision == "delete"


@pytest.mark.parametrize("which", BACKENDS)
def test_consolidation_pod_not_in_its_own_node_moves(which):
    nodes = two_nodes(lambda own, other: dict(node_affinity_required=[[host("NotIn", own)]]))
    assert consolidate(which, nodes, [["node-0"]])[0].decision == "delete"
    # NotIn both: the pod can only go to a new NodeClaim, a cheaper type than the node's
    nodes = two_nodes(lambda own, other: dict(node_affinity_required=[[host("NotIn", own, other)]]))
    c = consolidate(which, nodes, [["node-0"]])[0]
    assert c.decision == "replace" and c.n_new_node_claims == 1 and c.n_unscheduled == 0


@pytest.mark.parametrize("which", BACKENDS)
def test_single_node_pass_skips_the_pinned_candidate(which):
    nodes = two_nodes(lambda own, other: dict(node_selector={HOSTNAME_LABEL: own}))
    its = fake.default_instance_types()
    kw = dict(backend=oracle_lib.consolidate, solve_backend=oracle_lib.solve) if which == "oracle" else {}
    eng = Consolidation([pool()], {"default": its}, nodes, **kw)
    try:
        cmd, names, _ = SingleNodeConsolidation(eng).compute_command(nodes, {"default": 5})
    finally:
        eng.close()
    assert cmd is not None and names == ["node-1"]


# ---- refusals (GPU tier: the library) -------------------------------------------------------------------------------
def refused(pods, pools=None, state_nodes=(), its=None):
    pools = pools or [pool()]
    s = Scheduler(pools, {p.name: its or fake.default_instance_types() for p in pools}, state_nodes=state_nodes)
    h = _native.Handle()
    try:
        with pytest.raises(_native.SolverError) as e:
            h.solve(s.encode(pods).problem)
    finally:
        h.close()
    assert e.value.code == 5
    return str(e.value)


@pytest.mark.gpu
def test_refused_cases_name_what_is_missing():
    p = pod("p", 1)
    tp = NodePool(name="default", requirements=[req(CAPACITY_TYPE_LABEL, "In", "on-demand"), host("NotIn", "x")])
    assert "NodePool template" in refused([p], pools=[tp])
    its = fake.default_instance_types()
    its[0].requirements = list(its[0].requirements) + [host("In", "x")]
    assert "instance type" in refused([p], its=its)
    its = fake.default_instance_types()
    its[0].offerings = list(its[0].offerings)
    o = its[0].offerings[0]
    its[0].offerings[0] = type(o)(list(o.requirements) + [host("In", "x")], o.price, o.available)
    assert "offering" in refused([p], its=its)
    assert "Gt / Lt" in refused([pod("p", 1, node_affinity_required=[[req(HOSTNAME_LABEL, "Gt", "5")]])])
    mp = NodePool(name="default", requirements=[req(CAPACITY_TYPE_LABEL, "In", "on-demand"),
                                                NodeSelectorRequirement(HOSTNAME_LABEL, "Exists", (), 2)])
    assert "minValues on kubernetes.io/hostname" in refused([p], pools=[mp])
    aff = [PodAffinityTerm(LabelSelector.of({"app": "x"}), HOSTNAME_LABEL)]
    for kw in (dict(pod_affinity=aff), dict(pod_affinity_preferred=[WeightedPodAffinityTerm(1, aff[0])])):
        q = pod("q", 2, labels={"app": "x"}, node_selector={HOSTNAME_LABEL: "a"}, **kw)
        assert "pod affinity on kubernetes.io/hostname" in refused([q], state_nodes=[node("a")])


def test_cached_cpu_baseline_refuses_host_rules():
    """the cached CPU solver shares the table preparation but applies no host rule: it refuses, as before"""
    s = Scheduler([pool()], {"default": fake.default_instance_types()}, state_nodes=[node("a")])
    assert oracle_lib.cached_solve(s.encode([pod("p", 1, node_selector={HOSTNAME_LABEL: "a"})]).problem) is None
    assert oracle_lib.cached_solve(s.encode([pod("p", 1)]).problem) is not None


# ---- fuzz bands ------------------------------------------------------------------------------------------------------
def add_rules(seed, pools, nodes, pl, strip=False):
    """Host rules on about a third of the pod shapes (own random stream): In one or two existing hosts, In an unknown
    host, NotIn one to three hosts, Exists, DoesNotExist; as required terms, preferred terms or inside a spread pod's
    node affinity.  Pods with a rule lose their hostname-key pod affinity (the combination the library refuses)."""
    rng = random.Random(91_000 + seed)
    names = [n.name for n in nodes] or ["node-000"]
    shapes = {}
    for p in pl:
        shapes.setdefault(id(p.requests), []).append(p)
    for group in shapes.values():
        if rng.random() >= 0.35:
            continue
        kind = rng.choice(["in", "in", "unknown", "notin", "notin", "exists", "dne"])
        r = {"in": lambda: host("In", *rng.sample(names, min(len(names), rng.randint(1, 2)))),
             "unknown": lambda: host("In", "no-such-host"),
             "notin": lambda: host("NotIn", *rng.sample(names, min(len(names), rng.randint(1, 3)))),
             "exists": lambda: host("Exists"), "dne": lambda: host("DoesNotExist")}[kind]()
        how = rng.random()
        for p in group:
            p.pod_affinity = [t for t in p.pod_affinity if t.topology_key != HOSTNAME_LABEL]
            p.pod_affinity_preferred = [t for t in p.pod_affinity_preferred if t.term.topology_key != HOSTNAME_LABEL]
            if strip:
                continue
            if how < 0.3:
                p.node_affinity_preferred = list(p.node_affinity_preferred) + [PreferredSchedulingTerm(rng.choice([1, 50]), (r,))]
            elif p.node_affinity_required:
                p.node_affinity_required = [list(t) + [r] for t in p.node_affinity_required]
            else:
                p.node_affinity_required = [[r]]
    return pl


def encode_rules(seed, strip=False):
    pools, per_pool, nodes, pl = fuzz.problem(seed, n_pods=[5, 20, 60, 150][seed % 4])
    fuzz.soften(seed, pools, pl)
    add_rules(seed, pools, nodes, pl, strip)
    return Scheduler(pools, per_pool, nodes, claim_order="go" if seed % 3 else "stable",
                     preference_policy="Ignore" if seed % 5 == 0 else "Respect").encode(pl)


def test_rule_generator_changes_placements():
    """on the oracle, dropping the rules changes where pods go in enough seeds"""
    stats = collections.Counter()
    for seed in range(120):
        try:
            with_rules = oracle_lib.solve(encode_rules(seed).problem)
        except RuntimeError:
            stats["rejected"] += 1
            continue
        without = oracle_lib.solve(encode_rules(seed, strip=True).problem)
        stats["solved"] += 1
        stats["rules_matter"] += int(not np.array_equal(with_rules["pod_target"], without["pod_target"]))
    assert stats["solved"] >= 100 and stats["rules_matter"] >= 25, stats


def run_band(encoder, seeds, monkeypatch=None, env=None):
    for k in ("KP_SMEM_CAP", "KP_NO_DOMAIN_FP", "KP_NO_LEAN", "KP_COHORT", "KP_NO_COHORT"):
        monkeypatch.delenv(k, raising=False)
    for k, v in (env or {}).items():
        monkeypatch.setenv(k, v)
    h = _native.Handle()
    bad, ran = [], 0
    try:
        for seed in seeds:
            enc = encoder(seed)
            try:
                orc = oracle_lib.solve(enc.problem)
            except RuntimeError:
                continue
            try:
                gpu = h.solve(enc.problem)
            except _native.SolverError as e:
                bad.append((seed, f"gpu refused: {e}"))
                continue
            ran += 1
            try:
                assert_same(gpu, orc, f"seed {seed} ")
            except AssertionError as e:
                bad.append((seed, str(e)[:200]))
    finally:
        h.close()
    assert not bad, bad[:10]
    return ran


BANDS = {"default": {}, "no_domain_fp": {"KP_NO_DOMAIN_FP": "1"}, "no_lean": {"KP_NO_LEAN": "1"},
         "cap": {"KP_SMEM_CAP": "0,3,1,0"}}


@pytest.mark.gpu
@pytest.mark.parametrize("band", list(BANDS))
def test_fuzz_rules_parity_gpu(monkeypatch, band):
    assert run_band(encode_rules, range(300), monkeypatch, BANDS[band]) >= 250


def encode_volume_rules(seed):
    """two or three volume alternatives on a third of the pod shapes, each a zone and / or a host rule"""
    pools, per_pool, nodes, pl = fuzz.problem(seed, n_pods=[5, 20, 60, 150][seed % 4])
    rng = random.Random(97_000 + seed)
    names = [n.name for n in nodes] or ["node-000"]
    shapes = {}
    for p in pl:
        key = id(p.requests), tuple(sorted(p.labels.items())), p.namespace
        if key not in shapes:
            alts = []
            if rng.random() < 0.4:
                for _ in range(rng.randint(2, 3)):
                    alt = []
                    if rng.random() < 0.6:
                        alt.append(req(ZONE_LABEL, "In", *rng.sample(fuzz.ZONES, rng.randint(1, 2))))
                    if rng.random() < 0.7 or not alt:
                        alt.append(rng.choice([host("In", rng.choice(names)), host("In", "no-such-host"),
                                               host("NotIn", rng.choice(names))]))
                    alts.append(alt)
            shapes[key] = alts
        if shapes[key]:
            p.volume_requirements = shapes[key]
            p.pod_affinity = [t for t in p.pod_affinity if t.topology_key != HOSTNAME_LABEL]
    return Scheduler(pools, per_pool, nodes, claim_order="go" if seed % 3 else "stable").encode(pl)


@pytest.mark.gpu
def test_fuzz_volume_rules_parity_gpu(monkeypatch):
    assert run_band(encode_volume_rules, range(100), monkeypatch) >= 80


def consolidation_rules_case(seed):
    """a small cluster whose bound pods are pinned to their own node, to another node, or NotIn their own node; three
    seeds of four topology-free (k_consolidate), the fourth with topology (the general path)"""
    rng = random.Random(93_000 + seed)
    its = fuzz.instance_types(rng)
    pools = fuzz.node_pools(rng)
    per_pool = {p.name: its for p in pools}
    nodes = fuzz.state_nodes(rng, its, pools, rng.randint(3, 12), [])
    names = [n.name for n in nodes]
    for n in nodes:
        n.running_pods = []
        cand = fuzz.pods(rng, 10)
        if seed % 4:
            cand = [p for p in cand if not (p.topology_spread_constraints or p.pod_affinity or p.pod_anti_affinity)]
        n.pods = cand[:rng.randint(0, 4)]
        for p in n.pods:
            p.pod_affinity = [t for t in p.pod_affinity if t.topology_key != HOSTNAME_LABEL]
            x = rng.random()
            if x < 0.25:
                p.node_selector = dict(p.node_selector, **{HOSTNAME_LABEL: n.name})
            elif x < 0.45:
                p.node_selector = dict(p.node_selector, **{HOSTNAME_LABEL: rng.choice(names)})
            elif x < 0.65:
                p.node_affinity_required = [list(t) + [host("NotIn", n.name)] for t in p.node_affinity_required] or \
                    [[host("NotIn", n.name)]]
    sets = [rng.sample(names, rng.randint(1, min(3, len(names)))) for _ in range(rng.randint(1, 10))]
    return pools, per_pool, nodes, sets


@pytest.mark.gpu
def test_fuzz_consolidation_rules_parity_gpu():
    bad, ran, decisions = [], 0, collections.Counter()
    for seed in range(200):
        pools, per_pool, nodes, sets = consolidation_rules_case(seed)
        orc = Consolidation(pools, per_pool, nodes, backend=oracle_lib.consolidate)
        try:
            cmds = orc.compute(sets)
        except RuntimeError:
            continue
        gpu = Consolidation(pools, per_pool, nodes)
        try:
            gpu.compute(sets)
        except _native.SolverError as e:
            if e.code == 5 and "minValues" in str(e):  # kp_consolidate refuses NodePools with minValues (so does the oracle)
                continue
            bad.append((seed, str(e)))
            continue
        finally:
            gpu.close()
        ran += 1
        decisions.update(c.decision for c in cmds)
        for k in _abi.CONSOL_PARITY_KEYS:
            if not np.array_equal(gpu.raw[k], orc.raw[k]):
                bad.append((seed, k, gpu.raw[k].tolist()[:8], orc.raw[k].tolist()[:8]))
                break
    assert not bad, bad[:6]
    assert ran >= 120 and decisions["noop"] >= 5 and decisions["delete"] >= 5, (ran, decisions)


@pytest.mark.gpu
def test_batch_mixing_instances_with_and_without_rules():
    encs = [encode_rules(seed, strip=seed % 2 == 0).problem for seed in range(12)]
    ok = []
    for e in encs:
        try:
            oracle_lib.solve(e)
            ok.append(e)
        except RuntimeError:
            pass
    h = _native.Handle()
    try:
        alone = [h.solve(e) for e in ok]
        batch = h.solve_batch(ok)
    finally:
        h.close()
    assert len(ok) >= 8
    for i, (a, b) in enumerate(zip(alone, batch)):
        assert_same(b, a, f"instance {i} ")
