"""Consolidation of clusters whose pods have several volume-topology alternatives (PodData.VolumeRequirements: a PV node
affinity or a StorageClass allowedTopologies with several terms, volumetopology.go:44-125).  Every simulation tries the
alternatives in turn on each existing node (existingnode.go:98-113) and each NodeClaim (nodeclaim.go:136-176), for the
candidates' pods, the pending pods and the pods of deleting nodes alike (helpers.go:65-91).
CPU tier: the oracle; GPU tier: kp_consolidate (k_consolidate<false, true> for topology-free candidate sets, the
volume-alternative k_wsolve_batch instantiation on the general path), bit-identical to the oracle."""
import collections
import random
import re

import numpy as np
import pytest

from karpenter_b200 import _abi, _native, fake, workloads
from karpenter_b200.disruption import (Consolidation, MultiNodeConsolidation, SingleNodeConsolidation,
                                       validate_command)
from karpenter_b200.model import (CAPACITY_TYPE_LABEL, ZONE_LABEL, LabelSelector, NodePool, NodeSelectorRequirement,
                                  Pod, PodAffinityTerm, TopologySpreadConstraint)
from tests import fuzz, oracle_lib
from tests.test_fuzz_parity import consolidation_case, consolidation_extras
from tests.test_hostname_requirements import cnode

BACKENDS = [pytest.param("oracle", id="oracle"), pytest.param("gpu", id="gpu", marks=pytest.mark.gpu)]
ARM = {it.name: it for it in fake.default_instance_types()}["arm-instance-type"]


def zone(*z):
    return [NodeSelectorRequirement(ZONE_LABEL, "In", tuple(z))]


def pool():
    return NodePool(name="default", requirements=[NodeSelectorRequirement(CAPACITY_TYPE_LABEL, "In", ("on-demand",))])


def vpod(name, uid, alts=None, cpu="100m", **kw):
    return Pod(name=name, uid=uid, requests={"cpu": cpu}, volume_requirements=[zone(*a) for a in alts or []], **kw)


def engine(which, nodes, **kw):
    its = {"default": fake.default_instance_types()}
    if which == "oracle":
        kw = dict(kw, backend=oracle_lib.consolidate, solve_backend=oracle_lib.solve)
    return Consolidation([pool()], its, nodes, **kw)


def consolidate(which, nodes, sets, **kw):
    """Commands of the candidate sets; on the GPU tier every parity key also equals the oracle's"""
    eng = engine(which, nodes, **kw)
    try:
        cmds = eng.compute(sets)
        if which == "gpu":
            orc = engine("oracle", nodes, **kw)
            assert orc.compute(sets) == cmds
            for k in _abi.CONSOL_PARITY_KEYS:
                assert np.array_equal(eng.raw[k], orc.raw[k]), k
        return cmds
    finally:
        eng.close()


def zone_of(cmd):
    v = cmd.replacement_requirements[ZONE_LABEL]
    assert not v["complement"], v
    return list(v["values"])


def cluster(alts, other_zone="test-zone-2", other_room=True):
    """node-0: a half-empty arm node in test-zone-1 whose one pod has the alternatives `alts`; node-1: an arm node in
    `other_zone`, half-empty or full"""
    p0 = vpod("p0", 1, alts)
    fill = [vpod(f"f{i}", 100 + i, cpu="15") for i in range(0 if other_room else 1)]
    return [cnode("node-0", ARM, [p0]), cnode("node-1", ARM, [vpod("p1", 2)] + fill, zone=other_zone)]


# ---- hand-built clusters -------------------------------------------------------------------------------------------
@pytest.mark.parametrize("which", BACKENDS)
def test_pod_moves_through_its_second_alternative(which):  # existingnode.go:98-113
    c = consolidate(which, cluster([["test-zone-1"], ["test-zone-2"]]), [["node-0"]])[0]
    assert c.decision == "delete" and c.n_new_node_claims == 0 and c.n_unscheduled == 0
    # the first alternative alone admits no node: the pod needs a NodeClaim
    c = consolidate(which, cluster([["test-zone-1"]]), [["node-0"]])[0]
    assert c.decision == "replace"


@pytest.mark.parametrize("which", BACKENDS)
def test_replacement_takes_the_first_alternative(which):  # nodeclaim.go:136-153
    c = consolidate(which, cluster([["test-zone-1"], ["test-zone-3"]]), [["node-0"]])[0]
    assert c.decision == "replace" and c.n_new_node_claims == 1 and c.n_unscheduled == 0
    assert zone_of(c) == ["test-zone-1"]
    assert c.replacement_instance_types and "arm-instance-type" not in c.replacement_instance_types


@pytest.mark.parametrize("which", BACKENDS)
def test_replacement_pinned_to_the_second_alternative(which):
    c = consolidate(which, cluster([["no-such-zone"], ["test-zone-3"]]), [["node-0"]])[0]
    assert c.decision == "replace" and c.n_new_node_claims == 1 and zone_of(c) == ["test-zone-3"]


@pytest.mark.parametrize("which", BACKENDS)
def test_no_alternative_satisfiable_is_a_noop(which):
    c = consolidate(which, cluster([["no-such-zone"], ["nor-this-one"]]), [["node-0"]])[0]
    assert c.decision == "noop" and c.n_unscheduled == 1


@pytest.mark.parametrize("which", BACKENDS)
def test_pending_and_deleting_node_pods_walk_their_alternatives(which):  # helpers.go:65-91
    nodes = cluster(None)
    pend = [vpod("pend", 50, [["test-zone-3"], ["test-zone-2"]])]
    dele = [vpod("dele", 51, [["no-such-zone"], ["test-zone-2"]])]
    c = consolidate(which, nodes, [["node-0"]], pending_pods=pend, deleting_node_pods=dele)[0]
    assert c.decision == "delete" and c.n_unscheduled == 0  # both land on node-1 through their second alternative
    # a pod of a deleting node that fits nowhere blocks the command; a pending one is not counted (scheduler.go:330-334)
    stuck = [vpod("dele", 51, [["no-such-zone"], ["nor-this-one"]])]
    c = consolidate(which, nodes, [["node-0"]], pending_pods=pend, deleting_node_pods=stuck)[0]
    assert c.decision == "noop" and c.n_unscheduled == 1
    c = consolidate(which, nodes, [["node-0"]], pending_pods=stuck, deleting_node_pods=dele)[0]
    assert c.decision == "delete" and c.n_unscheduled == 0


@pytest.mark.parametrize("which", BACKENDS)
def test_chain_on_a_node_outside_the_set_changes_nothing(which):
    def nodes(alts):
        return [cnode("node-0", ARM, [vpod("p0", 1)]), cnode("node-1", ARM, [vpod("p1", 2)], zone="test-zone-2"),
                cnode("node-2", ARM, [vpod("p2", 3, alts)], zone="test-zone-3")]
    sets = [["node-0"], ["node-1"], ["node-0", "node-1"]]
    with_chain = consolidate(which, nodes([["test-zone-3"], ["test-zone-1"]]), sets)
    assert with_chain == consolidate(which, nodes(None), sets)
    assert {c.decision for c in with_chain} == {"delete"}


@pytest.mark.parametrize("which", BACKENDS)
def test_zonal_anti_affinity_with_two_zone_storage_class(which):  # suite_test.go:2994-3038 as a consolidation
    labels = {"app": "multi-zone-sc-app"}
    anti = [PodAffinityTerm(LabelSelector.of(labels), ZONE_LABEL)]

    def sc_pod(i):
        return vpod(f"sc-pod-{i}", 10 + i, [["test-zone-1"], ["test-zone-2"]], labels=labels, pod_anti_affinity=anti)
    nodes = [cnode("node-0", ARM, [sc_pod(0)]), cnode("node-1", ARM, [sc_pod(1)], zone="test-zone-2"),
             cnode("node-2", ARM, [vpod("p2", 3)], zone="test-zone-2")]
    pair, one = consolidate(which, nodes, [["node-0", "node-1"], ["node-0"]])
    # the first pod goes to node-2 through its second alternative; the anti-affinity keeps the second out of test-zone-2,
    # so it opens a NodeClaim through its first alternative
    assert pair.decision == "replace" and pair.n_new_node_claims == 1 and zone_of(pair) == ["test-zone-1"]
    # sc-pod-1 still runs in test-zone-2: sc-pod-0 can only go to a NodeClaim in test-zone-1
    assert one.decision == "replace" and zone_of(one) == ["test-zone-1"]


def frontend_cluster():
    """six nodes in three zones; half of them run a pod with two zone alternatives"""
    nodes, uid = [], 1
    for n in range(6):
        z = f"test-zone-{n % 3 + 1}"
        pl = [vpod(f"p{uid}", uid)]
        uid += 1
        if n % 2 == 0:
            pl.append(vpod(f"p{uid}", uid, [[f"test-zone-{(n + 1) % 3 + 1}"], [z]], cpu="500m"))
            uid += 1
        nodes.append(cnode(f"node-{n}", ARM, pl, zone=z))
    return nodes


@pytest.mark.parametrize("which", BACKENDS)
def test_frontend_passes_on_a_cluster_with_chains(which):
    nodes = frontend_cluster()
    budgets = {"default": 10}
    out = []
    for method in (SingleNodeConsolidation, MultiNodeConsolidation):
        eng = engine(which, nodes)
        try:
            cmd, names, _ = method(eng).compute_command(nodes, budgets)
            assert cmd is not None and names
            out.append((cmd, names, validate_command(eng, cmd, names)))
        finally:
            eng.close()
    assert all(ok for _, _, ok in out)
    if which == "gpu":
        ref = []
        for method in (SingleNodeConsolidation, MultiNodeConsolidation):
            eng = engine("oracle", nodes)
            cmd, names, _ = method(eng).compute_command(nodes, budgets)
            ref.append((cmd, names, validate_command(eng, cmd, names)))
        assert out == ref


# ---- fuzz band -----------------------------------------------------------------------------------------------------
def add_volume_alternatives(seed, pods):
    """2 - 3 zone alternatives (sometimes with a capacity type) on a third of the pod shapes (own random stream)"""
    rng = random.Random(61_000 + seed)
    shapes = {}
    for p in pods:
        key = id(p.requests), tuple(sorted(p.labels.items())), p.namespace
        if key not in shapes:
            alts = []
            if rng.random() < 1 / 3:
                for _ in range(rng.randint(2, 3)):
                    alt = [NodeSelectorRequirement(ZONE_LABEL, "In", tuple(rng.sample(fuzz.ZONES + ["no-such-zone"],
                                                                                      rng.randint(1, 2))))]
                    if rng.random() < 0.3:
                        alt.append(NodeSelectorRequirement(CAPACITY_TYPE_LABEL, "In", (rng.choice(fuzz.CTS),)))
                    alts.append(alt)
            shapes[key] = alts
        if shapes[key]:
            p.volume_requirements = shapes[key]


def volume_consolidation_case(seed):
    """consolidation_case with volume alternatives on the bound pods and the extra pods: three seeds of four
    topology-free (k_consolidate), the fourth with topology (the general path)"""
    pools, per_pool, nodes, sets, s2s = consolidation_case(seed)
    extras = consolidation_extras(seed)
    add_volume_alternatives(seed, [p for n in nodes for p in n.pods] + [p for v in extras.values() for p in v])
    kw = dict(spot_to_spot=s2s, filter_same_instance_type=seed % 2 == 1, price_order=seed % 5 == 0, **extras)
    return pools, per_pool, nodes, sets, kw


def test_volume_consolidation_generator_uses_later_alternatives():
    """on the oracle, cutting every chain to its first alternative changes the decisions in enough seeds"""
    stats = collections.Counter()
    for seed in range(120):
        pools, per_pool, nodes, sets, kw = volume_consolidation_case(seed)
        enc, consol = Consolidation(pools, per_pool, nodes, **kw)._encode(sets)
        nxt = enc.problem.get("class_vol_next")
        if nxt is None or not (nxt >= 0).any():
            continue
        try:
            full = oracle_lib.consolidate(enc.problem, consol)
        except RuntimeError:
            continue
        stats["chains"] += 1
        enc.problem.set("class_vol_next", np.full_like(nxt, -1))
        first = oracle_lib.consolidate(enc.problem, consol)
        stats["later_alternative_matters"] += int(any(not np.array_equal(full[k], first[k])
                                                      for k in _abi.CONSOL_PARITY_KEYS))
    assert stats["chains"] >= 60 and stats["later_alternative_matters"] >= 15, stats


@pytest.mark.gpu
def test_fuzz_volume_consolidation_parity_gpu():
    bad, ran, decisions, paths = [], 0, collections.Counter(), collections.Counter()
    for seed in range(200):
        pools, per_pool, nodes, sets, kw = volume_consolidation_case(seed)
        orc = Consolidation(pools, per_pool, nodes, backend=oracle_lib.consolidate, **kw)
        try:
            cmds = orc.compute(sets)
        except RuntimeError:
            continue
        gpu = Consolidation(pools, per_pool, nodes, **kw)
        try:
            gpu.compute(sets)
        except _native.SolverError as e:
            if e.code == 5 and "minValues" in str(e):  # BestEffort minValues stays refused (so does the oracle)
                continue
            bad.append((seed, str(e)))
            continue
        finally:
            gpu.close()
        ran += 1
        paths["general" if seed % 4 == 0 else "k_consolidate"] += 1
        decisions.update(c.decision for c in cmds)
        for k in _abi.CONSOL_PARITY_KEYS + (["repl_order_off", "repl_order"] if kw["price_order"] else []):
            if not np.array_equal(gpu.raw[k], orc.raw[k]):
                bad.append((seed, k, gpu.raw[k].tolist()[:8], orc.raw[k].tolist()[:8]))
                break
    assert not bad, bad[:6]
    assert ran >= 120 and min(decisions[d] for d in ("noop", "delete", "replace")) >= 5, (ran, decisions)
    assert paths["general"] >= 20, paths


# ---- which kernel serves it (KP_DEBUG) -----------------------------------------------------------------------------
CONSOL_PLAN = re.compile(r"\[kp\] consolidate plan: .*kernel (k_consolidate<[a-z, ]+>)")
SOLVE_KERNEL = re.compile(r"\[kp\] \d+ instance\(s\), kernel (k_wsolve_batch<[a-z, ]+>)")


def kernels_of(capfd, run):
    capfd.readouterr()
    out = run()
    err = capfd.readouterr().err
    return out, CONSOL_PLAN.findall(err), SOLVE_KERNEL.findall(err)


@pytest.mark.gpu
def test_instantiation_follows_the_chains(monkeypatch, capfd):
    monkeypatch.setenv("KP_DEBUG", "1")
    monkeypatch.delenv("KP_NO_LEAN", raising=False)
    sets = [["node-0"]]
    # topology-free: the volume-alternative k_consolidate with a chain, the lean one without
    _, consol, _ = kernels_of(capfd, lambda: consolidate("gpu", cluster([["test-zone-1"], ["test-zone-2"]]), sets))
    assert consol == ["k_consolidate<false, true>"]
    _, consol, _ = kernels_of(capfd, lambda: consolidate("gpu", cluster([["test-zone-1"]]), sets))
    assert consol == ["k_consolidate<true>"]
    # host ports leave the lean instantiation: k_consolidate<false>, as before
    nodes = cluster(None)
    nodes[0].pods[0].host_ports = [("", 80, "TCP")]
    _, consol, _ = kernels_of(capfd, lambda: consolidate("gpu", nodes, sets))
    assert consol == ["k_consolidate<false>"]
    # C4 as it is: the lean instantiation; with chains: the volume-alternative one
    for vol, want in ((0, "k_consolidate<true>"), (20, "k_consolidate<false, true>")):
        enc, kw = workloads.config_c4(n_nodes=300, n_pods=1500, n_candidates=12, max_subset=2, vol_alts=vol)
        h = _native.Handle()
        try:
            _, consol, _ = kernels_of(capfd, lambda: h.consolidate(enc.problem, _abi.ConsolInput(**kw)))
        finally:
            h.close()
        assert consol == [want]
    # topology on the evicted pods: the general path, whose chunk takes the volume-alternative k_wsolve_batch
    cmds, consol, solve = kernels_of(capfd, lambda: consolidate("gpu", topology_cluster(True), topology_sets()))
    assert consol == [] and solve and set(solve) == {"k_wsolve_batch<false, false, true>"}
    cmds, consol, solve = kernels_of(capfd, lambda: consolidate("gpu", topology_cluster(False), topology_sets()))
    assert consol == [] and solve and "k_wsolve_batch<false, false, true>" not in solve


# ---- the general path ----------------------------------------------------------------------------------------------
def topology_cluster(chains):
    """eight nodes whose pods spread over zones; with `chains` the pods of every other node also have two zone
    alternatives"""
    rng = random.Random(5)
    nodes, uid = [], 1
    for n in range(8):
        z = f"test-zone-{n % 3 + 1}"
        pl = []
        for _ in range(rng.randint(1, 3)):
            app = {"app": f"a{rng.randrange(3)}"}
            alts = [[f"test-zone-{rng.randint(1, 3)}"], [z]] if chains and n % 2 == 0 else None
            pl.append(vpod(f"p{uid}", uid, alts, cpu=rng.choice(["250m", "1", "2"]), labels=app,
                           topology_spread_constraints=[TopologySpreadConstraint(1, ZONE_LABEL, LabelSelector.of(app))]))
            uid += 1
        nodes.append(cnode(f"node-{n}", ARM, pl, zone=z))
    return nodes


def topology_sets():
    rng = random.Random(6)
    names = [f"node-{n}" for n in range(8)]
    return [rng.sample(names, rng.randint(1, 3)) for _ in range(24)]


def test_topology_cluster_has_chains_and_decisions():
    """the general-path cluster below: chains on the even nodes, sets with and without them, several decisions"""
    sets = topology_sets()
    touches = [any(int(n[-1]) % 2 == 0 for n in s) for s in sets]
    assert any(touches) and not all(touches)
    cmds = consolidate("oracle", topology_cluster(True), sets)
    assert len({c.decision for c in cmds}) >= 2


@pytest.mark.gpu
def test_general_path_chunk_mixing_sets_with_and_without_chains():
    nodes, sets = topology_cluster(True), topology_sets()
    together = consolidate("gpu", nodes, sets)  # one chunk, bit-identical to the oracle
    eng = engine("gpu", nodes)
    try:
        alone = [eng.compute([s])[0] for s in sets]
    finally:
        eng.close()
    assert together == alone


# ---- C4 with chains at full size -----------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def c4_vol():
    enc, consol = workloads.config_c4(vol_alts=1000)
    h = _native.Handle()
    try:
        full = h.consolidate(enc.problem, _abi.ConsolInput(**consol))
        part = h.consolidate(enc.problem, _abi.ConsolInput(**consol), deadline_ms=1)
    finally:
        h.close()
    return enc, consol, full, part


def chain_nodes(enc, consol):
    """nodes that run a pod with volume alternatives"""
    nxt = enc.problem.get("class_vol_next")
    cls = enc.problem.get("pod_class")
    off = consol["node_pod_off"]
    has = nxt[cls] >= 0
    return np.array([has[off[n]:off[n + 1]].any() for n in range(len(off) - 1)])


def test_c4_vol_alts_cluster():
    """config_c4(vol_alts=...) changes only the chosen pods' classes: that many chain nodes, every tenth candidate among them"""
    enc, consol = workloads.config_c4(n_nodes=2000, n_pods=40_000, vol_alts=100)
    plain, _ = workloads.config_c4(n_nodes=2000, n_pods=40_000)
    on = chain_nodes(enc, consol)
    assert on.sum() == 100 and on[np.unique(consol["subset_nodes"])].sum() == 10
    assert plain.problem.get("class_vol_next") is None or not (plain.problem.get("class_vol_next") >= 0).any()
    assert (enc.problem.get("pod_class") != plain.problem.get("pod_class")).sum() == 100


@pytest.mark.gpu
def test_c4_vol_alts_full_size_sampled_parity(c4_vol):
    enc, consol, gpu, _ = c4_vol
    assert enc.problem.n_nodes == 10000 and enc.problem.n_pods == 200000
    S = consol["n_subsets"]
    assert S == 166750 and len(gpu["decision"]) == S and not gpu["deadline"]
    dec, nnew, uns = gpu["decision"], gpu["n_new_claims"], gpu["n_unscheduled"]
    assert np.all(nnew[dec == 1] == 0) and np.all(nnew[dec == 2] == 1) and np.all(uns[dec != 0] == 0)
    assert np.all(gpu["replacement_its"][dec != 2] == 0) and np.all(gpu["replacement_its"][dec == 2].any(axis=1))
    assert len(set(dec.tolist())) == 3
    off, nodes = consol["subset_off"], consol["subset_nodes"]
    size = off[1:] - off[:-1]
    on = chain_nodes(enc, consol)
    touch = np.array([on[nodes[off[i]:off[i + 1]]].any() for i in range(S)])
    rng = np.random.default_rng(11)
    pick = [np.nonzero(size == 1)[0]]
    for k in (0, 1, 2):  # every delete, up to 1 200 no-ops and replaces
        idx = np.nonzero((dec == k) & (size > 1) & ~touch)[0]
        pick.append(rng.choice(idx, min(len(idx), 1200), replace=False))
    tidx = np.nonzero(touch)[0]
    pick.append(rng.choice(tidx, min(len(tidx), 1200), replace=False))
    pick = np.unique(np.concatenate(pick))
    assert (~touch[pick]).sum() >= 2000 and touch[pick].sum() >= 1000 and set(dec[pick].tolist()) == {0, 1, 2}
    assert len(set(dec[pick][touch[pick]].tolist())) >= 2
    smp = dict(consol, n_subsets=len(pick), subset_off=np.concatenate([[0], np.cumsum(size[pick])]).astype(np.int32),
               subset_nodes=np.concatenate([nodes[off[i]:off[i + 1]] for i in pick]).astype(np.int32))
    orc = oracle_lib.consolidate(enc.problem, _abi.ConsolInput(**smp), threads=8)
    for k in ("decision", "n_new_claims", "n_unscheduled", "replacement_its"):
        assert np.array_equal(gpu[k][pick], orc[k]), (k, np.argwhere(gpu[k][pick] != orc[k])[:5].tolist())


@pytest.mark.gpu
def test_c4_vol_alts_deadline_keeps_finished_subsets(c4_vol):
    _, _, full, part = c4_vol
    assert part["deadline"]
    done = part["decision"] != 255
    assert done.sum() < len(done)
    for k in ("decision", "n_new_claims", "n_unscheduled", "replacement_its"):
        assert np.array_equal(part[k][done], full[k][done]), k
