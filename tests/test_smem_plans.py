"""The solver CTA's shared-memory plan (kp_api.cu plan_solve) at every boundary it draws, and every instantiation of
k_wsolve_batch a batch can pick, against the CPU oracle bit for bit.

plan_solve decides per instance which state is on chip: the topology-key group state (tk_groups), the hot claim rows
(requests, threshold rows) of the first CQ claims, the cold rows (requirement slots, instance-type words) of the first
CR <= CQ, and the claim order / failure masks / template ids / c_dom of the first CS (migrated to HBM when a claim id
reaches CS).  KP_SMEM_CAP="CS,CQ,CR,TK" lowers that plan, so small problems cross every boundary; KP_DEBUG=1 makes the
library print the plan it used, which every test reads back to check that the layout it meant to test was the one that
ran and that the claims really outgrew it.  The CPU tier checks the topology-key generator."""
import collections
import os
import re

import numpy as np
import pytest

from karpenter_b200 import _native, kwok, workloads
from karpenter_b200.encode import ProblemBuilder
from karpenter_b200.model import (CAPACITY_TYPE_LABEL, HOSTNAME_LABEL, OS_LABEL, ZONE_LABEL, LabelSelector, NodePool,
                                  NodeSelectorRequirement, Pod, PodAffinityTerm, TopologySpreadConstraint)
from karpenter_b200.scheduler import Scheduler
from tests import oracle_lib
from tests.parity import assert_same
from tests.test_fuzz_parity import (SEEDS, encode, encode_ports, encode_replicas, encode_reserved, encode_soft,
                                    encode_volumes)

CAP = int(os.environ.get("KP_FUZZ_SEEDS", "0"))  # > 0: only that many seeds per band (runs under compute-sanitizer)
# cudaDevAttrMaxSharedMemoryPerBlockOptin of an H100 (sm_90): 227 KB.  No plan may ask for more.
SMEM_OPTIN = 227 * 1024
PLAN = re.compile(r"\[kp\] solver plan: tables (\d+) B, topology-key groups on chip (\d+), hot rows (\d+), cold rows (\d+), "
                  r"small arrays (\d+), (\d+) B shared")
RACK = "example.com/rack"
KNOBS = ("KP_SMEM_CAP", "KP_NO_DOMAIN_FP", "KP_NO_LEAN", "KP_COHORT", "KP_NO_COHORT")


def plans_of(err: str):
    """the solver plan lines of a solve's stderr, in upload order: dicts with tab, tk, CQ, CR, CS, smem"""
    out = [dict(zip(("tab", "tk", "CQ", "CR", "CS", "smem"), map(int, m))) for m in PLAN.findall(err)]
    for p in out:
        assert p["smem"] <= SMEM_OPTIN, p
        assert p["CR"] <= p["CQ"], p
    return out


def set_knobs(monkeypatch, **env):
    """exactly the given KP_* knobs (KP_DEBUG stays on); the library reads them at upload"""
    for k in KNOBS:
        monkeypatch.delenv(k, raising=False)
    for k, v in env.items():
        monkeypatch.setenv(k, v)


def solve_with_plan(h, problem, capfd, deadline_ms=0):
    capfd.readouterr()
    res = h.solve(problem, deadline_ms=deadline_ms)
    return res, plans_of(capfd.readouterr().err)


@pytest.fixture
def debug(monkeypatch):
    set_knobs(monkeypatch)
    monkeypatch.setenv("KP_DEBUG", "1")
    return monkeypatch


@pytest.fixture(scope="module")
def handle():
    h = _native.Handle()
    yield h
    h.close()


# ---- problems ------------------------------------------------------------------------------------------------------
def rack_problem(nv: int, n_apps: int, variant: str = "rack", n_its: int = 120):
    """Apps of nv + 1 pods each on a NodePool that requires a custom rack key In [r0 ... r(nv-1)], so that every rack
    value gets NodeClaims and counts.
    variant "rack": every app spreads on the rack (maxSkew 1) and is anti-affine to itself on the hostname;
    "hostname_mix": every other app keeps the hostname anti-affinity only (fast-path classes without a rack group);
    "ct_mix": every third app spreads on the capacity type instead of the rack (groups the slot map leaves at -1, classes
    off the domain fast path)."""
    racks = tuple(f"r{i}" for i in range(nv))
    pool = NodePool(name="default", requirements=[NodeSelectorRequirement(OS_LABEL, "In", ("linux",)),
                                                  NodeSelectorRequirement(CAPACITY_TYPE_LABEL, "In", ("on-demand", "spot")),
                                                  NodeSelectorRequirement(RACK, "In", racks)])
    pods, uid = [], 1
    for a in range(n_apps):
        labels = {"app": f"app-{a:04d}"}
        sel = LabelSelector.of(labels)
        tsc = [TopologySpreadConstraint(1, RACK, sel)]
        if variant == "hostname_mix" and a % 2:
            tsc = []
        elif variant == "ct_mix" and a % 3 == 2:
            tsc = [TopologySpreadConstraint(1, CAPACITY_TYPE_LABEL, sel)]
        # three request shapes shared by many apps: no class is alone in its (cpu, memory) rank, so the queue is not
        # cohort-shaped and the instance keeps its topology-key state on chip when it fits
        req = {"cpu": f"{250 * (1 + a % 3)}m", "memory": "256Mi"}
        for _ in range(nv + 1):
            pods.append(Pod(name=f"p{uid}", uid=uid * 7919, labels=labels, requests=req, topology_spread_constraints=tsc,
                            pod_anti_affinity=[PodAffinityTerm(sel, HOSTNAME_LABEL)]))
            uid += 1
    return Scheduler([pool], {"default": kwok.aws_instance_types(n_its)}).encode(pods)


def anti_affine_app(n_pods: int):
    """one app whose pods are anti-affine to each other on the hostname: every pod opens its own NodeClaim"""
    b = ProblemBuilder()
    its = kwok.aws_instance_types(100)
    for it in its:
        b.add_instance_type(it)
    b.add_nodepool(workloads.default_nodepool(), list(range(len(its))))
    labels = {"app": "solo"}
    cls = b.pod_class(Pod(labels=labels, requests={"cpu": "500m", "memory": "512Mi"},
                          pod_anti_affinity=[PodAffinityTerm(LabelSelector.of(labels), HOSTNAME_LABEL)]))
    d = workloads.draws(n_pods, 2, 77)
    b.set_pod_arrays(np.full(n_pods, cls, np.int32), np.zeros(n_pods, np.int64), d[:, 0], d[:, 1])
    return b.build().problem


def volume_deployments(n_deployments=30, replicas=100):
    """A Deployment-shaped queue (identical pods per Deployment, a CPU request of its own) where every third Deployment
    has two volume-topology alternatives: cohort-shaped, but the volume-alternative instantiation has no cohorts."""
    its = kwok.aws_instance_types(200)
    zones = kwok.AWS_ZONES
    pods, uid = [], 1
    for a in range(n_deployments):
        labels = {"app": f"vdep-{a:03d}"}
        vol = [[NodeSelectorRequirement(ZONE_LABEL, "In", (zones[a % 4],))],
               [NodeSelectorRequirement(ZONE_LABEL, "In", (zones[(a + 1) % 4],))]] if a % 3 == 0 else []
        for _ in range(replicas):
            pods.append(Pod(name=f"p{uid}", uid=uid * 104729, labels=labels,
                            requests={"cpu": f"{250 + a}m", "memory": "256Mi"}, volume_requirements=vol))
            uid += 1
    return Scheduler([workloads.default_nodepool()], {"default": its}).encode(pods)


_CACHE = {}


def cached(name):
    """(problem, oracle result) of a named problem, built and solved once per session"""
    if name not in _CACHE:
        enc = {
            "c1": lambda: workloads.config_c1(n_pods=1000),
            "c2": lambda: workloads.config_c2(n_pods=30000, n_its=500),
            "c2_300": lambda: workloads.config_c2(n_pods=300, n_its=500),
            "c3": lambda: workloads.config_c3(n_apps=40, replicas=120, n_its=300),
            "c3_1724": lambda: workloads.config_c3(n_apps=40, replicas=120, n_its=1724),
            "deployments": lambda: workloads.config_deployments(40, 300, n_its=300, topology=True),
            "deployments_flat": lambda: workloads.config_deployments(40, 300, n_its=300, topology=False),
            "existing_limits": lambda: workloads.config_existing(limits={"cpu": "3000"}),
            "reserved": lambda: encode_reserved(131),
            "host_ports": lambda: encode_ports(83),
            "volumes": lambda: encode_volumes(83),
            "min_values": lambda: encode_soft(115),
            "volume_deployments": volume_deployments,
        }[name]()
        _CACHE[name] = (enc.problem, oracle_lib.solve(enc.problem, threads=8))
    return _CACHE[name]


# ---- a. the plan-boundary matrix -----------------------------------------------------------------------------------
MATRIX = ["c2", "c3", "deployments", "existing_limits", "reserved", "host_ports", "volumes", "min_values", "c3_1724"]
# cap -> the region whose boundary the claims must cross (tk: the topology-key state is in HBM, nothing to cross)
CAPS = {"0,,,": "CS", ",0,0,": "CQ", ",1,0,": "CQ", ",33,7,": "CQ", "32,64,32,": "CS", ",,,0": "tk"}


def capped(base, cap):
    """the plan KP_SMEM_CAP=cap must leave of the uncapped plan `base`"""
    cs, cq, cr, tk = [None if f == "" else int(f) for f in cap.split(",")]
    want = dict(base)
    if cs is not None:
        want["CS"] = min(base["CS"], cs // 32 * 32)
    if cq is not None:
        want["CQ"] = min(base["CQ"], cq)
    if cr is not None:
        want["CR"] = min(base["CR"], cr)
    want["CR"] = min(want["CR"], want["CQ"])
    if tk is not None and tk < base["tk"]:
        want["tk"] = 0
    return want


@pytest.mark.gpu
@pytest.mark.parametrize("name", MATRIX)
def test_plan_boundary_matrix(handle, debug, capfd, name):
    problem, orc = cached(name)
    set_knobs(debug)
    base_res, (base,) = solve_with_plan(handle, problem, capfd)
    assert_same(base_res, orc, f"{name} uncapped ")
    n = orc["n_claims"]
    assert n > 33, (name, n)  # every cap below is crossed
    for cap, region in CAPS.items():
        set_knobs(debug, KP_SMEM_CAP=cap)
        res, (p,) = solve_with_plan(handle, problem, capfd)
        want = capped(base, cap)
        assert {k: p[k] for k in ("tk", "CQ", "CR", "CS")} == {k: want[k] for k in ("tk", "CQ", "CR", "CS")}, (name, cap, base, p)
        assert p["smem"] <= base["smem"], (name, cap)
        if region == "tk":
            assert p["tk"] == 0
        else:  # the claims outgrow the capped region (the cold rows end at CR <= CQ)
            assert n > p[region], (name, cap, p, n)
        assert_same(res, orc, f"{name} KP_SMEM_CAP={cap} ")
        assert_same(res, base_res, f"{name} KP_SMEM_CAP={cap} vs uncapped ")
        if cap == "32,64,32," and base["CS"] >= 32:
            assert p["CS"] == 32 and p["CQ"] == min(base["CQ"], 64)  # migration while the hot rows stay on chip
    if name.startswith("c3"):
        assert base["tk"] > 0, base  # so ",,,0" moved their topology-key state to HBM


# ---- b. the fuzz bands under caps and knobs ------------------------------------------------------------------------
BANDS = {"hard": (encode, SEEDS), "soft": (encode_soft, range(300)), "reserved": (encode_reserved, range(250)),
         "host_ports": (encode_ports, range(250)), "volumes": (encode_volumes, range(250)),
         # every third seed of the 120-seed band: its oracle solves (600 - 3 000 pods) dominate the run time
         "replicas": (encode_replicas, range(0, 120, 3))}
SETTINGS = {"default": {}, "cap": {"KP_SMEM_CAP": "0,3,1,0"}, "no_domain_fp": {"KP_NO_DOMAIN_FP": "1"},
            "no_lean": {"KP_NO_LEAN": "1"}, "cohort": {"KP_COHORT": "1"}}


@pytest.mark.gpu
@pytest.mark.parametrize("band", list(BANDS))
def test_fuzz_band_under_plans(debug, capfd, band):
    gen, seeds = BANDS[band]
    handles = {s: _native.Handle() for s in SETTINGS}
    bad, ran, crossed = [], 0, 0
    try:
        for seed in list(seeds)[:CAP or None]:
            enc = gen(seed)
            try:
                orc = oracle_lib.solve(enc.problem)
            except RuntimeError:
                continue  # unsupported feature combination (test_fuzz_parity_gpu checks that both sides refuse)
            ran += 1
            crossed += orc["n_claims"] > 3
            for s, env in SETTINGS.items():
                set_knobs(debug, **env)
                try:
                    gpu, plans = solve_with_plan(handles[s], enc.problem, capfd)
                except _native.SolverError as e:
                    bad.append((seed, s, f"gpu refused: {e}"))
                    continue
                if s == "cap":
                    assert all(p["CS"] == 0 and p["CQ"] <= 3 and p["CR"] <= 1 and p["tk"] == 0 for p in plans), (seed, plans)
                try:
                    assert_same(gpu, orc, f"seed {seed} {s} ")
                except AssertionError as e:
                    bad.append((seed, s, str(e)[:200]))
    finally:
        for h in handles.values():
            h.close()
    assert not bad, bad[:10]
    assert ran >= len(list(seeds)[:CAP or None]) * 3 // 4, ran
    assert crossed >= ran // 10, (crossed, ran)  # enough seeds open more claims than KP_SMEM_CAP=0,3,1,0 keeps on chip


# ---- c. topology-key shapes ----------------------------------------------------------------------------------------
# (nv, apps, variant, state on chip?).  On-chip state is the slot map (4 B per group) + 16 B of masks and 4 * nv B of
# counters per rack group: at nv = 64 the 64 KB limit lies near 230 apps.
RACK_CASES = [(1, 40, "rack", True), (3, 60, "rack", True), (32, 120, "rack", True), (33, 120, "rack", True),
              (64, 200, "rack", True), (64, 260, "rack", False), (64, 160, "hostname_mix", True),
              (33, 150, "ct_mix", True)]
RACK_IDS = [f"nv{nv}-{apps}-{v}" for nv, apps, v, _ in RACK_CASES]


def test_rack_generator_puts_groups_on_the_rack_key():
    for nv, apps, variant, _ in RACK_CASES:
        enc = rack_problem(nv, apps, variant)
        assert len(enc.values[RACK]) == nv, (nv, enc.values[RACK])
        p = enc.problem
        k = enc.key_id(RACK)
        assert p.get("key_value_off")[k + 1] - p.get("key_value_off")[k] == nv
        # distinct topology groups per key: plan_classes picks the non-hostname key most groups sit on
        cols = [np.asarray(p.get("tsc_" + c)) for c in ("type", "key", "selector", "nsset", "max_skew")]
        groups = collections.Counter(int(row[1]) for row in set(zip(*[c.tolist() for c in cols])))
        other = [n for key, n in groups.items() if key not in (k, enc.key_id(HOSTNAME_LABEL))]
        assert groups[k] > max(other, default=0), (nv, variant, groups)
        if variant == "ct_mix":
            assert groups[enc.key_id(CAPACITY_TYPE_LABEL)] > 0
        res = oracle_lib.solve(p)
        assert res["n_groups"] > apps and (res["pod_target"] != -1).all(), (nv, apps, variant)
        if variant == "rack":  # the spread pins every NodeClaim to one rack, and every rack gets some
            pinned = [tuple(enc.decode_requirements(res, c)[RACK]["values"]) for c in range(res["n_claims"])]
            assert all(len(v) == 1 for v in pinned) and len(set(pinned)) == nv, (nv, pinned[:5])


@pytest.mark.gpu
@pytest.mark.parametrize("nv,apps,variant,on_chip", RACK_CASES, ids=RACK_IDS)
def test_topology_key_shapes(handle, debug, capfd, nv, apps, variant, on_chip):
    enc = rack_problem(nv, apps, variant)
    orc = oracle_lib.solve(enc.problem, threads=8)
    res, (p,) = solve_with_plan(handle, enc.problem, capfd)
    assert (p["tk"] > 0) == on_chip, (nv, apps, variant, p)
    assert_same(res, orc, f"rack nv={nv} apps={apps} {variant} ")
    if on_chip:  # and the same problem with the state in HBM
        set_knobs(debug, KP_SMEM_CAP=",,,0")
        res, (p,) = solve_with_plan(handle, enc.problem, capfd)
        assert p["tk"] == 0
        assert_same(res, orc, f"rack nv={nv} apps={apps} {variant} in HBM ")


# ---- d. batches whose instances run in a foreign instantiation -----------------------------------------------------
BATCHES = {
    "c3+deployments": (["c3", "deployments"], True),             # cohort kernel: C3's planned on-chip state dropped
    "deployments+volumes": (["deployments", "volumes"], False),  # VOL kernel, an instance with d.cohort = 1
    "c2+c3": (["c2", "c3"], False),                              # a lean instance in the full kernel
    "c1+deployments_flat": (["c1", "deployments_flat"], True),   # the lean cohort kernel
    "volume_deployments": (["volume_deployments"], False),       # cohort-shaped, cohort reset by the volume alternatives
}


@pytest.mark.gpu
@pytest.mark.parametrize("batch", list(BATCHES))
def test_mixed_instantiation_batch(handle, debug, capfd, batch):
    names, cohort_kernel = BATCHES[batch]
    probs = [cached(n) for n in names]
    solo = [handle.solve(p) for p, _ in probs]
    for (p, orc), s, n in zip(probs, solo, names):
        assert_same(s, orc, f"{n} solo ")
    capfd.readouterr()
    runs = [("solve_batch", handle.solve_batch([p for p, _ in probs]), handle.stats())]
    handle.upload_batch([p for p, _ in probs])
    for i in range(2):
        runs.append((f"resident {i}", handle.solve_batch_resident(), handle.stats()))
    plans = plans_of(capfd.readouterr().err)
    assert len(plans) == 2 * len(names), plans  # one upload each for solve_batch and upload_batch: no claim growth
    for what, outs, st in runs:
        for (p, orc), s, n, o in zip(probs, solo, names, outs):
            assert_same(o, orc, f"{batch} {what} {n} ")
            assert_same(o, s, f"{batch} {what} {n} vs solo ")
        assert (st["cohort_pods"] > 0) == cohort_kernel, (batch, what, st["cohort_pods"])
    if batch == "c3+deployments":
        assert plans[0]["tk"] > 0  # C3 planned on-chip topology-key state the cohort kernel does not stage
    if batch == "volume_deployments":
        assert plans[0]["tk"] == 0


# ---- e. claim capacity ---------------------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("n_pods,uploads", [(5000, 2), (3000, 1)])
def test_claims_grow_or_fill_capacity(handle, debug, capfd, n_pods, uploads):
    """5 000 pods: the first upload has room for 4 096 claims (cmax_guess), the solve runs out and is redone with 5 000.
    3 000 pods: Cmax = P = 3 000 and the claims fill it exactly."""
    problem = anti_affine_app(n_pods)
    orc = oracle_lib.solve(problem, threads=8)
    assert orc["n_claims"] == n_pods
    res, plans = solve_with_plan(handle, problem, capfd)
    assert len(plans) == uploads, plans
    assert_same(res, orc, f"{n_pods} anti-affine pods ")


@pytest.mark.gpu
def test_batch_where_one_instance_grows(handle, debug, capfd):
    big = anti_affine_app(5000)
    small, small_orc = cached("c2_300")
    capfd.readouterr()
    outs = handle.solve_batch([big, small])
    plans = plans_of(capfd.readouterr().err)
    assert len(plans) == 4, plans  # two instances, uploaded twice
    assert_same(outs[0], oracle_lib.solve(big, threads=8), "batch grown ")
    assert_same(outs[1], small_orc, "batch C2[300] ")


# ---- f. the deadline with on-chip state ----------------------------------------------------------------------------
@pytest.mark.gpu
def test_deadline_flushes_on_chip_state(handle, debug, capfd):
    """A partial C3 solve with topology-key state and hot rows on chip: what it placed and the counters it reports must
    be written back at the deadline like at the end of a full solve."""
    apps, replicas = 400, 250
    enc = workloads.config_c3(n_apps=apps, replicas=replicas, n_its=1000)
    full, _ = solve_with_plan(handle, enc.problem, capfd)
    assert not full["deadline"]
    set_knobs(debug, KP_SMEM_CAP=",4,2,")  # (about 20 claims are open at the deadline)
    part, (p,) = solve_with_plan(handle, enc.problem, capfd, deadline_ms=20)
    assert part["deadline"], f"the solve finished inside 20 ms (full solve {full['solve_ms']:.1f} ms): make it larger"
    assert p["tk"] > 0 and p["CQ"] == 4 and part["n_claims"] > p["CQ"], (p, part["n_claims"])
    tgt = part["pod_target"]
    placed = tgt != -1
    assert 0 < placed.sum() < len(tgt)
    assert np.array_equal(tgt[placed], full["pod_target"][placed])
    assert np.all(tgt[placed] <= -2)  # no existing nodes: every placed pod is on a claim
    claim = -2 - tgt[placed]
    assert np.array_equal(part["claim_npods"], np.bincount(claim, minlength=part["n_claims"]))
    # the zone of every claim, from its requirement mask on the zone key
    zk = enc.key_id(ZONE_LABEL)
    woff = sum(0 if k == HOSTNAME_LABEL else (len(enc.values[k]) + 63) // 64 for k in enc.keys[:zk])
    nz = len(enc.values[ZONE_LABEL])
    masks = part["claim_req_mask"][:, woff].astype(np.uint64)
    zone = np.array([int(m).bit_length() - 1 if int(m) and not int(m) & (int(m) - 1) else -1 for m in masks])
    assert np.all(zone[claim] >= 0), "every claim of a zonal spread is pinned to one zone"
    app = (np.arange(len(tgt)) // replicas)[placed]
    want = np.zeros((apps, nz), np.int32)
    np.add.at(want, (app, zone[claim]), 1)
    off = part["group_domain_off"]
    got = [tuple(part["domain_counts"][off[g]:off[g + 1]]) for g in range(part["n_groups"]) if off[g + 1] > off[g]]
    assert len(got) == apps
    # one zone group per app; compared as multisets, so the test does not depend on the group numbering
    assert sorted(got) == sorted(tuple(r) for r in want)
