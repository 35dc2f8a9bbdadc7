"""Hostname topology records (kp_kernels.cuh host_record) and the bootstrap rule of hostname pod affinity.

The solver keeps one flag per hostname group, g_anypop: "some domain of the group is populated", set at prep from the
existing nodes' pods and by every record, never cleared during a solve.  A self-selecting hostname affinity may open a
fresh domain only while it is clear (topologygroup.go:356-374), and anti-affinity reads the presence bit the record sets.
Each case is checked against the oracle bit for bit; the C3 shape also checks that no NodeClaim holds two pods of one
app, which is what a stale presence bit would break."""
import numpy as np
import pytest

from karpenter_b200 import _native, fake, workloads
from karpenter_b200.model import (CAPACITY_TYPE_LABEL, HOSTNAME_LABEL, LabelSelector, NodePool, Pod, PodAffinityTerm,
                                  StateNode)
from karpenter_b200.scheduler import Scheduler
from tests import oracle_lib
from tests.parity import assert_same
from tests.test_reference_scenarios import req
from tests.test_smem_plans import plans_of

N_APPS, PER_APP = 4, 10


def app_labels(a):
    return {"app": f"aff-{a}"}


def self_affine(n_apps, per_app, uid0=1):
    """per_app pods of each app, each pod affine on the hostname to its own app's pods"""
    pods, uid = [], uid0
    for a in range(n_apps):
        labels = app_labels(a)
        for _ in range(per_app):
            pods.append(Pod(name=f"p{uid}", uid=uid, labels=labels,
                            pod_affinity=[PodAffinityTerm(LabelSelector.of(labels), HOSTNAME_LABEL)]))
            uid += 1
    return pods


def encode(pods, state_nodes=()):
    pool = NodePool(name="default", requirements=[req(CAPACITY_TYPE_LABEL, "In", "spot", "on-demand", "reserved")])
    its = fake.default_instance_types()
    return Scheduler([pool], {"default": its}, state_nodes=list(state_nodes)).encode(pods).problem


def empty_start():
    """nothing populated at the start: every app's first pod opens a domain, later pods must join it"""
    return encode(self_affine(N_APPS, PER_APP))


def existing_match():
    """an existing node already runs a pod of app 0, so app 0's group starts populated: its pods may only go to that
    node (room for two), never to a fresh NodeClaim.  The other apps start empty."""
    running = Pod(name="bound", uid=10 ** 6, labels=app_labels(0))
    node = StateNode(name="node-0", labels={HOSTNAME_LABEL: "node-0"}, managed=False, running_pods=[running],
                     available={"cpu": "2", "memory": "4Gi", "pods": 2}, capacity={"cpu": "4", "memory": "8Gi", "pods": 10})
    return encode(self_affine(N_APPS, PER_APP), [node])


def claims_of(res):
    t = res["pod_target"]
    return np.where(t <= -2, -2 - t, -1)


def check_one_domain_per_app(res, n_existing):
    """every app's placed pods share one domain, and no app places all its pods (that domain fills up and the group,
    once populated, may not open another)"""
    t = res["pod_target"]
    for a in range(N_APPS):
        ta = t[a * PER_APP:(a + 1) * PER_APP]
        placed = ta[ta != -1]
        assert 0 < len(placed) < PER_APP, (a, ta.tolist())
        assert len(set(placed.tolist())) == 1, (a, ta.tolist())
    if n_existing:
        ta = t[:PER_APP]
        assert (ta[ta != -1] == 0).all(), ta.tolist()  # app 0 joins the existing node's pod


@pytest.fixture(scope="module")
def handle():
    h = _native.Handle()
    yield h
    h.close()


@pytest.mark.gpu
def test_self_affinity_from_empty(handle):
    problem = empty_start()
    res = handle.solve(problem)
    assert_same(res, oracle_lib.solve(problem), "empty start ")
    check_one_domain_per_app(res, 0)


@pytest.mark.gpu
def test_self_affinity_existing_node_populates_at_prep(handle):
    problem = existing_match()
    res = handle.solve(problem)
    assert_same(res, oracle_lib.solve(problem), "existing node ")
    check_one_domain_per_app(res, 1)


@pytest.mark.gpu
@pytest.mark.parametrize("make", [empty_start, existing_match], ids=["empty_start", "existing_match"])
def test_flag_reset_between_resident_solves(handle, make):
    """the flags a solve sets must not survive into the next solve of the same upload"""
    problem = make()
    orc = oracle_lib.solve(problem)
    handle.upload(problem)
    for i in range(2):
        assert_same(handle.solve_resident(), orc, f"resident solve {i} ")


APPS, REPLICAS = 20, 200
_C3 = {}


def c3_shape():
    if not _C3:
        problem = workloads.config_c3(n_apps=APPS, replicas=REPLICAS, n_its=300).problem
        _C3["v"] = (problem, oracle_lib.solve(problem, threads=8))
    return _C3["v"]


@pytest.mark.gpu
@pytest.mark.parametrize("cap", [None, "0,0,0,0"], ids=["uncapped", "cap0"])
def test_c3_shape_one_pod_of_an_app_per_claim(handle, monkeypatch, capfd, cap):
    problem, orc = c3_shape()
    monkeypatch.setenv("KP_DEBUG", "1")
    if cap is None:
        monkeypatch.delenv("KP_SMEM_CAP", raising=False)
    else:
        monkeypatch.setenv("KP_SMEM_CAP", cap)
    capfd.readouterr()
    res = handle.solve(problem)
    (plan,) = plans_of(capfd.readouterr().err)
    if cap is not None:
        assert plan["tk"] == 0 and plan["CQ"] == 0 and plan["CR"] == 0 and plan["CS"] == 0, plan
    assert_same(res, orc, f"C3 shape KP_SMEM_CAP={cap} ")
    c = claims_of(res)
    app = np.arange(len(c)) // REPLICAS
    on_claims = c >= 0
    assert on_claims.sum() > 0
    pairs = c[on_claims].astype(np.int64) * APPS + app[on_claims]
    assert len(np.unique(pairs)) == len(pairs), "two pods of one app on a NodeClaim"
