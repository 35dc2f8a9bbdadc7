"""Every lane- and word-indexed table of the solver at its full width, and the refusal one past it.

The solver is built around fixed widths (karpenter_b200/csrc/kp_tables.hpp, kp_api.cu): one warp lane per label key (32),
one 64-bit instance-type word per lane (2 048 types), one lane per resource (8), 64-bit masks over NodePools, the values of
a key, reservations and host ports, one lane per offering requirement set (32), and 32- / 64-bit words over the existing
nodes.  A mistake there shows only at the last lane or bit, so every problem here (tests/widths.py) reaches one width and
asserts it on the encoded kp_problem, and the CPU tier checks that removing the last element changes the oracle's answer.

CPU tier: widths, the "edge matters" checks, the cached CPU solver (which runs the library's own kp_prep) against the
oracle, and kp_prep's KP_ERR_CAPACITY refusals one past each width.  GPU tier: kp_solve, kp_solve_batch, kp_feasibility
and kp_consolidate against the oracle bit for bit, the shared-memory plan at 32 words and 32 keys, and every refusal
(including the 65 NodePools and 65 host ports kp_api.cu checks) from kp_solve and kp_consolidate on a handle that then
still solves correctly."""
import ctypes as C

import numpy as np
import pytest

from karpenter_b200 import _abi, _native
from karpenter_b200.disruption import Consolidation
from karpenter_b200.model import host_port_key
from tests import oracle_lib
from tests import widths as W
from tests.parity import assert_same
from tests.test_smem_plans import SMEM_OPTIN, plans_of

E_SIZES = [31, 32, 33, 63, 64, 65, 129]
TYPE_CASES = [(t, m) for t in (1985, 2047, 2048) for m in (600, 64, 63)]

_CACHE = {}


def problem(name):
    """(encoded problem, oracle result) of a named full-width problem, built and solved once per session"""
    if name not in _CACHE:
        kind, _, arg = name.partition(":")
        if kind == "types":
            t, m = map(int, arg.split("/"))
            enc = W.types_problem(t, m)
        elif kind == "types32keys":
            enc = W.types_problem(2048, 600, n_fill=26)
        elif kind == "keys":
            enc = W.keys_problem()
        elif kind == "values":
            enc = W.values_problem()
        elif kind == "resources":
            enc = W.resources_problem()
        elif kind == "pools":
            enc = W.pools_problem()[0]
        elif kind == "offerings":
            enc = W.offerings_problem()
        elif kind == "reservations":
            enc = W.reservations_problem(strict=arg == "strict")
        elif kind == "ports":
            enc = W.ports_problem()[0]
        elif kind == "nodes":
            enc = W.nodes_problem(int(arg))
        else:
            raise KeyError(name)
        _CACHE[name] = (enc, oracle_lib.solve(enc.problem, threads=8))
    return _CACHE[name]


NAMES = ([f"types:{t}/{m}" for t, m in TYPE_CASES] + ["types32keys", "keys", "values", "resources", "pools", "offerings",
         "reservations:strict", "reservations:fallback", "ports"] + [f"nodes:{e}" for e in E_SIZES])


def widths_of(enc):
    p = enc.problem
    return dict(K=p.n_keys, T=p.n_its, ITW=(p.n_its + 63) // 64, R=p.n_resources, N=p.n_templates, E=p.n_nodes,
                HP=p.n_hostports, RSV=p.n_reservations, D=W.offering_sets(p))


def differs(a, b):
    """the two oracle answers place some pod differently or open different NodeClaims"""
    if a["n_claims"] != b["n_claims"] or not np.array_equal(a["pod_target"], b["pod_target"]):
        return True
    for k in ("claim_template", "claim_npods", "claim_its", "claim_req_mask", "claim_reservations", "claim_dropped"):
        x, y = np.asarray(a[k]), np.asarray(b[k])
        if x.shape != y.shape or not np.array_equal(x, y):
            return True
    return False


# ---- CPU tier: each problem reaches its width, and the oracle answers it --------------------------------------------
def test_instance_types_at_width():
    for t, m in TYPE_CASES:
        enc, res = problem(f"types:{t}/{m}")
        w = widths_of(enc)
        assert w["T"] == t and w["ITW"] == 32, w
        assert enc.problem.get("max_instance_types") == m
        # the word-31 pods land on claims of word-31 types only
        app = np.array([0] * 60 + [1] * 20 + [2] * 12 + [3] * 8 + [4] * 10)
        tgt = res["pod_target"]
        assert (tgt != -1).all() or m == 63, (t, m)
        for c in set((-2 - tgt[(app == 2) & (tgt <= -2)]).tolist()):
            its = res["claim_its"][c]
            assert its[:31].sum() == 0 and its[31] != 0, (t, m, c)
        # truncation keeps at most m types; the claim of the NodePool with minValues 64 on the instance-type key is dropped
        # exactly when those carry fewer than 64 distinct names.  (The catalog lists most names twice, linux and windows
        # at one price, so 64 or 63 kept types carry 32 names: dropped at 64 and 63, kept at 600.)  No other claim drops.
        mv = enc.tmpl_names.index("mv")
        dropped = res["claim_dropped"].astype(bool)
        assert (res["claim_template"][dropped] == mv).all(), (t, m)
        for c in np.flatnonzero(res["claim_template"] == mv):
            its = enc.decode_its(res, c)
            assert len(its) <= m and dropped[c] == (len(set(its)) < 64), (t, m, len(its), len(set(its)))
        assert dropped.any() == (m != 600), (t, m)
    enc, _ = problem("types32keys")
    assert widths_of(enc)["K"] == 32 and widths_of(enc)["T"] == 2048


def test_keys_at_width():
    enc, res = problem("keys")
    assert widths_of(enc)["K"] == 32
    assert [enc.key_id(k) for k in W.EDGE_KEYS] == [29, 30, 31], enc.keys
    p = enc.problem
    assert int(p.get("tsc_key")[0]) == 31  # the spread sits on the highest-numbered key
    assert (res["pod_target"] != -1).all()
    # Gt 3 / Lt 3 on the integer key e1 (key 30) pin the claims' values
    gt = [enc.decode_requirements(res, -2 - t)[W.EDGE_KEYS[1]]["values"] for t in res["pod_target"][100:110]]
    assert all(set(v) <= {"4", "8", "16"} and v for v in gt), gt


def test_values_at_width():
    enc, res = problem("values")
    k = enc.key_id(W.RACK)
    off = enc.problem.get("key_value_off")
    assert off[k + 1] - off[k] == 64 and enc.values[W.RACK][63] == "r63"
    tgt = res["pod_target"]
    in63 = tgt[:30]
    assert (in63 != -1).all()
    for t in in63:  # on a node carrying r63 or a claim pinned to it
        if t <= -2:
            assert enc.decode_requirements(res, -2 - t)[W.RACK]["values"] == ["r63"]
    assert (in63 >= 0).any() and (in63 <= -2).any()
    for t in tgt[30:50]:
        if t <= -2:
            assert "r63" not in enc.decode_requirements(res, -2 - t)[W.RACK]["values"]
        else:
            assert t == -1 or t >= 0 and enc.node_rows[t]["labels"][W.RACK] != "r63"


def test_resources_at_width():
    enc, res = problem("resources")
    assert enc.resources == W.RESOURCES and widths_of(enc)["R"] == 8
    assert enc.problem.get("res_flags")[5] & 4 and enc.problem.get("res_flags")[6] & 4  # hugepages
    tgt = res["pod_target"]
    fpga = [-2 - t for t in tgt[30:42]]
    assert all(t <= -2 for t in tgt[30:42])
    assert all(res["claim_requests"][c][7] >= 1 for c in fpga)


def test_nodepools_at_width():
    enc, res = problem("pools")
    assert widths_of(enc)["N"] == 64
    _, names = W.pools_problem()
    assert enc.tmpl_names == names  # template i is np-(99 - i)
    w = enc.problem.get("tmpl_limit_present")
    assert w[63] and not w[:63].any()
    tgt = res["pod_target"]
    tmpl = lambda s: {int(res["claim_template"][-2 - t]) for t in tgt[s] if t <= -2}
    # (the pods that tolerate every pool join the claims the others opened)
    assert tmpl(slice(10, 18)) == {31} and tmpl(slice(18, 26)) == {32} and (tgt[:26] <= -2).all()
    assert tmpl(slice(26, 38)) == {63} and (tgt[26:38] == -1).any()  # the limit on pool 63 binds
    assert tmpl(slice(38, 44)) <= {31, 63}


def test_offering_sets_at_width():
    enc, res = problem("offerings")
    assert widths_of(enc)["D"] == 32
    tgt = res["pod_target"]
    assert (tgt[20:35] <= -2).all()
    for t in tgt[20:35]:
        r = enc.decode_requirements(res, -2 - t)
        assert r["topology.kubernetes.io/zone"]["values"] == ["wz-15"]


@pytest.mark.parametrize("mode", ["strict", "fallback"])
def test_reservations_at_width(mode):
    enc, res = problem(f"reservations:{mode}")
    assert widths_of(enc)["RSV"] == 64
    rid = enc.problem.get("off_reservation_id")[enc.problem.get("off_reserved") != 0]
    assert 63 in rid.tolist()
    held = np.bitwise_or.reduce(res["claim_reservations"].astype(np.uint64)) if res["n_claims"] else np.uint64(0)
    assert int(held) >> 63 & 1, hex(int(held))


def test_host_ports_at_width():
    enc, b = W.ports_problem()
    assert widths_of(enc)["HP"] == 64 and b.hostports[host_port_key(W.PORTS[63])] == 63
    conf = enc.problem.get("hostport_conflicts")
    assert int(conf[63]) == 1 << 63
    assert int(enc.problem.get("node_hostports")[1]) == 1 << 63
    _, res = problem("ports")
    tgt = res["pod_target"]
    assert (tgt != -1).all() and not (tgt[:6] == 1).any()  # no port-63 pod on node-1


@pytest.mark.parametrize("E", E_SIZES)
def test_existing_nodes_at_width(E):
    enc, res = problem(f"nodes:{E}")
    assert widths_of(enc)["E"] == E
    assert enc.node_names[:E] == [f"node-{i:03d}" for i in range(E)]
    named = W.named_nodes(E)
    tgt = res["pod_target"]
    n_in = len(named) + 2
    # one pod of the In rule on each named node (about one fits), the two left over stay pending
    assert sorted(tgt[:n_in].tolist()) == [-1, -1] + named, tgt[:n_in]
    assert not set(tgt[n_in:n_in + 20].tolist()) & set(named)
    anti = tgt[n_in + 20:n_in + 20 + min(E, 40)]
    assert not (anti >= 64).any() and not (anti == E - 1).any()


# ---- CPU tier: removing the edge element changes the answer ----------------------------------------------------------
EDGES = {
    "types": lambda e: W.types_problem(2048, 600, edge=e),
    "keys": lambda e: W.keys_problem(edge=e),
    "values": lambda e: W.values_problem(edge=e),
    "resources": lambda e: W.resources_problem(edge=e),
    "pools": lambda e: W.pools_problem(edge=e)[0],
    "offerings": lambda e: W.offerings_problem(edge=e),
    "reservations": lambda e: W.reservations_problem(edge=e),
    "ports": lambda e: W.ports_problem(edge=e)[0],
    **{f"nodes{E}": (lambda E: lambda e: W.nodes_problem(E, edge=e))(E) for E in E_SIZES},
}


@pytest.mark.parametrize("dim", list(EDGES))
def test_edge_matters(dim):
    full, cut = EDGES[dim](True), EDGES[dim](False)
    assert differs(oracle_lib.solve(full.problem, threads=8), oracle_lib.solve(cut.problem, threads=8)), dim


# ---- CPU tier: the cached solver (the library's kp_prep) equals the oracle where it serves ---------------------------
PLAIN = {
    "types2048": lambda: W.types_problem(2048, 0, min_values=False),
    "types2048_32keys": lambda: W.types_problem(2048, 0, min_values=False, n_fill=26),
    "types1985": lambda: W.types_problem(1985, 0, min_values=False),
    "keys": lambda: W.keys_problem(bounds=False),
    "values": W.values_problem,
    "resources": W.resources_problem,
    "pools": lambda: W.pools_problem(limits=False)[0],
    "offerings": W.offerings_problem,
}


@pytest.mark.parametrize("name", list(PLAIN))
def test_cached_solver_at_width(name):
    enc = PLAIN[name]()
    if name == "types2048_32keys":
        assert enc.problem.n_keys == 32
    orc = oracle_lib.solve(enc.problem, threads=8)
    got = oracle_lib.cached_solve(enc.problem)
    assert got is not None, f"{name}: outside what the cached solver serves"
    for k in oracle_lib.CACHED_KEYS:
        assert np.array_equal(np.asarray(got[0][k]), np.asarray(orc[k])), (name, k)


# ---- refusals one past each width -------------------------------------------------------------------------------------
def _patch_ports(enc, n):
    """n host ports in the encoded arrays (the encoder itself refuses more than 64): entries 64 .. n-1 conflict only with
    themselves and nobody uses them"""
    p = enc.problem
    conf = np.zeros(n, np.uint64)  # (an entry past 64 has no bit of its own in a 64-bit mask: it conflicts with nothing)
    conf[:64] = p.get("hostport_conflicts")
    p.set("hostport_conflicts", conf)
    p.set("n_hostports", n)
    return enc


def _patch_pools(enc, n):
    """n NodePool templates in the encoded arrays, the ones past 64 copies of the last (65 pools through the encoder would
    give the karpenter.sh/nodepool key 65 values, which is refused first)"""
    p = enc.problem
    N = p.n_templates
    rows = list(range(N)) + [N - 1] * (n - N)
    off = p.get("tmpl_it_off")
    its = p.get("tmpl_its")
    p.set("tmpl_reqset", p.get("tmpl_reqset")[rows])
    p.set("tmpl_taintset", p.get("tmpl_taintset")[rows])
    p.set("tmpl_its", np.concatenate([its[off[r]:off[r + 1]] for r in rows]).astype(np.int32))
    p.set("tmpl_it_off", np.concatenate([[0], np.cumsum([off[r + 1] - off[r] for r in rows])]).astype(np.int32))
    for k in ("tmpl_daemon", "tmpl_limits", "tmpl_limit_present"):
        p.set(k, p.get(k)[rows])
    p.set("n_templates", n)
    return enc


# (width, one past) generators and the message of the refusal
REFUSALS = {
    "keys": (lambda: W.keys_problem(bounds=False), lambda: W.keys_problem(bounds=False, n_fill=25), "more than 32 active label keys"),
    "types": (lambda: W.types_problem(2048, min_values=False), lambda: W.types_problem(2049, min_values=False),
              "more than 2048 instance types"),
    "values": (W.values_problem, lambda: W.values_problem(n_values=65), "more than 64 distinct values"),
    "resources": (W.resources_problem, lambda: W.resources_problem(extra=True), "resource count out of range"),
    "offerings": (W.offerings_problem, lambda: W.offerings_problem(33), "more than 32 distinct offering requirement sets"),
    "reservations": (W.reservations_problem, lambda: W.reservations_problem(n_reservations=65), "more than 64 capacity reservations"),
}
API_REFUSALS = {  # checked by kp_api.cu, not by kp_prep
    "nodepools": (lambda: W.pools_problem(limits=False)[0], lambda: _patch_pools(W.pools_problem(limits=False)[0], 65),
                  "more than 64 NodePools"),
    "host_ports": (lambda: W.ports_problem()[0], lambda: _patch_ports(W.ports_problem()[0], 65), "more than 64 distinct host ports"),
}


def cached_rc(problem):
    r = _abi.kp_result()
    prep = C.c_double()
    lib = oracle_lib.cached_lib()
    rc = lib.orc_cached_solve(problem.ref(), C.byref(r), C.byref(prep))
    if rc == 0:
        lib.orc_cached_free(C.byref(r))
    return rc


@pytest.mark.parametrize("dim", list(REFUSALS))
def test_prep_refuses_one_past_width(dim):
    at, past, _ = REFUSALS[dim]
    w = at()
    rc = cached_rc(w.problem)
    # reservations are outside what the cached solver serves (KP_ERR_UNSUPPORTED): what matters is that kp_prep passed them
    assert rc == (5 if dim == "reservations" else 0), (dim, rc)
    assert cached_rc(past().problem) == 4, dim


def test_oracle_has_no_such_limits():
    """the library's refusal is what stands between these problems and a wrong answer: the oracle solves them"""
    for dim in ("types", "keys", "offerings"):
        res = oracle_lib.solve(REFUSALS[dim][1]().problem, threads=8)
        assert res["n_claims"] > 0, dim


# ---- GPU tier ---------------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def handle():
    h = _native.Handle()
    yield h
    h.close()


@pytest.mark.gpu
@pytest.mark.parametrize("name", NAMES)
def test_solve_at_width(handle, name):
    enc, orc = problem(name)
    assert_same(handle.solve(enc.problem), orc, f"{name} ")


@pytest.mark.gpu
def test_plan_at_32_words_and_32_keys(handle, monkeypatch, capfd):
    enc, orc = problem("types32keys")
    assert enc.problem.n_keys == 32 and (enc.problem.n_its + 63) // 64 == 32
    for k in ("KP_SMEM_CAP", "KP_NO_DOMAIN_FP", "KP_NO_LEAN", "KP_COHORT", "KP_NO_COHORT"):
        monkeypatch.delenv(k, raising=False)
    monkeypatch.setenv("KP_DEBUG", "1")
    capfd.readouterr()
    res = handle.solve(enc.problem)
    plans = plans_of(capfd.readouterr().err)
    assert len(plans) == 1 and plans[0]["smem"] <= SMEM_OPTIN, plans
    assert_same(res, orc, "types32keys with KP_DEBUG ")


@pytest.mark.gpu
def test_batch_full_width_beside_narrow(handle):
    wide, wide_orc = problem("types32keys")
    narrow, narrow_orc = problem("offerings")
    assert narrow.problem.n_its <= 64 and narrow.problem.n_keys < 8
    solo = [handle.solve(wide.problem), handle.solve(narrow.problem)]
    for order in ((0, 1), (1, 0)):
        probs = [(wide, wide_orc), (narrow, narrow_orc)]
        outs = handle.solve_batch([probs[i][0].problem for i in order])
        for i, o in zip(order, outs):
            assert_same(o, probs[i][1], f"batch {order} instance {i} ")
            assert_same(o, solo[i], f"batch {order} instance {i} vs solo ")


@pytest.mark.gpu
def test_feasibility_at_width(handle):
    # with the Strict minValues NodePool: classes whose requirements leave it fewer than 64 types get no types from it
    enc, _ = problem("types32keys")
    assert enc.problem.n_keys == 32 and enc.tmpl_names[1] == "mv"
    got = handle.feasibility(enc.problem)
    assert got.shape[2] == 32
    assert np.array_equal(got, oracle_lib.feasibility(enc.problem))
    assert got[:, :, 31].any()
    on_default, on_mv = got[:, 0].any(axis=1), got[:, 1].any(axis=1)
    assert on_mv.any() and (on_default & ~on_mv).any(), (on_default, on_mv)  # minValues removes some classes' types


CONSOL_CASES = [(E, 2048, 64) for E in (63, 64, 65, 129)]


def cut_in_tie(enc, kept):
    """a type the 600-type cut left out ties in price with the last type kept and has at least its capacity, so it was a
    cheaper option as well: the cut fell inside a price tie"""
    p = enc.problem
    off, price, cap = p.get("it_off_off"), p.get("off_price"), p.get("it_capacity")
    cheapest = np.array([price[off[t]:off[t + 1]].min() for t in range(p.n_its)])
    last = kept[-1]
    out = np.setdiff1d(np.arange(p.n_its), kept)
    return bool(((cheapest[out] == cheapest[last]) & (cap[out] >= cap[last]).all(axis=1)).any())


@pytest.mark.parametrize("E", [63, 129])
def test_consolidation_case_replaces_at_the_cut(E):
    """the removal of an edge node is a replacement whose options are cut at 600 types (SimulateScheduling's
    MaxInstanceTypes) inside a price tie; the pinned pods make some sets a no-op, and node 6's pod moves to node E - 1"""
    pools, per_pool, nodes, sets = W.consolidation_case(E)
    eng = Consolidation(pools, per_pool, nodes, backend=oracle_lib.consolidate, price_order=True)
    cmds = eng.compute(sets)
    enc, _ = eng._encode(sets)
    dec = dict(zip(map(tuple, sets), (c.decision for c in cmds)))
    assert dec[("node-006",)] == "delete" and dec[("node-005", "node-031")] == "noop"
    assert E <= 63 or dec[("node-063",)] == "noop"  # one pod of node 63 is pinned to it
    edge = [s for s in sets if s[-1] in (f"node-{E - 1:03d}", "node-031", "node-032") and "node-005" not in s]
    off, order = eng.raw["repl_order_off"], eng.raw["repl_order"]
    for s in edge:
        k = sets.index(s)
        assert cmds[k].decision == "replace", (s, cmds[k].decision)
        kept = order[off[k]:off[k + 1]]
        assert len(kept) == 600 and cut_in_tie(enc, kept), (s, len(kept))


@pytest.mark.gpu
@pytest.mark.parametrize("E,n_types,n_pools", CONSOL_CASES, ids=[f"E{e}" for e, _, _ in CONSOL_CASES])
def test_consolidate_at_width(E, n_types, n_pools):
    pools, per_pool, nodes, sets = W.consolidation_case(E, n_types, n_pools)
    orc = Consolidation(pools, per_pool, nodes, backend=oracle_lib.consolidate, price_order=True)
    cmds = orc.compute(sets)
    gpu = Consolidation(pools, per_pool, nodes, price_order=True)
    try:
        gpu.compute(sets)
    finally:
        gpu.close()
    for k in _abi.CONSOL_PARITY_KEYS + ["repl_order_off", "repl_order"]:
        assert np.array_equal(gpu.raw[k], orc.raw[k]), (E, k)
    decisions = [c.decision for c in cmds]
    assert {"replace", "delete", "noop"} <= set(decisions), decisions
    assert (np.diff(orc.raw["repl_order_off"]) == 600).sum() == decisions.count("replace")  # every replacement is cut at 600


def _consol_input(problem):
    """a kp_consol_input that treats every pod of `problem` as a pending extra pod and asks about no candidate set"""
    E = problem.n_nodes
    return _abi.ConsolInput(node_pod_off=np.zeros(E + 1, np.int32), node_it=np.full(max(E, 1), -1, np.int32),
                            node_is_spot=np.zeros(max(E, 1), np.uint8), n_subsets=0, subset_off=np.zeros(1, np.int32),
                            subset_nodes=np.zeros(1, np.int32), spot_to_spot_enabled=0, capacity_type_key=-1, ct_reserved=-1,
                            ct_spot=-1, ct_on_demand=-1, filter_same_instance_type=0, n_extra_pods=problem.n_pods,
                            extra_pod_kind=np.full(problem.n_pods, _abi.KP_EXTRA_PENDING, np.uint8), export_price_order=0)


@pytest.mark.gpu
@pytest.mark.parametrize("dim", list(REFUSALS) + list(API_REFUSALS))
def test_every_refusal(handle, dim):
    at, past, msg = {**REFUSALS, **API_REFUSALS}[dim]
    small, small_orc = problem("offerings")
    bad = past().problem
    with pytest.raises(_native.SolverError) as e:
        handle.solve(bad)
    assert e.value.code == 4 and msg in str(e.value), str(e.value)
    assert_same(handle.solve(small.problem), small_orc, f"after the {dim} refusal ")
    with pytest.raises(_native.SolverError) as e:
        handle.consolidate(bad, _consol_input(bad))
    assert e.value.code == 4 and msg in str(e.value), str(e.value)
    assert_same(handle.solve(small.problem), small_orc, f"after the {dim} refusal in kp_consolidate ")
    w = at().problem  # and at the width itself the library does not refuse
    handle.solve(w)
