// TEST / BENCH INFRASTRUCTURE -- never linked into, imported by or executed from the product path.
//
// orc_cached.cpp: the CUDA solver's ALGORITHM on one host core, for bench.py's cpu_baseline legs.  The oracle
// (orc_solver.cpp) restates the reference: every pod re-evaluates every NodeClaim in front of its target.  libkarpsolve.so
// removes what that recomputes -- monotone failure bits per (claim, requirement signature / request vector), the
// "adds nothing" fast path, threshold bitmaps instead of the per-type loop, scan lower bounds, the incremental form of Go's
// sort.Slice -- and then walks the remaining chain with one warp.  This file walks the SAME chain with the SAME caches, over
// the SAME prepared tables and class plan (kp_prep.cpp: the host half of libkarpsolve.so), as plain scalar C++: the ratio oracle : this
// is the algorithm's share of a speed-up, the ratio this : GPU the hardware's.
//
// Scope: Scheduler.Solve with existing nodes, in-flight and new NodeClaims -- requirement algebra without Gt / Lt bounds,
// taints, topology groups (spread, affinity, anti-affinity, node filters and policies, the domain fast path) -- and
// kp_consolidate's fast path (topology-free candidate pods: simulation on a private view of the nodes + computeConsolidation
// with the price lists).  Not served: minValues, reservations, host ports, volume alternatives, NodePool limits, the
// preference ladder, consolidation with topology or extra pods: KP_ERR_UNSUPPORTED.  Results are checked against the oracle
// (tests/test_cached_cpu_baseline.py) and, inside bench.py, against the GPU's; each step cites the device code it mirrors.
#include <chrono>
#include <cstdlib>
#include <cstring>
#include <numeric>
#include <string>
#include <vector>

#include "../karpenter_b200/csrc/kp_gosort_host.hpp"
#include "../karpenter_b200/csrc/kp_prep.hpp"

namespace {

struct Claim {
  std::vector<Slot> s;        // requirement slot per key
  std::vector<int64_t> q;     // Spec.Resources.Requests
  std::vector<int> j;         // threshold row per resource (fits_word)
  std::vector<uint64_t> its;  // InstanceTypeOptions
  int tmpl = 0;
  int dom = 0xff;  // the topology-key value the claim is pinned to (c_dom), 0xff: none
};

struct Solver {
  const kp_problem* p;
  HostTables t;
  const ClassPlan& pl = t.plan;  // signatures and shortcuts per class (kp_prep.cpp plan_classes)
  int K, R, ITW, N, X;
  std::vector<uint64_t> tmpl_its;
  std::vector<Claim> claims;
  std::vector<int32_t> ord;  // claim order (sort.Slice(newNodeClaims, len(Pods)))
  std::vector<int> cnt;      // pods per claim id
  std::vector<std::vector<uint64_t>> failm, deadm, accm;  // per claim: bits over fsig / rv / asig ids
  std::vector<int> lbf, lbr;                              // scan lower bounds per fsig / rv
  long long slow_sorts = 0, fast_commits = 0;
  // topology (kp_kernels.cuh): counters per group and domain, hostname groups counted per NodeClaim
  int GH = 0;
  std::vector<int32_t> dom_cnt, g_ndomains, g_nempty;
  std::vector<uint64_t> dom_reg, dom_pop;
  std::vector<int32_t> host_cnt;            // [host * GH + row]; host = node index, or E + NodeClaim id
  // existing nodes (ExistingNode, existingnode.go:40-66): remaining resources, label slots; candidate bitmaps per class
  // signature (k_node_cand): nstat[nsig] = taints tolerated and labels compatible, nfit[rv] = the request vector fits
  int E = 0;
  std::vector<int64_t> node_rem;
  std::vector<uint32_t> node_rem_present;
  std::vector<Slot> node_slot;
  std::vector<int32_t> node_npods;
  std::vector<std::vector<uint64_t>> nstat, nfit;       // bit per node
  std::vector<uint64_t> nactive;

  KeyInfo ki(int k) const { return KeyInfo{t.val_int.data() + (size_t)k * 64, t.val_isint[k], t.key_univ[k]}; }
  Slot rs_slot(int rs, int k) const {
    const size_t i = (size_t)rs * K + k;
    return Slot{t.rs_flags[i], t.rs_mask[i], 0, 0};
  }
  static bool bit(const std::vector<uint64_t>& m, int i) { return (m[i >> 6] >> (i & 63)) & 1ull; }
  static void set(std::vector<uint64_t>& m, int i) { m[i >> 6] |= 1ull << (i & 63); }

  // kp_kernels.cuh fits_word: advance the threshold rows for the total requests q, AND the rows that advanced
  bool fits(const std::vector<int64_t>& q, std::vector<int>& j, std::vector<uint64_t>& its) const {
    bool fresh_any = false;
    for (int r = 0; r < R; r++) {
      const int end = t.ge_off[r + 1];
      int lo = j[r];
      const bool fresh = lo < t.ge_off[r];
      if (fresh) lo = t.ge_off[r];
      const int start = lo;
      while (lo < end && t.ge_vals[lo] < q[r]) lo++;
      j[r] = lo;
      if (fresh) fresh_any = true;
      if (fresh || lo != start) {
        if (lo == end) {
          std::fill(its.begin(), its.end(), 0ull);
        } else {
          for (int w = 0; w < ITW; w++) its[w] &= t.ge_bits[(size_t)lo * ITW + w];
        }
      }
    }
    if (fresh_any)
      for (int w = 0; w < ITW; w++) its[w] &= t.it_valid[w];
    for (int w = 0; w < ITW; w++)
      if (its[w]) return true;
    return false;
  }
  // kp_kernels.cuh compat_off_word: compatible(it, S) & hasOffering(it, S)
  void compat_off(const std::vector<Slot>& S, std::vector<uint64_t>& out) const {
    std::vector<uint64_t> ow(ITW, 0ull);
    for (int dd = 0; dd < t.D; dd++) {
      bool ok = true;
      for (uint32_t keys = t.off_keys[dd]; keys && ok; keys &= keys - 1) {
        const int k = __builtin_ctz(keys);
        ok = slot_compatible(ki(k), S[k], t.off_slots[(size_t)dd * K + k], t.key_wellknown[k], true);
      }
      if (ok)
        for (int w = 0; w < ITW; w++) ow[w] |= t.offset_bits[(size_t)dd * ITW + w];
    }
    for (int w = 0; w < ITW; w++) {
      uint64_t cw = ~0ull;
      for (int k = 0; k < K; k++) {
        const Slot& s = S[k];
        if (!slot_present(s)) continue;
        const KeyInfo kk = ki(k);
        uint64_t allowed = slot_allowed(kk, s);
        uint64_t bw = t.it_nokey[(size_t)k * ITW + w];
        if (allowed == kk.univ) {
          bw |= t.it_nonempty[(size_t)k * ITW + w];
        } else {
          for (; allowed; allowed &= allowed - 1) bw |= t.itv[((size_t)t.itv_off[k] + __builtin_ctzll(allowed)) * ITW + w];
        }
        if (op_is_negative(slot_op(s))) bw |= t.it_dne[(size_t)k * ITW + w];
        cw &= bw;
      }
      out[w] &= cw & ow[w];
    }
  }

  bool tolerated(int tolset, int taintset) const {
    if (taintset < 0 || t.n_taintsets == 0) return true;
    return t.tol_ok[(size_t)(tolset + 1) * t.n_taintsets + taintset];
  }
  // kp_kernels.cuh topo_domains: TopologyGroup.Get for a non-hostname key (topologygroup.go:226-428)
  Slot topo_domains(int g, const KpGroup& G, bool self, const Slot& pod_d, const Slot& node_d) const {
    const KeyInfo kk = ki(G.key);
    const int32_t* cnt = dom_cnt.data() + G.dom_off;
    const uint64_t reg = dom_reg[g], pop = dom_pop[g];
    const uint64_t pod_allowed = slot_allowed(kk, pod_d), node_allowed = slot_allowed(kk, node_d);
    const bool node_in = slot_present(node_d) && slot_op(node_d) == OP_IN;
    Slot out{SF_PRESENT, 0ull, 0, 0};
    if (G.type == KP_TOPO_SPREAD) {
      const uint64_t sup = reg & pod_allowed;
      long long mn = 2147483647LL;
      for (uint64_t m = sup; m; m &= m - 1) mn = std::min<long long>(mn, cnt[__builtin_ctzll(m)]);
      if (G.min_domains >= 0 && __builtin_popcountll(sup) < G.min_domains) mn = 0;
      long long best_c = 2147483647LL;
      int best = -1;
      for (uint64_t cand = node_in ? (node_d.m & reg) : (reg & node_allowed); cand; cand &= cand - 1) {
        const int v = __builtin_ctzll(cand);
        const long long c = (long long)cnt[v] + (self ? 1 : 0);
        if (c - mn <= (long long)G.max_skew && c < best_c) {
          best = v;
          best_c = c;
        }
      }
      if (best >= 0) out.m = 1ull << best;
      return out;
    }
    if (G.type == KP_TOPO_AFFINITY) {
      const uint64_t opts = node_in ? (node_d.m & pod_allowed & reg & pop) : (reg & pod_allowed & pop & node_allowed);
      if (opts) {
        out.m = opts;
        return out;
      }
      const bool none_populated = (reg & pop) == 0, any_compat = (reg & pop & pod_allowed) != 0;
      if (self && (none_populated || !any_compat)) {
        const Slot pd = slot_present(pod_d) ? pod_d : slot_exists(), nd = slot_present(node_d) ? node_d : slot_exists();
        const uint64_t a = reg & slot_allowed(kk, slot_intersection(kk, pd, nd));
        if (a) out.m |= a & (~a + 1);
        const uint64_t b = reg & pod_allowed;
        if (b) out.m |= b & (~b + 1);
      }
      return out;
    }
    out.m = reg & ~pop & node_allowed & pod_allowed;
    return out;
  }
  // kp_kernels.cuh domain_mask: the verdict of the class's topology-key groups for every claim pinned to one value
  uint64_t domain_mask(int cls, bool* exact) const {
    uint64_t ez = ~0ull;
    *exact = true;
    const Slot strict = rs_slot(t.cls_strict_rs[cls], pl.tk_key);
    const uint64_t univ = t.key_univ[pl.tk_key];
    const uint64_t pod_allowed = (strict.f & SF_PRESENT) ? (((strict.f & SF_COMPLEMENT) ? ~strict.m : strict.m) & univ) : univ;
    for (int i = t.cls_match_off[cls]; i < t.cls_match_off[cls + 1]; i++) {
      const int e = t.cls_match[i], g = e & 0x3fffffff;
      const KpGroup& G = t.groups[g];
      if (G.key != pl.tk_key) continue;
      const bool self = (e >> 30) & 1;
      const uint64_t reg = dom_reg[g], pop = dom_pop[g];
      if (G.type == KP_TOPO_SPREAD) {
        const int32_t* cnt = dom_cnt.data() + G.dom_off;
        const uint64_t sup = reg & pod_allowed;
        long long mn = 2147483647LL;
        for (uint64_t m = sup; m; m &= m - 1) mn = std::min<long long>(mn, cnt[__builtin_ctzll(m)]);
        if (G.min_domains >= 0 && __builtin_popcountll(sup) < G.min_domains) mn = 0;
        uint64_t okm = 0;
        for (uint64_t m = reg; m; m &= m - 1) {
          const int v = __builtin_ctzll(m);
          if ((long long)cnt[v] + (self ? 1 : 0) - mn <= (long long)G.max_skew) okm |= 1ull << v;
        }
        ez &= okm;
      } else if (G.type == KP_TOPO_ANTI_AFFINITY) {
        ez &= reg & ~pop & pod_allowed;
      } else {
        const bool none_populated = (reg & pop) == 0, any_compat = (reg & pop & pod_allowed) != 0;
        if (self && (none_populated || !any_compat))
          *exact = false;
        else
          ez &= reg & pop & pod_allowed;
      }
    }
    return ez;
  }
  void host_record(int row, int g, int host) {
    int32_t& c = host_cnt[(size_t)host * GH + row];
    if (c == 0) g_nempty[g]--;
    c++;
  }
  // kp_kernels.cuh topo_record: Topology.Record (topology.go:197-220) of a placement with final requirements F
  void topo_record(int cls, const std::vector<Slot>& F, int taintset, int host) {
    for (int i = t.cls_rec_off[cls]; i < t.cls_rec_off[cls + 1]; i++) {
      const int g = t.cls_rec[i];
      const KpGroup& G = t.groups[g];
      bool counts = true;
      if (!G.inverse) {
        if (G.affinity_policy == 1 && G.filter_n > 0) {
          bool any_alt = false;
          for (int a = 0; a < G.filter_n && !any_alt; a++) {
            const int rs = t.filter_rs[G.filter_off + a];
            bool bad = false;
            for (int k = 0; k < K && !bad; k++) bad = !slot_compatible(ki(k), F[k], rs_slot(rs, k), t.key_wellknown[k], false);
            any_alt = !bad;
          }
          counts = any_alt;
        }
        if (counts && G.taint_policy == 1) counts = tolerated(G.tolset, taintset);
      }
      if (!counts) continue;
      if (G.key == t.hostname_key) {
        host_record(G.host_row, g, host);
      } else if (F[G.key].f & SF_PRESENT) {
        uint64_t rec = 0;
        if (G.inverse || G.type == KP_TOPO_ANTI_AFFINITY)
          rec = F[G.key].m;
        else if (!(F[G.key].f & SF_COMPLEMENT) && __builtin_popcountll(F[G.key].m) == 1)
          rec = F[G.key].m;
        for (uint64_t b = rec; b; b &= b - 1) dom_cnt[G.dom_off + __builtin_ctzll(b)]++;
        dom_reg[g] |= rec;
        dom_pop[g] |= rec;
      }
    }
  }
  // kp_kernels.cuh topo_record_fast: the claim's requirements are unchanged and its topology-key slot is In{z}
  void topo_record_fast(int cls, int z, int taintset, int host) {
    for (int i = t.cls_rec_off[cls]; i < t.cls_rec_off[cls + 1]; i++) {
      const int g = t.cls_rec[i];
      const KpGroup& G = t.groups[g];
      if (!G.inverse && G.taint_policy == 1 && !tolerated(G.tolset, taintset)) continue;
      if (G.key == t.hostname_key) {
        host_record(G.host_row, g, host);
      } else if (z >= 0) {
        dom_cnt[G.dom_off + z]++;
        dom_reg[g] |= 1ull << z;
        dom_pop[g] |= 1ull << z;
      }
    }
  }
  static int pinned(const Slot& s) {
    return (s.f == SF_PRESENT && __builtin_popcountll(s.m) == 1) ? __builtin_ctzll(s.m) : 0xff;
  }

  // kp_kernels.cuh eval_candidate, is_claim: NodeClaim.CanAdd (nodeclaim.go:114-202)
  struct Eval {
    bool ok = false, res_dead = false, changed = false, compat_fail = false, pod_noop = false;
    std::vector<Slot> F;
    std::vector<int64_t> q;
    std::vector<int> j;
    std::vector<uint64_t> its;
  };
  // is_claim = false: ExistingNode.CanAdd after the taint / Fits checks (existingnode.go:70-143): no undefined-key allowance,
  // no instance types
  void eval(int cls, int host, const std::vector<Slot>& base, const std::vector<int64_t>& bq, const std::vector<uint64_t>& bits,
            const std::vector<int>& bj, Eval& ev, bool is_claim = true) const {
    ev = Eval();
    evals_++;
    const int rs = t.cls_rs[cls];
    ev.F.resize(K);
    for (int k = 0; k < K; k++) {
      const Slot pod = rs_slot(rs, k);
      if (!slot_compatible_nb(base[k], pod, t.key_wellknown[k], is_claim)) {
        ev.compat_fail = true;
        return;
      }
      ev.F[k] = slot_add_nb(base[k], pod);
      if (!slot_eq(ev.F[k], base[k])) ev.changed = true;
    }
    ev.pod_noop = !ev.changed;
    // Topology.AddRequirements (topology.go:226-248), eval_candidate's topology branch
    const int moff = t.cls_match_off[cls], mend = t.cls_match_off[cls + 1];
    if (mend > moff) {
      std::vector<Slot>& M = ev.F;
      std::vector<Slot> Tt = M;
      for (int i = moff; i < mend; i++) {
        const int e = t.cls_match[i], g = e & 0x3fffffff;
        const bool self = (e >> 30) & 1;
        const KpGroup& G = t.groups[g];
        if (G.key == t.hostname_key) {  // a NodeClaim is exactly one hostname domain
          const int c = (size_t)(host + 1) * GH <= host_cnt.size() ? host_cnt[(size_t)host * GH + G.host_row] : 0;
          bool ok;
          if (G.type == KP_TOPO_SPREAD)
            ok = c + (self ? 1 : 0) <= G.max_skew;
          else if (G.type == KP_TOPO_AFFINITY)
            ok = c > 0 || (self && (g_ndomains[g] - g_nempty[g]) == 0);
          else
            ok = c == 0;
          if (!ok) return;
        } else {
          const Slot dm = topo_domains(g, G, self, rs_slot(t.cls_strict_rs[cls], G.key), M[G.key]);
          if (dm.m == 0) return;  // topologyError: no eligible domain
          Tt[G.key] = slot_add(ki(G.key), Tt[G.key], dm);
        }
      }
      for (int k = 0; k < K; k++)
        if (!slot_compatible(ki(k), M[k], Tt[k], t.key_wellknown[k], is_claim)) return;
      ev.changed = false;
      for (int k = 0; k < K; k++) {
        M[k] = slot_add(ki(k), M[k], Tt[k]);
        if (!slot_eq(M[k], base[k])) ev.changed = true;
      }
    }
    if (!is_claim) {
      ev.ok = true;
      return;
    }
    ev.q = bq;
    for (int r = 0; r < R; r++) ev.q[r] += t.cls_req[(size_t)cls * R + r];
    ev.j = bj;
    ev.its = bits;
    const bool any_fit = fits(ev.q, ev.j, ev.its);
    ev.res_dead = !any_fit;
    if (ev.changed) compat_off(ev.F, ev.its);
    ev.ok = false;
    for (int w = 0; w < ITW; w++)
      if (ev.its[w]) ev.ok = true;
  }
  mutable long long evals_ = 0;

  int prepare(std::string& err) {
    std::vector<uint8_t> active(p->n_nodes, 0);
    for (int i = 0; i < p->n_nodes; i++) active[i] = (p->node_flags[i] & KP_NODE_SCHEDULABLE) != 0;
    std::vector<int32_t> pending(p->pod_class, p->pod_class + p->n_pods);
    int rc = kp_prepare(p, active, {}, pending, t, err);
    if (rc != KP_OK) return rc;
    K = t.K, R = t.R, ITW = t.ITW, N = t.N, X = t.X;
    bool relax = false;
    for (int x = 0; x < X; x++) relax = relax || t.cls_relax[x] >= 0;
    bool limits = false;
    for (int n = 0; n < N; n++) limits = limits || t.tmpl_limit_present[n] != 0;
    bool lazy = false;
    for (int32_t b : t.g_born) lazy = lazy || b == 0;
    if (t.has_bounds || t.has_min_values || t.n_rsv > 0 || p->n_hostports > 0 || t.has_vol_alts || relax || limits || lazy || N > 64) {
      err = "orc_cached: shape outside what the cached CPU baseline serves";
      return KP_ERR_UNSUPPORTED;
    }
    GH = t.GH;
    E = t.E;
    node_rem = t.node_rem, node_rem_present = t.node_rem_present, node_npods.assign(std::max(E, 1), 0);
    node_slot.resize((size_t)std::max(E, 1) * K);
    for (size_t i = 0; i < (size_t)E * K; i++) node_slot[i] = Slot{t.node_sflags[i], t.node_smask[i], 0, 0};
    touched.assign(std::max(E, 1), 0);
    nactive.assign((size_t)(std::max(E, 1) + 63) / 64, 0ull);
    for (int n = 0; n < E; n++)
      if (t.node_flags[n] & KP_NODE_SCHEDULABLE) set(nactive, n);
    host_cnt.assign((size_t)E * GH, 0);
    for (int r = 0; r < GH; r++)
      for (int n = 0; n < E; n++) host_cnt[(size_t)n * GH + r] = t.host_cnt_nodes[(size_t)r * E + n];
    dom_cnt = t.dom_cnt, dom_reg = t.dom_reg, dom_pop = t.dom_pop, g_ndomains = t.g_ndomains, g_nempty = t.g_nempty;
    lbf.assign(std::max(pl.n_fsig, 1), 0), lbr.assign(std::max(t.n_rv, 1), 0);
    // k_feasibility, prefilter_only: NewScheduler keeps the template's types that pass its own requirements with zero
    // requests (scheduler.go:147)
    tmpl_its.assign((size_t)std::max(N, 1) * ITW, 0ull);
    for (int n = 0; n < N; n++) {
      std::vector<Slot> S(K);
      for (int k = 0; k < K; k++) S[k] = rs_slot(t.tmpl_rs[n], k);
      std::vector<int64_t> q(R, 0);
      std::vector<int> j(R, -1);
      std::vector<uint64_t> w(ITW, ~0ull);
      fits(q, j, w);
      compat_off(S, w);
      for (int i = 0; i < ITW; i++) tmpl_its[(size_t)n * ITW + i] = w[i] & t.tmpl_its_raw[(size_t)n * ITW + i];
    }
    // k_node_cand: candidate bitmaps of the existing nodes per (requirement set, toleration set) and per request vector
    const size_t ew = nactive.size();
    for (size_t s = 0; s < pl.nsig_rs.size(); s++) {
      const int rs = pl.nsig_rs[s];
      nstat.emplace_back(ew, 0ull);
      for (int n = 0; n < E; n++) {
        bool ok = tolerated(pl.nsig_tolset[s], t.node_taintset[n]);
        for (int k = 0; k < K && ok; k++) {
          const Slot pod = rs_slot(rs, k);
          if (!slot_present(pod)) continue;
          const Slot nd = node_slot[(size_t)n * K + k];
          if (!slot_present(nd)) {
            if (pl.strict_undefined && !op_is_negative(slot_op(pod))) ok = false;
          } else if (!slot_has_intersection(ki(k), nd, pod) && !(op_is_negative(slot_op(pod)) && op_is_negative(slot_op(nd)))) {
            ok = false;
          }
        }
        if (ok) set(nstat.back(), n);
      }
    }
    nfit.assign(std::max(t.n_rv, 1), std::vector<uint64_t>(ew, 0ull));
    std::vector<uint8_t> rv_done(std::max(t.n_rv, 1), 0);
    for (int x = 0; x < X; x++) {
      const int rv = t.cls_rv[x];
      if (rv_done[rv]) continue;
      rv_done[rv] = 1;
      for (int n = 0; n < E; n++) {
        bool ok = true;
        for (int r = 0; r < R; r++) {
          const int64_t rem = node_rem[(size_t)n * R + r];
          const bool present = (node_rem_present[n] >> r) & 1;
          if (present && rem < 0) ok = false;
          if (t.cls_req[(size_t)x * R + r] > (present ? rem : 0)) ok = false;
        }
        if (ok) set(nfit[rv], n);
      }
    }
    return KP_OK;
  }

  // NewQueue (queue.go:72-108): class rank by cpu desc, memory desc; then creation time, then UID
  void sort_rows(std::vector<int32_t>& rows) {
    std::stable_sort(rows.begin(), rows.end(), [&](int32_t a, int32_t b) {
      const int64_t ra = pl.rank[p->pod_class[a]], rb = pl.rank[p->pod_class[b]];
      if (ra != rb) return ra < rb;
      const int64_t ta = p->pod_creation ? p->pod_creation[a] : 0, tb = p->pod_creation ? p->pod_creation[b] : 0;
      if (ta != tb) return ta < tb;
      if (p->pod_uid_hi[a] != p->pod_uid_hi[b]) return p->pod_uid_hi[a] < p->pod_uid_hi[b];
      return p->pod_uid_lo[a] < p->pod_uid_lo[b];
    });
  }
  // a consolidation simulation works on a private view of the existing nodes: what it changes is logged and undone
  struct NodeUndo {
    int node;
    std::vector<int64_t> rem;
    uint32_t present;
    std::vector<Slot> slot;
    int32_t npods;
  };
  std::vector<NodeUndo> undo;
  std::vector<uint8_t> touched;
  void reset_claims() {
    claims.clear(), ord.clear(), cnt.clear(), failm.clear(), deadm.clear(), accm.clear();
    std::fill(lbf.begin(), lbf.end(), 0);
    std::fill(lbr.begin(), lbr.end(), 0);
  }
  void undo_nodes() {
    for (const NodeUndo& u : undo) {
      std::copy(u.rem.begin(), u.rem.end(), node_rem.begin() + (size_t)u.node * R);
      node_rem_present[u.node] = u.present;
      std::copy(u.slot.begin(), u.slot.end(), node_slot.begin() + (size_t)u.node * K);
      node_npods[u.node] = u.npods;
      touched[u.node] = 0;
    }
    undo.clear();
  }

  // One Scheduler.Solve over the pods `rows` (in queue order): target / perr per position in `rows`
  void run(const std::vector<int32_t>& rows, std::vector<int32_t>& target, std::vector<uint8_t>& perr, bool overlay) {
    const int64_t P = (int64_t)rows.size();
    std::vector<int32_t> queue(P);
    std::iota(queue.begin(), queue.end(), 0);
    target.assign(P, KP_TARGET_UNSCHEDULED);
    perr.assign(P, 0);
    std::vector<int32_t> last_len(P, 0);
    const uint64_t tmpl_all = N >= 64 ? ~0ull : ((1ull << N) - 1);
    int alive_tmpl = 0;
    for (int n = 0; n < N; n++) {
      bool any = false;
      for (int w = 0; w < ITW; w++) any = any || tmpl_its[(size_t)n * ITW + w];
      alive_tmpl += any;
    }
    enum { PERT_NONE, PERT_INC, PERT_APPEND };
    int pert = PERT_NONE, pert_pos = 0;
    size_t head = 0;
    const size_t fw = (size_t)(std::max(pl.n_fsig, 1) + 63) / 64, rw = (size_t)(std::max(t.n_rv, 1) + 63) / 64,
                 aw = (size_t)(std::max(pl.n_asig, 1) + 63) / 64;
    Eval ev;
    while (head < queue.size()) {
      // ---- Queue.Pop (queue.go:46-60)
      const int64_t len = (int64_t)queue.size() - (int64_t)head;
      const int32_t li = queue[head];
      if ((int64_t)head >= P && last_len[li] == len) break;  // a full cycle without progress
      head++;
      const int cls = p->pod_class[rows[li]], rv = t.cls_rv[cls], fs = pl.fsig[cls];
      const int nC = (int)claims.size();
      // ---- addToExistingNode (scheduler.go:520-555): the first node in order that passes
      if (E > 0) {
        bool placed = false;
        const std::vector<uint64_t>&fitrow = nfit[rv], &strow = nstat[pl.nsig[cls]];
        for (size_t w = 0; w < nactive.size() && !placed; w++) {
          for (uint64_t bits = fitrow[w] & strow[w] & nactive[w]; bits && !placed; bits &= bits - 1) {
            const int node = (int)w * 64 + __builtin_ctzll(bits);
            bool bad = false;  // resources.Fits(pod requests, remaining) (resources.go:150-163)
            for (int r = 0; r < R; r++) {
              const int64_t rem = node_rem[(size_t)node * R + r];
              const bool present = (node_rem_present[node] >> r) & 1;
              if (present && rem < 0) bad = true;
              if (t.cls_req[(size_t)cls * R + r] > (present ? rem : 0)) bad = true;
            }
            if (bad) {
              if (!overlay) nfit[rv][w] &= ~(1ull << (node & 63));  // monotone: remaining resources only shrink
              continue;
            }
            std::vector<Slot> nb(node_slot.begin() + (size_t)node * K, node_slot.begin() + (size_t)(node + 1) * K);
            eval(cls, node, nb, {}, {}, {}, ev, false);
            if (!ev.ok) continue;
            if (overlay && !touched[node]) {
              touched[node] = 1;
              undo.push_back(NodeUndo{node, std::vector<int64_t>(node_rem.begin() + (size_t)node * R, node_rem.begin() + (size_t)(node + 1) * R),
                                      node_rem_present[node], nb, node_npods[node]});
            }
            if (ev.changed)
              for (int k = 0; k < K; k++) node_slot[(size_t)node * K + k] = ev.F[k];
            for (int r = 0; r < R; r++) node_rem[(size_t)node * R + r] -= t.cls_req[(size_t)cls * R + r];
            node_rem_present[node] |= (1u << R) - 1;
            node_npods[node]++;
            target[li] = node;
            perr[li] = KP_PODERR_NONE;
            if (t.cls_rec_off[cls + 1] > t.cls_rec_off[cls]) topo_record(cls, ev.F, t.node_taintset[node], node);
            placed = true;
          }
        }
        if (placed) continue;
      }
      // ---- sort.Slice(newNodeClaims, len(Pods) asc) (scheduler.go:504), wsolve_run's sort stage
      if (pert != PERT_NONE) {
        const int q = pert_pos;
        const bool inversion = pert == PERT_INC ? (q + 1 < nC && cnt[ord[q + 1]] < cnt[ord[q]])
                                                : (nC >= 2 && cnt[ord[nC - 1]] < cnt[ord[nC - 2]]);
        if (inversion) {
          bool stable = p->claim_order_mode == 1 || nC <= 12;
          if (!stable && nC >= 50) {
            const int q4 = nC / 4;
            stable = pert == PERT_APPEND || !(q == q4 - 1 || q == q4 || q == 2 * q4 - 1 || q == 2 * q4 || q == 3 * q4 - 1 || q == 3 * q4);
          }
          if (stable) {
            if (pert == PERT_INC) {  // elevated count: smaller successors move left
              const int eo = ord[q], ec = cnt[eo];
              int i0 = q;
              while (i0 + 1 < nC && cnt[ord[i0 + 1]] < ec) {
                ord[i0] = ord[i0 + 1];
                i0++;
              }
              ord[i0] = eo;
              for (int& b : lbf)
                if (q < b && b <= i0) b--;
              for (int& b : lbr)
                if (q < b && b <= i0) b--;
            } else {  // appended claim: larger predecessors move right
              const int eo = ord[nC - 1], ec = cnt[eo];
              int i0 = nC - 1;
              while (i0 - 1 >= 0 && cnt[ord[i0 - 1]] > ec) {
                ord[i0] = ord[i0 - 1];
                i0--;
              }
              ord[i0] = eo;
              for (int& b : lbf)
                if (b > i0) b = i0;
              for (int& b : lbr)
                if (b > i0) b = i0;
            }
          } else {  // the real pdqsort (kp_gosort_host.hpp)
            HostGoSort<int> s{cnt.data(), ord.data()};
            s.pdqsort(0, nC, HostGoSort<int>::bits_len((unsigned long long)nC));
            slow_sorts++;
            std::fill(lbf.begin(), lbf.end(), 0);
            std::fill(lbr.begin(), lbr.end(), 0);
          }
        } else if (pert == PERT_APPEND) {
          for (int& b : lbf)
            if (b > nC - 1) b = nC - 1;
          for (int& b : lbr)
            if (b > nC - 1) b = nC - 1;
        }
        pert = PERT_NONE;
      }
      // ---- addToInflightNode (scheduler.go:557-589)
      bool found = false;
      {
        const int lbf_ = fs >= 0 ? lbf[fs] : 0, lbr_ = lbr[rv];
        const int lb = std::max(lbf_, lbr_);
        const bool scanned = (pl.tok[cls] & tmpl_all) != 0;
        int first_clear = -1, first_rclear = -1;
        // the class's shortcuts (wsolve_run: tkinfo): topology-free fast path, or the domain fast path with its mask
        const bool topo = t.cls_match_off[cls + 1] > t.cls_match_off[cls] || t.cls_rec_off[cls + 1] > t.cls_rec_off[cls];
        const bool fast_ok = pl.fast[cls];
        bool dom_fp = topo && pl.fp[cls], use_ez = false;
        const bool has_tk = pl.has_tk[cls];
        uint64_t ez = ~0ull;
        if (dom_fp && has_tk) {
          bool exact;
          ez = domain_mask(cls, &exact);
          use_ez = exact;
          dom_fp = exact;
        }
        for (int pos = lb; scanned && pos < nC && !found; pos++) {
          const int c = ord[pos];
          const bool fclear = fs < 0 || !bit(failm[c], fs), rclear = !bit(deadm[c], rv);
          if (fs >= 0 && first_clear < 0 && fclear) first_clear = pos;
          if (first_rclear < 0 && rclear) first_rclear = pos;
          if (!fclear || !rclear) continue;
          Claim& cl = claims[c];
          if (!((pl.tok[cls] >> cl.tmpl) & 1ull)) continue;
          if (use_ez && cl.dom != 0xff && !((ez >> cl.dom) & 1ull)) continue;  // pinned to a value the pod may not use
          {  // hostname groups: a NodeClaim is one hostname domain (next_candidate)
            bool pass = true;
            for (int i = pl.hchk_off[cls]; i < pl.hchk_off[cls + 1]; i++) {
              const HostCheck& hc = pl.hchk[i];
              const int hcnt = host_cnt[(size_t)(E + c) * GH + hc.row];
              if (hc.type == KP_TOPO_SPREAD)
                pass = hcnt + hc.self <= hc.max_skew;
              else if (hc.type == KP_TOPO_AFFINITY)
                pass = hcnt > 0 || (hc.self && (g_ndomains[hc.g] - g_nempty[hc.g]) == 0);
              else
                pass = hcnt == 0;
              if (!pass) break;
            }
            if (!pass) continue;
          }
          int zdom = -1;
          bool fp = false;
          if ((fast_ok || dom_fp) && bit(accm[c], pl.asig[cls])) {
            fp = true;
            if (!fast_ok && has_tk) {
              zdom = cl.dom;
              fp = zdom != 0xff;
            }
          }
          if (fp) {
            // the accepted-signature fast path (fp_fit): the requirements stay, only the resource test can fail
            evals_++;
            std::vector<int64_t>& q = ev.q;
            q = cl.q;
            for (int r = 0; r < R; r++) q[r] += t.cls_req[(size_t)cls * R + r];
            ev.j = cl.j;
            ev.its = cl.its;
            if (!fits(q, ev.j, ev.its)) {
              set(deadm[c], rv);
              continue;
            }
            cl.q.swap(q);
            cl.j.swap(ev.j);
            cl.its.swap(ev.its);
            fast_commits++;
            if (!fast_ok) topo_record_fast(cls, zdom, t.tmpl_taintset[cl.tmpl], E + c);
          } else {
            eval(cls, E + c, cl.s, cl.q, cl.its, cl.j, ev);
            if (ev.pod_noop) set(accm[c], pl.asig[cls]);
            if (!ev.ok) {
              if (ev.res_dead) set(deadm[c], rv);
              if (ev.compat_fail && fs >= 0) set(failm[c], fs);
              continue;
            }
            if (ev.changed) {
              cl.s = ev.F;
              if (pl.tk_key >= 0) cl.dom = pinned(ev.F[pl.tk_key]);
            }
            cl.q = ev.q;
            cl.j = ev.j;
            cl.its = ev.its;
            if (topo) topo_record(cls, ev.F, t.tmpl_taintset[cl.tmpl], E + c);
          }
          cnt[c]++;
          target[li] = KP_TARGET_CLAIM(c);
          perr[li] = KP_PODERR_NONE;
          pert = PERT_INC;
          pert_pos = pos;
          found = true;
        }
        if (fs >= 0 && scanned && lbf_ == lb) lbf[fs] = first_clear >= 0 ? first_clear : nC;
        if (scanned && lbr_ == lb) lbr[rv] = first_rclear >= 0 ? first_rclear : nC;
      }
      if (found) continue;
      // ---- addToNewNodeClaim (scheduler.go:592-684)
      int err = alive_tmpl ? KP_PODERR_INCOMPATIBLE : KP_PODERR_NO_TEMPLATES;
      for (int n = 0; n < N && !found; n++) {
        std::vector<uint64_t> tw(tmpl_its.begin() + (size_t)n * ITW, tmpl_its.begin() + (size_t)(n + 1) * ITW);
        bool alive = false;
        for (uint64_t w : tw) alive = alive || w;
        if (!alive) continue;
        if (!((pl.tok[cls] >> n) & 1ull)) continue;
        std::vector<Slot> b(K);
        for (int k = 0; k < K; k++) b[k] = rs_slot(t.tmpl_rs[n], k);
        std::vector<int64_t> bq(t.tmpl_daemon.begin() + (size_t)n * R, t.tmpl_daemon.begin() + (size_t)(n + 1) * R);
        eval(cls, E + (int)claims.size(), b, bq, tw, std::vector<int>(R, -1), ev);
        if (!ev.ok) continue;
        Claim cl;
        cl.s = ev.F;
        if (pl.tk_key >= 0) cl.dom = pinned(ev.F[pl.tk_key]);
        cl.q = ev.q;
        cl.j = ev.j;
        cl.its = ev.its;
        cl.tmpl = n;
        const int cnew = (int)claims.size();
        claims.push_back(std::move(cl));
        ord.push_back(cnew);
        cnt.push_back(1);
        failm.emplace_back(fw, 0ull);
        deadm.emplace_back(rw, 0ull);
        accm.emplace_back(aw, 0ull);
        if (ev.pod_noop) set(accm[cnew], pl.asig[cls]);
        if (GH > 0) {  // Topology.Register(hostname) (nodeclaim.go:213): every hostname group learns the new, empty domain
          host_cnt.resize((size_t)(E + cnew + 1) * GH, 0);
          for (int g = 0; g < t.G; g++)
            if (t.groups[g].key == t.hostname_key) {
              g_ndomains[g]++;
              g_nempty[g]++;
            }
        }
        if (t.cls_rec_off[cls + 1] > t.cls_rec_off[cls]) topo_record(cls, claims[cnew].s, t.tmpl_taintset[n], E + cnew);
        target[li] = KP_TARGET_CLAIM(cnew);
        perr[li] = KP_PODERR_NONE;
        pert = PERT_APPEND;
        pert_pos = cnew;
        found = true;
      }
      if (found) continue;
      // scheduler.go:415-421: record the error and requeue the pod
      perr[li] = (uint8_t)err;
      target[li] = KP_TARGET_UNSCHEDULED;
      queue.push_back(li);
      last_len[li] = (int32_t)((int64_t)queue.size() - (int64_t)head);
    }
  }

  int solve(kp_result* out) {
    const int64_t P = p->n_pods;
    std::vector<int32_t> rows(P);
    std::iota(rows.begin(), rows.end(), 0);
    sort_rows(rows);
    std::vector<int32_t> tl;
    std::vector<uint8_t> el;
    run(rows, tl, el, false);
    std::vector<int32_t> target(P, KP_TARGET_UNSCHEDULED);
    std::vector<uint8_t> perr(P, 0);
    for (int64_t i = 0; i < P; i++) {
      target[rows[i]] = tl[i];
      perr[rows[i]] = el[i];
    }
    // ---- result (the fields the parity test compares)
    memset(out, 0, sizeof(*out));
    const int C = (int)claims.size();
    const size_t c1 = C ? C : 1;
    out->n_pods = P;
    out->pod_target = (int32_t*)malloc(sizeof(int32_t) * (P ? P : 1));
    out->pod_error = (uint8_t*)malloc(P ? P : 1);
    memcpy(out->pod_target, target.data(), sizeof(int32_t) * P);
    memcpy(out->pod_error, perr.data(), P);
    out->n_claims = C;
    out->it_words = ITW;
    out->claim_template = (int32_t*)calloc(c1, 4);
    out->claim_npods = (int32_t*)calloc(c1, 4);
    out->claim_rank = (int32_t*)calloc(c1, 4);
    out->claim_requests = (int64_t*)calloc(c1 * R, 8);
    out->claim_its = (uint64_t*)calloc(c1 * ITW, 8);
    for (int pos = 0; pos < C; pos++) out->claim_rank[ord[pos]] = pos;
    for (int c = 0; c < C; c++) {
      out->claim_template[c] = claims[c].tmpl;
      out->claim_npods[c] = cnt[c];
      for (int r = 0; r < R; r++) out->claim_requests[(size_t)c * R + r] = claims[c].q[r];
      for (int w = 0; w < ITW; w++) out->claim_its[(size_t)c * ITW + w] = claims[c].its[w];
    }
    out->n_inflight_evals = evals_;
    out->n_commits = fast_commits;
    return KP_OK;
  }

  // ---- consolidation: SimulateScheduling + computeConsolidation per candidate set (disruption/helpers.go:51-142,
  // consolidation.go:136-229) -- k_consolidate and consol_decide on one core, topology-free pods only
  unsigned offering_ok_mask(const std::vector<Slot>& S) const {
    unsigned m = 0;
    for (int dd = 0; dd < t.D; dd++) {
      bool ok = true;
      for (uint32_t keys = t.off_keys[dd]; keys && ok; keys &= keys - 1) {
        const int k = __builtin_ctz(keys);
        ok = slot_compatible(ki(k), S[k], t.off_slots[(size_t)dd * K + k], t.key_wellknown[k], true);
      }
      if (ok) m |= 1u << dd;
    }
    return m;
  }
  int consolidate(const kp_consol_input* in, kp_consol_result* out, std::string& err) {
    if (t.G > 0 || in->n_extra_pods > 0) {
      err = "orc_cached: consolidation of topology-free candidate pods without extra pods only";
      return KP_ERR_UNSUPPORTED;
    }
    const int S = in->n_subsets, ct_key = in->capacity_type_key;
    // getCandidatePrices, the WorstLaunchPrice lists per capacity type and the OrderByPrice lists (kp_prep.cpp)
    const ConsolPrices cp = consol_prices(p, t, in);
    const std::vector<double>& node_price = cp.node_price;
    const PriceLists ml = order_by_price(p, t);
    const double INF = 1.7976931348623157e308;
    auto worst = [&](int ty, unsigned okmask) {
      for (int ci = 0; ci < 3; ci++) {
        if (ct_key < 0 || !((cp.ct_valid >> ci) & 1)) continue;
        for (int e = cp.worst.off[(size_t)ty * 3 + ci]; e < cp.worst.off[(size_t)ty * 3 + ci + 1]; e++)
          if ((okmask >> cp.worst.set[e]) & 1u) return cp.worst.price[e];
      }
      return INF;
    };
    auto has = [&](const std::vector<uint64_t>& m, int ty) { return (m[ty >> 6] >> (ty & 63)) & 1ull; };
    // ---- result arrays
    memset(out, 0, sizeof(*out));
    const size_t s1 = S ? S : 1;
    out->n_subsets = S;
    out->it_words = ITW;
    out->decision = (uint8_t*)calloc(s1, 1);
    out->replacement_its = (uint64_t*)calloc(s1 * ITW, 8);
    out->n_new_claims = (int32_t*)calloc(s1, 4);
    out->n_unscheduled = (int32_t*)calloc(s1, 4);
    std::vector<int32_t> rows, tl;
    std::vector<uint8_t> el;
    auto t0 = std::chrono::steady_clock::now();
    for (int s_i = 0; s_i < S; s_i++) {
      const int32_t* snodes = in->subset_nodes + in->subset_off[s_i];
      const int sn = in->subset_off[s_i + 1] - in->subset_off[s_i];
      // ---- SimulateScheduling: the candidates leave, their pods are scheduled against the rest of the cluster
      rows.clear();
      for (int i = 0; i < sn; i++) {
        const int n = snodes[i];
        nactive[n >> 6] &= ~(1ull << (n & 63));
        for (int j = in->node_pod_off[n]; j < in->node_pod_off[n + 1]; j++) rows.push_back(j);
      }
      sort_rows(rows);
      reset_claims();
      run(rows, tl, el, true);
      int unscheduled = 0;
      for (size_t i = 0; i < tl.size(); i++) {
        if (tl[i] == KP_TARGET_UNSCHEDULED)
          unscheduled++;
        else if (tl[i] >= 0 && !(p->node_flags[tl[i]] & KP_NODE_INITIALIZED))
          unscheduled++;  // helpers.go:121-140 UninitializedNodeError
      }
      undo_nodes();
      for (int i = 0; i < sn; i++)
        if (p->node_flags[snodes[i]] & KP_NODE_SCHEDULABLE) nactive[snodes[i] >> 6] |= 1ull << (snodes[i] & 63);
      const int n_new = (int)claims.size();
      out->n_new_claims[s_i] = n_new;
      out->n_unscheduled[s_i] = unscheduled;
      // ---- computeConsolidation (consol_decide)
      int decision = KP_DECISION_NOOP;
      std::vector<uint64_t> rep(ITW, 0ull);
      if (!unscheduled && n_new == 0) decision = KP_DECISION_DELETE;
      if (!unscheduled && n_new == 1) {
        std::vector<Slot> Sx = claims[0].s;
        std::vector<uint64_t> cur = claims[0].its;
        int n_its = 0;
        for (uint64_t w : cur) n_its += __builtin_popcountll(w);
        double price = 0;
        bool zero = false, all_spot = true;
        for (int i = 0; i < sn; i++) {
          const double np = node_price[snodes[i]];
          if (np < 0) zero = true;
          price += np;
          if (!in->node_is_spot[snodes[i]]) all_spot = false;
        }
        if (zero) price = 0.0;
        const bool spot_ok = ct_key >= 0 && in->ct_spot >= 0 && slot_has(ki(ct_key), Sx[ct_key], in->ct_spot);
        unsigned okmask = offering_ok_mask(Sx);
        const bool spot_path = all_spot && spot_ok;
        // OrderByPrice + Truncate(600): the order only matters when it truncates or for the 15-cheapest rule
        std::vector<int32_t> order;  // types in price order
        if (n_its > 600 || (spot_path && in->spot_to_spot_enabled)) {
          std::vector<int32_t> types, perm;
          std::vector<double> key;
          for (int w = 0; w < ITW; w++)
            for (uint64_t b = cur[w]; b; b &= b - 1) {
              const int ty = w * 64 + __builtin_ctzll(b);
              double mp = INF;
              for (int e = ml.off[ty]; e < ml.off[ty + 1]; e++)
                if ((okmask >> ml.set[e]) & 1u) {
                  mp = ml.price[e];
                  break;
                }
              types.push_back(ty);
              key.push_back(mp);
            }
          perm.resize(types.size());
          std::iota(perm.begin(), perm.end(), 0);
          HostGoSort<double> gs{key.data(), perm.data()};
          gs.pdqsort(0, (int)perm.size(), HostGoSort<double>::bits_len((unsigned long long)perm.size()));
          for (int32_t i : perm) order.push_back(types[i]);
          if (order.size() > 600) {
            order.resize(600);
            std::fill(cur.begin(), cur.end(), 0ull);
            for (int32_t ty : order) cur[ty >> 6] |= 1ull << (ty & 63);
          }
        }
        if (!(spot_path && !in->spot_to_spot_enabled)) {
          if (spot_path) {  // restrict the claim to spot and drop types without such an offering (consolidation.go:252-257)
            Sx[ct_key] = slot_add(ki(ct_key), Sx[ct_key], Slot{SF_PRESENT, 1ull << in->ct_spot, 0, 0});
            okmask = offering_ok_mask(Sx);
            for (int w = 0; w < ITW; w++) {
              uint64_t keep = 0;
              for (uint64_t b = cur[w]; b; b &= b - 1) {
                const int ty = w * 64 + __builtin_ctzll(b);
                for (int e = ml.off[ty]; e < ml.off[ty + 1]; e++)
                  if ((okmask >> ml.set[e]) & 1u) {
                    keep |= 1ull << (ty & 63);
                    break;
                  }
              }
              cur[w] = keep;
            }
          }
          // RemoveInstanceTypeOptionsByPriceAndMinValues (nodeclaim.go:309-318): keep WorstLaunchPrice < price
          bool any = false;
          for (int w = 0; w < ITW; w++)
            for (uint64_t b = cur[w]; b; b &= b - 1) {
              const int ty = w * 64 + __builtin_ctzll(b);
              if (worst(ty, okmask) < price) {
                rep[w] |= 1ull << (ty & 63);
                any = true;
              }
            }
          if (any && spot_path && sn == 1) {  // at least 15 cheaper types, only the 15 cheapest go out (consolidation.go:283-312)
            int total = 0;
            for (uint64_t w : rep) total += __builtin_popcountll(w);
            if (total < 15) {
              any = false;
            } else {
              std::vector<uint64_t> first(ITW, 0ull);
              int taken = 0;
              for (int32_t ty : order) {
                if (taken >= 15) break;
                if (has(rep, ty)) {
                  first[ty >> 6] |= 1ull << (ty & 63);
                  taken++;
                }
              }
              rep = first;
            }
          }
          if (any && in->filter_same_instance_type && sn >= 2) {  // filterOutSameInstanceType (multinodeconsolidation.go:189-226)
            double max_price = INF;
            for (int i = 0; i < sn; i++) {
              const int ty = in->node_it[snodes[i]];
              if (ty < 0 || !has(rep, ty)) continue;
              double mine = INF;
              for (int j = 0; j < sn; j++)
                if (in->node_it[snodes[j]] == ty && node_price[snodes[j]] >= 0 && node_price[snodes[j]] < mine) mine = node_price[snodes[j]];
              if (mine > 1e308) mine = 0.0;
              if (mine < max_price) max_price = mine;
            }
            if (max_price < 1e308) {
              any = false;
              for (int w = 0; w < ITW; w++) {
                uint64_t keep = 0;
                for (uint64_t b = rep[w]; b; b &= b - 1) {
                  const int ty = w * 64 + __builtin_ctzll(b);
                  if (worst(ty, okmask) < max_price) keep |= 1ull << (ty & 63);
                }
                rep[w] = keep;
                any = any || keep;
              }
            }
          }
          if (any) decision = KP_DECISION_REPLACE;
        }
      }
      out->decision[s_i] = (uint8_t)decision;
      if (decision == KP_DECISION_REPLACE)
        for (int w = 0; w < ITW; w++) out->replacement_its[(size_t)s_i * ITW + w] = rep[w];
    }
    out->solve_ms = std::chrono::duration<double, std::milli>(std::chrono::steady_clock::now() - t0).count();
    return KP_OK;
  }
};

}  // namespace

extern "C" {
// kp_consolidate's fast path on one host core: decision, replacement_its, n_new_claims, n_unscheduled of `out` (free with
// orc_cached_consol_free); solve_ms = the simulations + decisions alone (tables and price lists prepared before)
int orc_cached_consolidate(const kp_problem* p, const kp_consol_input* in, kp_consol_result* out, double* prep_ms) {
  Solver s;
  s.p = p;
  std::string err;
  auto t0 = std::chrono::steady_clock::now();
  int rc = s.prepare(err);
  if (rc != KP_OK) return rc;
  auto t1 = std::chrono::steady_clock::now();
  rc = s.consolidate(in, out, err);
  if (prep_ms) *prep_ms = std::chrono::duration<double, std::milli>(t1 - t0).count();
  return rc;
}
void orc_cached_consol_free(kp_consol_result* r) {
  free(r->decision);
  free(r->replacement_its);
  free(r->n_new_claims);
  free(r->n_unscheduled);
  memset(r, 0, sizeof(*r));
}

// One Scheduler.Solve with the CUDA solver's caches on one host core.  Fills pod_target, pod_error, n_claims,
// claim_template / npods / rank / requests / its of `out` (free with orc_cached_free); solve_ms = the solve alone (tables
// prepared before the clock starts, like the resident GPU number), KP_ERR_UNSUPPORTED outside the lean shape.
int orc_cached_solve(const kp_problem* p, kp_result* out, double* prep_ms) {
  Solver s;
  s.p = p;
  std::string err;
  auto t0 = std::chrono::steady_clock::now();
  int rc = s.prepare(err);
  if (rc != KP_OK) return rc;
  auto t1 = std::chrono::steady_clock::now();
  rc = s.solve(out);
  auto t2 = std::chrono::steady_clock::now();
  if (prep_ms) *prep_ms = std::chrono::duration<double, std::milli>(t1 - t0).count();
  out->solve_ms = std::chrono::duration<double, std::milli>(t2 - t1).count();
  return rc;
}
void orc_cached_free(kp_result* r) {
  free(r->pod_target);
  free(r->pod_error);
  free(r->claim_template);
  free(r->claim_npods);
  free(r->claim_rank);
  free(r->claim_requests);
  free(r->claim_its);
  memset(r, 0, sizeof(*r));
}
}
