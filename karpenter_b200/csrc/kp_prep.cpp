// kp_prep.cpp -- see kp_prep.hpp
#include "kp_prep.hpp"

#include <sstream>

namespace {

struct Ctx {
  const kp_problem* p;
  const HostTables& h;
  int K, R;
  Ctx(const kp_problem* pp, const HostTables& hh) : p(pp), h(hh), K(pp->n_keys), R(pp->n_resources) {}

  KeyInfo ki(int k) const { return KeyInfo{h.val_int.data() + (size_t)k * 64, h.val_isint[k], h.key_univ[k]}; }
  Slot rs_slot(int rs, int k) const {
    size_t i = (size_t)rs * K + k;
    return Slot{h.rs_flags[i], h.rs_mask[i], h.rs_gte[i], h.rs_lte[i]};
  }
  // Taints.Tolerates(tolerations) (pkg/scheduling/taints.go:54-66) via corev1.Toleration.ToleratesTaint
  bool tolerates_taint(int tol, int taint) const {
    uint8_t te = p->tol_effect[tol];
    if (te != KP_EFFECT_NONE && te != p->taint_effect[taint]) return false;
    if (p->tol_key[tol] != 0 && p->tol_key[tol] != p->taint_key[taint]) return false;
    switch (p->tol_op[tol]) {
      case KP_TOL_EQUAL:
        return p->tol_value[tol] == p->taint_value[taint];
      case KP_TOL_EXISTS:
        return true;
      default: {
        int a = p->taint_value[taint], b = p->tol_value[tol];
        if (!p->tt_is_int || !p->tt_is_int[a] || !p->tt_is_int[b]) return false;
        return p->tol_op[tol] == KP_TOL_LT ? p->tt_int[a] < p->tt_int[b] : p->tt_int[a] > p->tt_int[b];
      }
    }
  }
  bool tolerates(int taintset, int tolset) const {
    if (taintset < 0) return true;
    for (int i = p->taintset_off[taintset]; i < p->taintset_off[taintset + 1]; i++) {
      bool ok = false;
      if (tolset >= 0)
        for (int j = p->tolset_off[tolset]; j < p->tolset_off[tolset + 1] && !ok; j++)
          ok = tolerates_taint(p->tolset_ids[j], p->taintset_ids[i]);
      if (!ok) return false;
    }
    return true;
  }
  int taintset_size(int ts) const { return ts < 0 ? 0 : p->taintset_off[ts + 1] - p->taintset_off[ts]; }

  bool label_lookup(int ls, int key, int* val) const {
    if (ls < 0) return false;
    for (int i = p->labelset_off[ls]; i < p->labelset_off[ls + 1]; i++)
      if (p->label_key[i] == key) {
        *val = p->label_val[i];
        return true;
      }
    return false;
  }
  // labels.Selector.Matches for a metav1.LabelSelector; nil selector matches nothing (topologygroup.go:101-104)
  bool selector_matches(int sel, int ls) const {
    if (sel < 0) return false;
    for (int e = p->selector_off[sel]; e < p->selector_off[sel + 1]; e++) {
      int val = 0;
      bool has = label_lookup(ls, p->selx_key[e], &val), in = false;
      if (has)
        for (int i = p->selx_val_off[e]; i < p->selx_val_off[e + 1]; i++) in |= p->selx_vals[i] == val;
      int op = p->selx_op[e];
      if (op == KP_SEL_IN && !(has && in)) return false;
      if (op == KP_SEL_NOT_IN && has && in) return false;
      if (op == KP_SEL_EXISTS && !has) return false;
      if (op == KP_SEL_DOES_NOT_EXIST && has) return false;
    }
    return true;
  }
  bool nsset_has(int nsset, int ns) const {
    for (int i = p->nsset_off[nsset]; i < p->nsset_off[nsset + 1]; i++)
      if (p->nsset_ids[i] == ns) return true;
    return false;
  }
  // requirements.Compatible(A, B) over whole slot rows given by accessors
  template <class FA, class FB>
  bool rows_compatible(FA a, FB b, bool allow_undefined) const {
    for (int k = 0; k < K; k++)
      if (!slot_compatible(ki(k), a(k), b(k), h.key_wellknown[k], allow_undefined)) return false;
    return true;
  }
};

struct HGroup {
  KpGroup g;
  bool lazy = false;  // only a relaxed class owns it: born mid-solve (KpDev::g_born)
  int nsset, selector;
  std::vector<int> filter;
  std::set<int> owners;
  uint64_t reg = 0;
  int32_t cnt[64];
  std::map<int, int32_t> host_cnt;  // node index -> count (hostname groups)
  std::set<int> host_reg;           // registered hostname domains (node indices)
  HGroup() {
    memset(&g, 0, sizeof(g));
    memset(cnt, 0, sizeof(cnt));
  }
};

}  // namespace

// One O(input) pass over everything the encoder indexes with: a buggy caller gets KP_ERR_INVALID and a message, not a
// corrupted controller process.  (Counts, CSR offsets monotone and inside their arrays, every id inside its table.)
static int validate_problem(const kp_problem* p, std::string& err) {
#define KP_BAD(msg) return err = std::string("invalid problem: ") + msg, KP_ERR_INVALID
  auto csr = [](const int32_t* off, int64_t n, int64_t limit) {
    if (n == 0) return true;
    if (!off || off[0] != 0) return false;
    for (int64_t i = 0; i < n; i++)
      if (off[i + 1] < off[i]) return false;
    return limit < 0 || off[n] <= limit;
  };
  auto in = [](int64_t v, int64_t n) { return v >= 0 && v < n; };
  if (p->n_keys < 0 || p->n_reqsets < 0 || p->n_reqs < 0 || p->n_resources < 0 || p->n_its < 0 || p->n_templates < 0 ||
      p->n_classes < 0 || p->n_pods < 0 || p->n_nodes < 0 || p->n_running < 0 || p->n_taints < 0 || p->n_taintsets < 0 ||
      p->n_tolerations < 0 || p->n_tolsets < 0 || p->n_labelsets < 0 || p->n_selectors < 0 || p->n_nssets < 0 ||
      p->n_tt_strings < 0 || p->n_minvalue_keys < 0)
    KP_BAD("negative count");
  if (p->n_keys > 0 && (!p->key_flags || !csr(p->key_value_off, p->n_keys, -1))) KP_BAD("key_value_off");
  const int64_t n_values = p->n_keys > 0 ? p->key_value_off[p->n_keys] : 0;
  (void)n_values;
  if (!csr(p->reqset_off, p->n_reqsets, p->n_reqs) || (p->n_reqsets > 0 && p->reqset_off[p->n_reqsets] != p->n_reqs)) KP_BAD("reqset_off");
  if (p->n_reqs > 0 && (!p->req_key || !p->req_flags || !csr(p->req_val_off, p->n_reqs, -1))) KP_BAD("req_val_off");
  for (int i = 0; i < p->n_reqs; i++) {
    if (!in(p->req_key[i], p->n_keys)) KP_BAD("req_key out of range");
    const int nv = p->key_value_off[p->req_key[i] + 1] - p->key_value_off[p->req_key[i]];
    for (int e = p->req_val_off[i]; e < p->req_val_off[i + 1]; e++)
      if (!in(p->req_vals[e], nv)) KP_BAD("req_vals: value id outside its key");
  }
  if (!csr(p->taintset_off, p->n_taintsets, -1) || !csr(p->tolset_off, p->n_tolsets, -1)) KP_BAD("taintset_off / tolset_off");
  for (int i = 0; i < (p->n_taintsets ? p->taintset_off[p->n_taintsets] : 0); i++)
    if (!in(p->taintset_ids[i], p->n_taints)) KP_BAD("taintset_ids");
  for (int i = 0; i < (p->n_tolsets ? p->tolset_off[p->n_tolsets] : 0); i++)
    if (!in(p->tolset_ids[i], p->n_tolerations)) KP_BAD("tolset_ids");
  for (int i = 0; i < p->n_taints; i++)
    if (!in(p->taint_key[i], p->n_tt_strings) || !in(p->taint_value[i], p->n_tt_strings)) KP_BAD("taint strings");
  for (int i = 0; i < p->n_tolerations; i++)
    if (!in(p->tol_key[i], p->n_tt_strings) || !in(p->tol_value[i], p->n_tt_strings)) KP_BAD("toleration strings");
  if (!csr(p->it_off_off, p->n_its, -1)) KP_BAD("it_off_off");
  const int n_off = p->n_its ? p->it_off_off[p->n_its] : 0;
  for (int i = 0; i < p->n_its; i++)
    if (!in(p->it_reqset[i], p->n_reqsets)) KP_BAD("it_reqset");
  for (int i = 0; i < n_off; i++)
    if (!in(p->off_reqset[i], p->n_reqsets)) KP_BAD("off_reqset");
  if (!csr(p->tmpl_it_off, p->n_templates, -1)) KP_BAD("tmpl_it_off");
  for (int n = 0; n < p->n_templates; n++) {
    if (!in(p->tmpl_reqset[n], p->n_reqsets)) KP_BAD("tmpl_reqset");
    if (p->tmpl_taintset[n] < -1 || p->tmpl_taintset[n] >= p->n_taintsets) KP_BAD("tmpl_taintset");
    for (int i = p->tmpl_it_off[n]; i < p->tmpl_it_off[n + 1]; i++)
      if (!in(p->tmpl_its[i], p->n_its)) KP_BAD("tmpl_its");
  }
  if (!csr(p->labelset_off, p->n_labelsets, -1) || !csr(p->selector_off, p->n_selectors, -1) || !csr(p->nsset_off, p->n_nssets, -1))
    KP_BAD("labelset_off / selector_off / nsset_off");
  if (p->n_selectors > 0 && !csr(p->selx_val_off, p->selector_off[p->n_selectors], -1)) KP_BAD("selx_val_off");
  if (p->n_classes > 0 && (!csr(p->class_filter_off, p->n_classes, -1) || !csr(p->class_tsc_off, p->n_classes, -1)))
    KP_BAD("class_filter_off / class_tsc_off");
  for (int x = 0; x < p->n_classes; x++) {
    if (!in(p->class_reqset[x], p->n_reqsets) || !in(p->class_strict_reqset[x], p->n_reqsets)) KP_BAD("class_reqset");
    if (p->class_tolset[x] < -1 || p->class_tolset[x] >= p->n_tolsets) KP_BAD("class_tolset");
    if (p->class_labelset[x] < -1 || p->class_labelset[x] >= p->n_labelsets) KP_BAD("class_labelset");
    for (int i = p->class_filter_off[x]; i < p->class_filter_off[x + 1]; i++)
      if (!in(p->class_filter_reqsets[i], p->n_reqsets)) KP_BAD("class_filter_reqsets");
    if (p->class_relax_next && (p->class_relax_next[x] < -1 || p->class_relax_next[x] >= p->n_classes)) KP_BAD("class_relax_next");
    if (p->class_vol_next) {
      if (p->class_vol_next[x] < -1 || p->class_vol_next[x] >= p->n_classes) KP_BAD("class_vol_next");
      int steps = 0;  // a chain ends, and its members are the same pod: same requests
      for (int c = p->class_vol_next[x]; c >= 0; c = p->class_vol_next[c]) {
        if (c >= p->n_classes || ++steps > p->n_classes) KP_BAD("class_vol_next (cyclic)");
        for (int r = 0; r < p->n_resources; r++)
          if (p->class_requests[(size_t)c * p->n_resources + r] != p->class_requests[(size_t)x * p->n_resources + r]) KP_BAD("class_vol_next (requests differ)");
      }
    }
    for (int i = p->class_tsc_off[x]; i < p->class_tsc_off[x + 1]; i++) {
      if (!in(p->tsc_key[i], p->n_keys)) KP_BAD("tsc_key");
      if (p->tsc_selector[i] < -1 || p->tsc_selector[i] >= p->n_selectors) KP_BAD("tsc_selector");
      if (p->tsc_nsset[i] < -1 || p->tsc_nsset[i] >= p->n_nssets) KP_BAD("tsc_nsset");
      if (p->tsc_type[i] > KP_TOPO_ANTI_AFFINITY) KP_BAD("tsc_type");
    }
  }
  for (int64_t i = 0; i < p->n_pods; i++)
    if (!in(p->pod_class[i], p->n_classes)) KP_BAD("pod_class");
  for (int n = 0; n < p->n_nodes; n++) {
    if (!in(p->node_reqset[n], p->n_reqsets)) KP_BAD("node_reqset");
    if (p->node_taintset[n] < -1 || p->node_taintset[n] >= p->n_taintsets) KP_BAD("node_taintset");
    if (p->node_template && (p->node_template[n] < -1 || p->node_template[n] >= p->n_templates)) KP_BAD("node_template");
  }
  for (int64_t i = 0; i < p->n_running; i++)
    if (!in(p->run_class[i], p->n_classes) || !in(p->run_node[i], p->n_nodes)) KP_BAD("run_class / run_node");
  for (int m = 0; m < p->n_minvalue_keys; m++)
    if (!in(p->minvalue_key[m], p->n_keys)) KP_BAD("minvalue_key");
  if (p->n_minvalue_keys > 0 && !csr(p->minvalue_it_off, (int64_t)p->n_minvalue_keys * p->n_its, -1)) KP_BAD("minvalue_it_off");
#undef KP_BAD
  return KP_OK;
}

// ---- which shortcuts each class may take (ClassPlan), from the finished tables ----
static void plan_classes(const Ctx& c, HostTables& h) {
  const int K = h.K, N = h.N, X = h.X, X1 = std::max(X, 1);
  ClassPlan& pl = h.plan;
  pl = ClassPlan();
  // A key a NodeClaim does not define makes Compatible fail (requirements.go:181-197) until some pod with a NotIn /
  // DoesNotExist requirement defines it -- the one way CanAdd can flip from false to true for a topology-free pod.
  // It cannot happen for a row whose positive keys are all well-known (AllowUndefinedWellKnownLabels) or defined by
  // every NodePool template; only such rows get a permanent failure bit.
  auto row_monotone = [&](int rs) {
    for (int k = 0; k < K; k++) {
      const Slot s = c.rs_slot(rs, k);
      if (!slot_present(s) || op_is_negative(slot_op(s)) || h.key_wellknown[k]) continue;
      for (int n = 0; n < N; n++)
        if (!(h.rs_flags[(size_t)h.tmpl_rs[n] * K + k] & SF_PRESENT)) return false;
    }
    return true;
  };
  bool offerings_monotone = true;
  for (int dd = 0; dd < h.D; dd++) offerings_monotone = offerings_monotone && row_monotone(h.offset_rs[dd]);
  // set inclusion of requirement slots without bounds: values(a) within values(b)
  auto slot_subset = [&](int rs_a, int rs_b, int k) {
    const size_t ia = (size_t)rs_a * K + k, ib = (size_t)rs_b * K + k;
    const bool ac = h.rs_flags[ia] & SF_COMPLEMENT, bc = h.rs_flags[ib] & SF_COMPLEMENT;
    const uint64_t am = h.rs_mask[ia], bm = h.rs_mask[ib];
    if (!ac && !bc) return (am & ~bm) == 0;
    if (!ac && bc) return (am & bm) == 0;
    if (ac && bc) return (bm & ~am) == 0;
    return false;
  };
  // TopologyNodeFilter.Matches (topologynodefilter.go:68-97) holds for every claim whose requirements the class's
  // own requirement set leaves unchanged: some alternative is empty, or constrains only keys the class constrains
  // at least as tightly
  auto filter_implied = [&](int x, const KpGroup& G) {
    for (int a = 0; a < G.filter_n; a++) {
      const int rs = h.filter_rs[G.filter_off + a];
      bool ok = true;
      for (int k = 0; k < K && ok; k++) {
        if (!(h.rs_flags[(size_t)rs * K + k] & SF_PRESENT)) continue;
        ok = (h.rs_flags[(size_t)h.cls_rs[x] * K + k] & SF_PRESENT) && slot_subset(h.cls_rs[x], rs, k);
      }
      if (ok) return true;
    }
    return false;
  };
  {  // the topology key of the domain fast path: the non-hostname key most groups sit on
    std::vector<int> per_key(std::max(K, 1), 0);
    for (int g = 0; g < h.G; g++)
      if (h.groups[g].key != h.hostname_key && h.groups[g].key >= 0) per_key[h.groups[g].key]++;
    for (int k = 0; k < K; k++)
      if (per_key[k] > 0 && (pl.tk_key < 0 || per_key[k] > per_key[pl.tk_key])) pl.tk_key = k;
  }
  // can a pod ever define a new key on an existing node? (negative requirement on an undefined key, or a topology
  // domain choice) -- if not, an undefined key fails the strict Compatible of existingnode.go:89 forever
  bool nodes_gain_keys = false;
  for (int g = 0; g < h.G; g++) nodes_gain_keys = nodes_gain_keys || h.groups[g].key != h.hostname_key;
  for (int x = 0; x < X; x++)
    for (int k = 0; k < K; k++) {
      const Slot s = c.rs_slot(h.cls_rs[x], k);
      if (slot_present(s) && op_is_negative(slot_op(s))) nodes_gain_keys = true;
    }
  pl.strict_undefined = !nodes_gain_keys;
  // classes of a volume-alternative chain: the candidate loop tries the chain on every candidate, so nothing a single
  // requirement set says about a candidate may be cached (signatures, shortcut flags), and every node is a candidate
  pl.chain.assign(X1, 0);
  for (int x = 0; x < X; x++)
    if (h.cls_vol_next[x] >= 0) pl.chain[x] = pl.chain[h.cls_vol_next[x]] = 1;
  // the domain fast path re-checks no bound, group birth, Strict minValues or reservation
  bool lazy = false;
  for (int32_t b : h.g_born) lazy = lazy || b == 0;
  const bool fp_global = !h.has_bounds && !lazy && !h.min_values_strict && h.n_rsv == 0;
  pl.fsig.assign(X1, -1);
  pl.asig.assign(X1, 0);
  pl.fast.assign(X1, 0);
  pl.fp.assign(X1, 0);
  pl.has_tk.assign(X1, 0);
  pl.tok.assign(X1, 0);
  pl.nsig.assign(X1, 0);
  pl.rank.assign(X1, 0);
  pl.hchk_off.assign(X + 1, 0);
  std::map<int, int> fsigs, asigs;
  std::map<std::pair<int, int>, int> nsigs;
  for (int x = 0; x < X; x++) {
    const int rs = h.cls_rs[x];
    const int moff = h.cls_match_off[x], mend = h.cls_match_off[x + 1], roff = h.cls_rec_off[x], rend = h.cls_rec_off[x + 1];
    pl.asig[x] = asigs.emplace(rs, (int)asigs.size()).first->second;
    if (!pl.chain[x] && mend == moff && offerings_monotone && row_monotone(rs)) {
      pl.fsig[x] = fsigs.emplace(rs, (int)fsigs.size()).first->second;  // failure bits record requirement incompatibility only
      // the accepted-signature fast path: topology-free, counted by no group, nothing to re-check on the type list
      pl.fast[x] = rend == roff && !h.min_values_strict && h.n_rsv == 0;
    }
    // the domain fast path: every group that constrains or counts the class sits on the hostname key or on tk_key, and
    // none needs the node filter's requirement check at record time
    bool fp = fp_global && !pl.chain[x] && mend + rend > moff + roff, has_tk = false;
    for (int i = moff; i < mend && fp; i++) {
      const KpGroup& G = h.groups[h.cls_match[i] & 0x3fffffff];
      if (G.key == pl.tk_key)
        has_tk = true;
      else if (G.key != h.hostname_key)
        fp = false;
    }
    for (int i = roff; i < rend && fp; i++) {
      const KpGroup& G = h.groups[h.cls_rec[i]];
      if (G.key == pl.tk_key)
        has_tk = true;
      else if (G.key != h.hostname_key)
        fp = false;
      if (fp && !G.inverse && G.affinity_policy == 1 && G.filter_n > 0 && !filter_implied(x, G)) fp = false;
    }
    pl.fp[x] = fp;
    pl.has_tk[x] = fp && has_tk;
    for (int n = 0; n < std::min(N, 64); n++) {
      const int ts = h.tmpl_taintset[n];
      if (ts < 0 || h.n_taintsets == 0 || h.tol_ok[(size_t)(h.cls_tolset[x] + 1) * h.n_taintsets + ts]) pl.tok[x] |= 1ull << n;
    }
    const auto key = std::make_pair(pl.chain[x] ? -1 : rs, h.cls_tolset[x]);
    auto it = nsigs.find(key);
    if (it == nsigs.end()) {
      it = nsigs.emplace(key, (int)nsigs.size()).first;
      pl.nsig_rs.push_back(key.first);
      pl.nsig_tolset.push_back(key.second);
    }
    pl.nsig[x] = it->second;
    for (int i = moff; i < mend; i++) {
      const int e = h.cls_match[i], g = e & 0x3fffffff;
      const KpGroup& G = h.groups[g];
      if (G.key == h.hostname_key) pl.hchk.push_back(HostCheck{G.host_row, G.type, (e >> 30) & 1, G.max_skew, g});
    }
    pl.hchk_off[x + 1] = (int)pl.hchk.size();
  }
  pl.n_fsig = (int)fsigs.size();
  pl.n_asig = (int)asigs.size();
  std::vector<int> idx(X);
  for (int x = 0; x < X; x++) idx[x] = x;
  auto rank_key = [&](int x) { return std::make_pair(-h.cls_sort_cpu[x], -h.cls_sort_mem[x]); };
  std::sort(idx.begin(), idx.end(), [&](int a, int b) { return rank_key(a) < rank_key(b); });
  for (int i = 0, r = -1; i < X; i++) {
    if (i == 0 || rank_key(idx[i]) != rank_key(idx[i - 1])) r++;
    pl.rank[idx[i]] = r;
  }
}

int kp_prepare(const kp_problem* p, const std::vector<uint8_t>& node_active,
               const std::vector<std::pair<int, int>>& extra_bound, const std::vector<int32_t>& pending_classes,
               HostTables& h, std::string& err) {
  {
    int rc = validate_problem(p, err);
    if (rc != KP_OK) return rc;
  }
  Ctx c(p, h);
  const int K = p->n_keys, R = p->n_resources, T = p->n_its, N = p->n_templates, X = p->n_classes, E = p->n_nodes;
  if (K > KP_MAXK) return err = "more than 32 active label keys", KP_ERR_CAPACITY;
  if (R > KP_MAXR || R < 1) return err = "resource count out of range", KP_ERR_CAPACITY;
  const int ITW = (T + 63) / 64;
  if (ITW > KP_MAX_ITW) return err = "more than 2048 instance types", KP_ERR_CAPACITY;
  // reserved offerings run through the ReservationManager (reservationmanager.go:28-110): every one needs its id
  h.n_rsv = 0;
  h.rsv_strict = p->reserved_offering_strict != 0;
  if (p->off_reserved) {
    bool any = false;
    for (int t = 0; t < T; t++)
      for (int o = p->it_off_off[t]; o < p->it_off_off[t + 1]; o++) any = any || p->off_reserved[o];
    if (any) {
      if (!p->off_reservation_id || !p->off_reservation_capacity || p->n_reservations <= 0)
        return err = "reserved offerings need off_reservation_id / off_reservation_capacity / n_reservations", KP_ERR_INVALID;
      if (p->n_reservations > 64) return err = "more than 64 capacity reservations", KP_ERR_CAPACITY;
      h.n_rsv = p->n_reservations;
      h.rsv_cap0.assign(h.n_rsv, -1);
      for (int t = 0; t < T; t++)
        for (int o = p->it_off_off[t]; o < p->it_off_off[t + 1]; o++) {
          if (!p->off_reserved[o]) continue;
          const int id = p->off_reservation_id[o];
          if (id < 0 || id >= h.n_rsv) return err = "off_reservation_id out of range", KP_ERR_INVALID;
          const int cap = p->off_reservation_capacity[o];  // NewReservationManager keeps the smallest (:38-47)
          if (h.rsv_cap0[id] < 0 || h.rsv_cap0[id] > cap) h.rsv_cap0[id] = cap;
        }
      for (int32_t& v : h.rsv_cap0)
        if (v < 0) v = 0;
    }
  }
  h.K = K;
  h.R = R;
  h.T = T;
  h.ITW = ITW;
  h.N = N;
  h.X = X;
  h.E = E;
  for (int k = 0; k < K; k++)
    if (p->key_flags[k] & KP_KEY_HOSTNAME) h.hostname_key = k;
  for (int r = 0; r < R; r++) {
    if (p->res_flags[r] & KP_RES_NODES) h.nodes_res = r;
    if (p->res_flags[r] & KP_RES_CPU) h.cpu_res = r;
    if (p->res_flags[r] & KP_RES_MEMORY) h.mem_res = r;
  }
  // ---- key universe ----
  h.key_wellknown.assign(K, 0);
  h.key_univ.assign(K, 0);
  h.val_isint.assign(K, 0);
  h.val_int.assign((size_t)K * 64, 0);
  for (int k = 0; k < K; k++) {
    h.key_wellknown[k] = (p->key_flags[k] & KP_KEY_WELL_KNOWN) ? 1 : 0;
    if (k == h.hostname_key) continue;
    int nv = p->key_value_off[k + 1] - p->key_value_off[k];
    if (nv > 64) return err = "a label key has more than 64 distinct values", KP_ERR_CAPACITY;
    h.key_univ[k] = nv == 64 ? ~0ull : ((1ull << nv) - 1);
    for (int v = 0; v < nv; v++) {
      int idx = p->key_value_off[k] + v;
      if (p->value_is_int[idx]) {
        h.val_isint[k] |= 1ull << v;
        h.val_int[(size_t)k * 64 + v] = p->value_int[idx];
      }
    }
  }
  // ---- requirement sets -> slot rows (entries repeating a key fold with Requirements.Add) ----
  h.n_reqsets = p->n_reqsets;
  size_t nrs = (size_t)p->n_reqsets * K;
  h.rs_flags.assign(nrs ? nrs : 1, 0);
  h.rs_mask.assign(nrs ? nrs : 1, 0);
  h.rs_gte.assign(nrs ? nrs : 1, 0);
  h.rs_lte.assign(nrs ? nrs : 1, 0);
  h.rs_keys.assign(p->n_reqsets ? p->n_reqsets : 1, 0);
  for (int s = 0; s < p->n_reqsets; s++) {
    for (int e = p->reqset_off[s]; e < p->reqset_off[s + 1]; e++) {
      int k = p->req_key[e];
      uint8_t f = p->req_flags[e];
      if (k == h.hostname_key) return err = "requirements on kubernetes.io/hostname are not supported yet", KP_ERR_UNSUPPORTED;
      Slot in;
      in.f = SF_PRESENT | ((f & KP_REQ_COMPLEMENT) ? SF_COMPLEMENT : 0) | ((f & KP_REQ_HAS_GTE) ? SF_HAS_GTE : 0) |
             ((f & KP_REQ_HAS_LTE) ? SF_HAS_LTE : 0);
      in.gte = (f & KP_REQ_HAS_GTE) ? p->req_gte[e] : 0;
      in.lte = (f & KP_REQ_HAS_LTE) ? p->req_lte[e] : 0;
      in.m = 0;
      for (int i = p->req_val_off[e]; i < p->req_val_off[e + 1]; i++) in.m |= 1ull << p->req_vals[i];
      if (f & (KP_REQ_HAS_GTE | KP_REQ_HAS_LTE)) h.has_bounds = 1;
      size_t i = (size_t)s * K + k;
      Slot cur{h.rs_flags[i], h.rs_mask[i], h.rs_gte[i], h.rs_lte[i]};
      Slot out = slot_add(c.ki(k), cur, in);
      h.rs_flags[i] = (uint8_t)out.f;
      h.rs_mask[i] = out.m;
      h.rs_gte[i] = out.gte;
      h.rs_lte[i] = out.lte;
      h.rs_keys[s] |= 1u << k;
    }
  }
  // ---- taints ----
  h.n_taintsets = p->n_taintsets;
  h.n_tolsets = p->n_tolsets;
  h.tol_ok.assign((size_t)(p->n_tolsets + 1) * std::max(1, p->n_taintsets), 0);
  for (int a = -1; a < p->n_tolsets; a++)
    for (int b = 0; b < p->n_taintsets; b++) h.tol_ok[(size_t)(a + 1) * p->n_taintsets + b] = c.tolerates(b, a);
  // ---- instance types ----
  h.itv_off.assign(K + 1, 0);
  for (int k = 0; k < K; k++)
    h.itv_off[k + 1] = h.itv_off[k] + (k == h.hostname_key ? 0 : p->key_value_off[k + 1] - p->key_value_off[k]);
  h.itv.assign((size_t)std::max(h.itv_off[K], 1) * ITW, 0);
  h.it_nokey.assign((size_t)K * ITW, 0);
  h.it_dne.assign((size_t)K * ITW, 0);
  h.it_nonempty.assign((size_t)K * ITW, 0);
  h.it_valid.assign(ITW ? ITW : 1, 0);
  h.it_alloc.assign((size_t)T * R, 0);
  h.it_capacity.assign((size_t)T * R, 0);
  for (int t = 0; t < T; t++) {
    int w = t >> 6;
    uint64_t bit = 1ull << (t & 63);
    int rs = p->it_reqset[t];
    for (int k = 0; k < K; k++) {
      Slot s = c.rs_slot(rs, k);
      if (!slot_present(s)) {
        h.it_nokey[(size_t)k * ITW + w] |= bit;
        continue;
      }
      if (s.f & (SF_COMPLEMENT | SF_HAS_GTE | SF_HAS_LTE))
        return err = "instance types with NotIn/Exists/Gt/Lt requirements are not supported yet", KP_ERR_UNSUPPORTED;
      if (!s.m) {
        h.it_dne[(size_t)k * ITW + w] |= bit;
        continue;
      }
      h.it_nonempty[(size_t)k * ITW + w] |= bit;
      for (int v = 0; v < 64; v++)
        if (s.m >> v & 1) h.itv[((size_t)h.itv_off[k] + v) * ITW + w] |= bit;
    }
    // Allocatable (types.go:198-216)
    uint32_t cp = p->it_cap_present ? p->it_cap_present[t] : ((1u << R) - 1);
    bool neg = false;
    int64_t alloc[KP_MAXR];
    for (int r = 0; r < R; r++) {
      int64_t cap = (cp >> r & 1) ? p->it_capacity[(size_t)t * R + r] : 0;
      h.it_capacity[(size_t)t * R + r] = cap;
      alloc[r] = (cp >> r & 1) ? cap - (p->it_overhead ? p->it_overhead[(size_t)t * R + r] : 0) : 0;
    }
    for (int r = 0; r < R; r++)
      if ((cp >> r & 1) && (p->res_flags[r] & KP_RES_HUGEPAGES) && h.mem_res >= 0) {
        alloc[h.mem_res] -= p->it_capacity[(size_t)t * R + r];
        if (alloc[h.mem_res] < 0) alloc[h.mem_res] = 0;
      }
    for (int r = 0; r < R; r++) {
      h.it_alloc[(size_t)t * R + r] = alloc[r];
      if (alloc[r] < 0) neg = true;  // Fits: a negative total never fits (resources.go:151-156)
    }
    if (!neg) h.it_valid[w] |= bit;
  }
  // ">= threshold" tables per resource (rows of all resources concatenated)
  h.ge_off.assign(R + 1, 0);
  h.ge_vals.clear();
  h.ge_bits.clear();
  for (int r = 0; r < R; r++) {
    std::vector<int64_t> vals;
    for (int t = 0; t < T; t++) vals.push_back(h.it_alloc[(size_t)t * R + r]);
    std::sort(vals.begin(), vals.end());
    vals.erase(std::unique(vals.begin(), vals.end()), vals.end());
    for (size_t j = 0; j < vals.size(); j++) {
      h.ge_vals.push_back(vals[j]);
      size_t base = h.ge_bits.size();
      h.ge_bits.resize(base + ITW, 0);
      for (int t = 0; t < T; t++)
        if (h.it_alloc[(size_t)t * R + r] >= vals[j]) h.ge_bits[base + (t >> 6)] |= 1ull << (t & 63);
    }
    h.ge_off[r + 1] = (int)h.ge_vals.size();
  }
  if (h.ge_vals.empty()) {
    h.ge_vals.push_back(0);
    h.ge_bits.assign(std::max(ITW, 1), 0);
  }
  // distinct offering requirement sets (by content of their slot rows)
  {
    std::map<std::string, int> seen;
    for (int t = 0; t < T; t++)
      for (int o = p->it_off_off[t]; o < p->it_off_off[t + 1]; o++) {
        int rs = p->off_reqset[o];
        // a distinct set = (requirements, reservation id): every set has at most one reservation behind it
        const int32_t rid = (h.n_rsv > 0 && p->off_reserved[o]) ? p->off_reservation_id[o] : -1;
        std::string key((const char*)&h.rs_flags[(size_t)rs * K], K);
        key.append((const char*)&rid, 4);
        key.append((const char*)&h.rs_mask[(size_t)rs * K], K * 8);
        key.append((const char*)&h.rs_gte[(size_t)rs * K], K * 8);
        key.append((const char*)&h.rs_lte[(size_t)rs * K], K * 8);
        auto it = seen.find(key);
        int d;
        if (it == seen.end()) {
          d = (int)h.offset_rs.size();
          if (d >= KP_MAX_OFFSETS) return err = "more than 32 distinct offering requirement sets", KP_ERR_CAPACITY;
          seen[key] = d;
          h.offset_rs.push_back(rs);
          h.set_rsv.push_back(rid);
          h.offset_bits.resize((size_t)(d + 1) * ITW, 0);
        } else {
          d = it->second;
        }
        if ((int)h.off_set.size() <= o) h.off_set.resize(o + 1, 0);
        h.off_set[o] = d;
        if (p->off_available[o]) h.offset_bits[(size_t)d * ITW + (t >> 6)] |= 1ull << (t & 63);
      }
    h.D = (int)h.offset_rs.size();
    if (h.off_set.empty()) h.off_set.push_back(0);
    if (h.offset_rs.empty()) {
      h.offset_rs.push_back(0);
      h.offset_bits.assign(std::max(ITW, 1), 0);
    }
    h.off_slots.assign((size_t)std::max(h.D, 1) * K, Slot{0u, 0ull, 0, 0});
    h.off_keys.assign(std::max(h.D, 1), 0);
    for (int dd = 0; dd < h.D; dd++) {
      h.off_keys[dd] = h.rs_keys[h.offset_rs[dd]];
      for (int k = 0; k < K; k++) h.off_slots[(size_t)dd * K + k] = c.rs_slot(h.offset_rs[dd], k);
    }
  }
  // ---- templates ----
  h.tmpl_rs.assign(p->tmpl_reqset, p->tmpl_reqset + N);
  h.tmpl_taintset.assign(p->tmpl_taintset, p->tmpl_taintset + N);
  h.tmpl_its_raw.assign((size_t)std::max(N, 1) * std::max(ITW, 1), 0);
  h.tmpl_daemon.assign((size_t)std::max(N, 1) * R, 0);
  h.tmpl_remaining.assign((size_t)std::max(N, 1) * R, 0);
  h.tmpl_limit_present.assign(std::max(N, 1), 0);
  for (int n = 0; n < N; n++) {
    for (int i = p->tmpl_it_off[n]; i < p->tmpl_it_off[n + 1]; i++) {
      int t = p->tmpl_its[i];
      h.tmpl_its_raw[(size_t)n * ITW + (t >> 6)] |= 1ull << (t & 63);
    }
    for (int r = 0; r < R; r++) {
      if (p->tmpl_daemon) h.tmpl_daemon[(size_t)n * R + r] = p->tmpl_daemon[(size_t)n * R + r];
      if (p->tmpl_limits) h.tmpl_remaining[(size_t)n * R + r] = p->tmpl_limits[(size_t)n * R + r];
    }
    h.tmpl_limit_present[n] = p->tmpl_limit_present ? p->tmpl_limit_present[n] : 0;
  }
  // ---- minValues (cloudprovider/types.go:301-337) ----
  // Only NodePool requirements can carry minValues (pods have none), and Requirements.Add keeps the larger one
  // (requirement.go:180), so a NodeClaim's minValues are its template's.  Per key with minValues: one instance-type
  // bitmap per distinct value; SatisfiesMinValues == "at least `need` of those bitmaps meet the remaining types".
  h.tmpl_mv_off.assign(1, 0);
  h.mv_val_off.assign(1, 0);
  {
    const int M = p->n_minvalue_keys;
    for (int m = 0; m < M; m++) {
      std::map<int32_t, int> dense;
      size_t base = h.mv_masks.size();
      for (int t = 0; t < T; t++) {
        size_t row = (size_t)m * T + t;
        for (int i = p->minvalue_it_off[row]; i < p->minvalue_it_off[row + 1]; i++) {
          auto ins = dense.emplace(p->minvalue_it_vals[i], (int)dense.size());
          if (ins.second) h.mv_masks.resize(h.mv_masks.size() + std::max(ITW, 1), 0);
          h.mv_masks[base + (size_t)ins.first->second * ITW + (t >> 6)] |= 1ull << (t & 63);
        }
      }
      h.mv_val_off.push_back(h.mv_val_off.back() + (int)dense.size());
    }
    for (int n = 0; n < N; n++) {
      std::map<int, int> need;  // key -> minValues
      int s = p->tmpl_reqset[n];
      for (int e = p->reqset_off[s]; e < p->reqset_off[s + 1]; e++)
        if (p->req_flags[e] & KP_REQ_HAS_MINVALUES) {
          int& v = need[p->req_key[e]];
          v = std::max(v, p->req_min_values[e]);
        }
      for (auto& kv : need) {
        int m = -1;
        for (int i = 0; i < M; i++)
          if (p->minvalue_key[i] == kv.first) m = i;
        if (m < 0) {  // no table for the key: no instance type offers a value (Get(key).Values() is empty everywhere)
          if (kv.second > 0) m = M;  // sentinel: an empty value range, never satisfiable
          else continue;
        }
        h.tmpl_mv_key.push_back(m);
        h.tmpl_mv_need.push_back(kv.second);
        h.has_min_values = true;
      }
      h.tmpl_mv_off.push_back((int)h.tmpl_mv_key.size());
    }
    h.mv_val_off.push_back(h.mv_val_off.back());  // the sentinel's empty range
    if (h.mv_masks.empty()) h.mv_masks.assign(1, 0);
    if (h.tmpl_mv_key.empty()) {
      h.tmpl_mv_key.assign(1, 0);
      h.tmpl_mv_need.assign(1, 0);
    }
    // minValues on any other requirement set (a pod, an instance type) has no meaning in the reference's API
    for (int s = 0; s < p->n_reqsets; s++) {
      bool is_tmpl = false;
      for (int n = 0; n < N; n++) is_tmpl |= p->tmpl_reqset[n] == s;
      if (is_tmpl) continue;
      for (int e = p->reqset_off[s]; e < p->reqset_off[s + 1]; e++)
        if (p->req_flags[e] & KP_REQ_HAS_MINVALUES)
          return err = "minValues outside NodePool requirements", KP_ERR_INVALID;
    }
  }
  h.min_values_strict = h.has_min_values && !p->min_values_best_effort;
  // ---- existing nodes ----
  h.node_taintset.assign(std::max(E, 1), -1);
  h.node_flags.assign(std::max(E, 1), 0);
  h.node_rem.assign((size_t)std::max(E, 1) * R, 0);
  h.node_rem_present.assign(std::max(E, 1), 0);
  h.node_sflags.assign((size_t)std::max(E, 1) * K, 0);
  h.node_smask.assign((size_t)std::max(E, 1) * K, 0);
  h.node_sgte.assign((size_t)std::max(E, 1) * K, 0);
  h.node_slte.assign((size_t)std::max(E, 1) * K, 0);
  std::map<int, int> host_to_node;
  for (int i = 0; i < E; i++) {
    h.node_taintset[i] = p->node_taintset[i];
    h.node_flags[i] = (uint8_t)((p->node_flags[i] & ~KP_NODE_SCHEDULABLE) | (node_active[i] ? KP_NODE_SCHEDULABLE : 0));
    h.node_rem_present[i] = p->node_avail_present ? p->node_avail_present[i] : ((1u << R) - 1);
    for (int r = 0; r < R; r++) h.node_rem[(size_t)i * R + r] = p->node_available[(size_t)i * R + r];
    int rs = p->node_reqset[i];
    for (int k = 0; k < K; k++) {
      Slot s = c.rs_slot(rs, k);
      h.node_sflags[(size_t)i * K + k] = (uint8_t)s.f;
      h.node_smask[(size_t)i * K + k] = s.m;
      h.node_sgte[(size_t)i * K + k] = s.gte;
      h.node_slte[(size_t)i * K + k] = s.lte;
    }
    host_to_node[p->node_hostname[i]] = i;
    int t = p->node_template ? p->node_template[i] : -1;  // updateRemainingResources (scheduler.go:728-735)
    if (node_active[i] && t >= 0 && p->node_capacity)
      for (int r = 0; r < R; r++)
        if (h.tmpl_limit_present[t] >> r & 1) h.tmpl_remaining[(size_t)t * R + r] -= p->node_capacity[(size_t)i * R + r];
  }
  // ---- classes ----
  h.cls_req.assign(p->class_requests, p->class_requests + (size_t)X * R);
  h.cls_rs.assign(p->class_reqset, p->class_reqset + X);
  h.cls_strict_rs.assign(p->class_strict_reqset, p->class_strict_reqset + X);
  h.cls_tolset.assign(p->class_tolset, p->class_tolset + X);
  h.cls_vol_next.assign(std::max(X, 1), -1);
  if (p->class_vol_next)
    for (int x = 0; x < X; x++) {
      h.cls_vol_next[x] = p->class_vol_next[x];
      h.has_vol_alts = h.has_vol_alts || p->class_vol_next[x] >= 0;
    }
  h.cls_relax.assign(std::max(X, 1), -1);
  if (p->class_relax_next)
    for (int x = 0; x < X; x++) h.cls_relax[x] = p->class_relax_next[x];
  h.cls_rv.assign(std::max(X, 1), 0);
  h.cls_sort_cpu.assign(std::max(X, 1), 0);
  h.cls_sort_mem.assign(std::max(X, 1), 0);
  {
    std::map<std::vector<int64_t>, int> rv;
    for (int x = 0; x < X; x++) {
      std::vector<int64_t> v(p->class_requests + (size_t)x * R, p->class_requests + (size_t)(x + 1) * R);
      auto it = rv.find(v);
      if (it == rv.end()) it = rv.emplace(v, (int)rv.size()).first;
      h.cls_rv[x] = it->second;
      h.cls_sort_cpu[x] = h.cpu_res >= 0 ? v[h.cpu_res] : 0;
      h.cls_sort_mem[x] = h.mem_res >= 0 ? v[h.mem_res] : 0;
    }
    h.n_rv = (int)std::max<size_t>(rv.size(), 1);
  }

  // ---- topology (NewTopology, topology.go:68-103) ----
  // domain universe per key (buildDomainGroups, topology.go:105-143): value -> taint sets it is reachable under
  std::vector<std::map<int, std::vector<int>>> universe(K);
  auto dg_insert = [&](int k, int v, int ts) {
    auto& d = universe[k];
    bool empty = c.taintset_size(ts) == 0;
    auto it = d.find(v);
    if (it == d.end() || empty) {
      d[v] = {ts};
      return;
    }
    if (c.taintset_size(it->second[0]) == 0) return;
    it->second.push_back(ts);
  };
  for (int n = 0; n < N; n++) {
    int trs = p->tmpl_reqset[n], ts = p->tmpl_taintset[n];
    // distinct instance-type requirement sets only: the universe is a set union
    std::set<int> it_sets;
    for (int i = p->tmpl_it_off[n]; i < p->tmpl_it_off[n + 1]; i++) it_sets.insert(p->it_reqset[p->tmpl_its[i]]);
    for (int irs : it_sets)
      for (int k = 0; k < K; k++) {
        Slot m = slot_add(c.ki(k), c.rs_slot(trs, k), c.rs_slot(irs, k));
        if (!slot_present(m)) continue;
        for (int v = 0; v < 64; v++)
          if (m.m >> v & 1) dg_insert(k, v, ts);
      }
    for (int k = 0; k < K; k++) {
      Slot s = c.rs_slot(trs, k);
      if (slot_present(s) && slot_op(s) == OP_IN)
        for (int v = 0; v < 64; v++)
          if (s.m >> v & 1) dg_insert(k, v, ts);
    }
  }
  // all bound pods: (class, node)
  std::vector<std::pair<int, int>> bound;
  for (int64_t i = 0; i < p->n_running; i++) bound.push_back({p->run_class[i], p->run_node[i]});
  bound.insert(bound.end(), extra_bound.begin(), extra_bound.end());

  std::vector<HGroup> regular, inverse;
  std::map<std::string, int> reg_index, inv_index;
  auto node_slot = [&](int node, int k) {
    size_t i = (size_t)node * K + k;
    return Slot{h.node_sflags[i], h.node_smask[i], h.node_sgte[i], h.node_slte[i]};
  };
  auto filter_matches = [&](const HGroup& g, int taintset, auto slot_of) {
    bool aff = true;
    if (g.g.affinity_policy == 1 && !g.filter.empty()) {
      aff = false;
      for (int rs : g.filter)
        if (c.rows_compatible(slot_of, [&](int k) { return c.rs_slot(rs, k); }, false)) {
          aff = true;
          break;
        }
    }
    bool tnt = true;
    if (g.g.taint_policy == 1) tnt = c.tolerates(taintset, g.g.tolset);
    return aff && tnt;
  };
  auto make_group = [&](int cls, int ci, bool inv) {
    HGroup g;
    g.g.type = p->tsc_type[ci];
    g.g.key = p->tsc_key[ci];
    g.g.inverse = inv;
    g.nsset = p->tsc_nsset[ci];
    g.selector = p->tsc_selector[ci];
    g.g.tolset = -1;
    g.g.host_row = -1;
    if (g.g.type == KP_TOPO_SPREAD) {
      g.g.max_skew = p->tsc_max_skew[ci];
      g.g.min_domains = p->tsc_min_domains[ci];
      g.g.taint_policy = p->tsc_taint_policy[ci] ? 1 : 0;
      g.g.affinity_policy = p->tsc_affinity_policy[ci] ? 1 : 0;
      g.g.tolset = p->class_tolset[cls];
      for (int i = p->class_filter_off[cls]; i < p->class_filter_off[cls + 1]; i++)
        g.filter.push_back(p->class_filter_reqsets[i]);
    } else {
      g.g.max_skew = INT32_MAX;
      g.g.min_domains = -1;
      g.g.taint_policy = 2;
      g.g.affinity_policy = 2;
    }
    // initial domains (ForEachDomain, topologydomaingroup.go:56-72)
    if (g.g.key != h.hostname_key)
      for (auto& kv : universe[g.g.key]) {
        bool take = g.g.taint_policy == 0;
        if (!take)
          for (int ts : kv.second)
            if (c.tolerates(ts, p->class_tolset[cls])) {
              take = true;
              break;
            }
        if (take) g.reg |= 1ull << kv.first;
      }
    return g;
  };
  auto hash_of = [&](const HGroup& g) {
    std::ostringstream o;
    o << g.g.key << "|" << g.g.type << "|" << g.g.max_skew << "|";
    std::set<int> ns(p->nsset_ids + p->nsset_off[g.nsset], p->nsset_ids + p->nsset_off[g.nsset + 1]);
    for (int x : ns) o << x << ",";
    o << "|" << g.g.taint_policy << g.g.affinity_policy << "|";
    std::set<std::string> rs;
    for (int r : g.filter) {
      std::string s((const char*)&h.rs_flags[(size_t)r * K], K);
      s.append((const char*)&h.rs_mask[(size_t)r * K], K * 8);
      s.append((const char*)&h.rs_gte[(size_t)r * K], K * 8);
      s.append((const char*)&h.rs_lte[(size_t)r * K], K * 8);
      rs.insert(s);
    }
    for (auto& s : rs) o << s << "#";
    o << "|";
    if (g.g.tolset >= 0) {
      std::set<std::string> ts;
      for (int j = p->tolset_off[g.g.tolset]; j < p->tolset_off[g.g.tolset + 1]; j++) {
        int t = p->tolset_ids[j];
        std::ostringstream q;
        q << p->tol_key[t] << "/" << (int)p->tol_op[t] << "/" << p->tol_value[t] << "/" << (int)p->tol_effect[t];
        ts.insert(q.str());
      }
      for (auto& s : ts) o << s << ",";
    }
    o << "|";
    if (g.selector < 0)
      o << "nil";
    else {
      std::set<std::string> ex;
      for (int e = p->selector_off[g.selector]; e < p->selector_off[g.selector + 1]; e++) {
        std::ostringstream q;
        q << p->selx_key[e] << "/" << (int)p->selx_op[e] << "/";
        std::set<int> vs(p->selx_vals + p->selx_val_off[e], p->selx_vals + p->selx_val_off[e + 1]);
        for (int v : vs) q << v << ",";
        ex.insert(q.str());
      }
      for (auto& s : ex) o << s << ";";
    }
    return o.str();
  };
  // domain of a node for a topology key: label value, or the node itself for hostname (topology.go:405-415)
  auto node_domain = [&](int node, int key, int* out) {
    if (key == h.hostname_key) {
      *out = node;
      return true;
    }
    Slot s = node_slot(node, key);
    if (!slot_present(s) || (s.f & SF_COMPLEMENT) || !s.m) return false;
    *out = __builtin_ctzll(s.m);
    return true;
  };
  auto group_record = [&](HGroup& g, int domain) {
    if (g.g.key == h.hostname_key) {
      g.host_cnt[domain]++;
      g.host_reg.insert(domain);
    } else {
      g.cnt[domain]++;
      g.reg |= 1ull << domain;
    }
  };
  auto group_register = [&](HGroup& g, int domain) {
    if (g.g.key == h.hostname_key)
      g.host_reg.insert(domain);
    else
      g.reg |= 1ull << domain;
  };
  // updateInverseAntiAffinity (topology.go:297-322)
  auto update_inverse = [&](int cls, int node) {
    for (int ci = p->class_tsc_off[cls]; ci < p->class_tsc_off[cls + 1]; ci++) {
      if (p->tsc_type[ci] != KP_TOPO_ANTI_AFFINITY) continue;
      if (p->tsc_preferred && p->tsc_preferred[ci]) continue;  // required terms only (topology.go:297-322)
      HGroup g = make_group(cls, ci, true);
      std::string hk = hash_of(g);
      auto it = inv_index.find(hk);
      int gi;
      if (it == inv_index.end()) {
        gi = (int)inverse.size();
        inv_index[hk] = gi;
        inverse.push_back(std::move(g));
      } else {
        gi = it->second;
      }
      if (node >= 0) {
        int d;
        if (node_domain(node, inverse[gi].g.key, &d)) group_record(inverse[gi], d);
      }
      inverse[gi].owners.insert(cls);
    }
  };
  for (auto& bp : bound) update_inverse(bp.first, bp.second);
  // Update (topology.go:162-194) per pending pod, class-level (every pod of a class carries the same constraints)
  std::vector<uint8_t> seen_cls(std::max(X, 1), 0);
  // A pod that fails is retried as its relaxed class (Preferences.Relax, preferences.go:38-57) after a Topology.Update
  // of the relaxed pod.  The relaxed classes are made owners of their groups up front, behind the pending classes.
  // A group only relaxed classes own is one the reference creates in the middle of the solve (the relaxation changed
  // its identity: the node filter of a spread holds the pod's tolerations and required node-affinity terms,
  // topologynodefilter.go:30-64): it is built here with its cluster counts and marked lazy; the solver gives birth to
  // it when a pod is first tried as the relaxed class (KpDev::g_born).
  std::vector<int32_t> pending_closure;
  for (int cls0 : pending_classes)
    if (!seen_cls[cls0]) {
      seen_cls[cls0] = 1;
      pending_closure.push_back(cls0);
    }
  const size_t n_direct = pending_closure.size();
  if (p->class_relax_next)
    for (int x = 0; x < X; x++)
    {
      int steps = 0;
      for (int c = p->class_relax_next[x]; c >= 0; c = p->class_relax_next[c])
        if (c >= X || ++steps > X) return err = "class_relax_next out of range or cyclic", KP_ERR_INVALID;
    }
  for (size_t i = 0; i < n_direct; i++)
    for (int c = p->class_relax_next ? p->class_relax_next[pending_closure[i]] : -1; c >= 0 && !seen_cls[c];
         c = p->class_relax_next[c]) {
      seen_cls[c] = 1;
      pending_closure.push_back(c);
    }
  std::vector<std::vector<int>> cls_lazy(std::max(X, 1));
  for (size_t pi = 0; pi < pending_closure.size(); pi++) {
    const int cls = pending_closure[pi];
    bool anti = false;
    for (int ci = p->class_tsc_off[cls]; ci < p->class_tsc_off[cls + 1]; ci++)
      anti |= p->tsc_type[ci] == KP_TOPO_ANTI_AFFINITY && !(p->tsc_preferred && p->tsc_preferred[ci]);
    if (anti) update_inverse(cls, -1);
    for (int ci = p->class_tsc_off[cls]; ci < p->class_tsc_off[cls + 1]; ci++) {
      HGroup g = make_group(cls, ci, false);
      std::string hk = hash_of(g);
      auto it = reg_index.find(hk);
      int gi;
      if (it == reg_index.end()) {
        // countDomains (topology.go:328-426)
        for (int n = 0; n < E; n++) {
          if (!node_active[n]) continue;
          if (!filter_matches(g, p->node_taintset[n], [&](int k) { return node_slot(n, k); })) continue;
          int d;
          if (node_domain(n, g.g.key, &d)) group_register(g, d);
        }
        for (auto& bp : bound) {
          int bc = bp.first, node = bp.second;
          if (!c.nsset_has(g.nsset, p->class_namespace[bc])) continue;
          if (g.selector >= 0 && !c.selector_matches(g.selector, p->class_labelset[bc])) continue;
          int d;
          if (!node_domain(node, g.g.key, &d)) continue;
          if (!filter_matches(g, p->node_taintset[node], [&](int k) { return node_slot(node, k); })) continue;
          group_record(g, d);
        }
        g.lazy = pi >= n_direct;
        gi = (int)regular.size();
        reg_index[hk] = gi;
        regular.push_back(std::move(g));
      } else {
        gi = it->second;
      }
      regular[gi].owners.insert(cls);
      if (regular[gi].lazy && std::find(cls_lazy[cls].begin(), cls_lazy[cls].end(), gi) == cls_lazy[cls].end())
        cls_lazy[cls].push_back(gi);
    }
  }
  // NewExistingNode registers every schedulable node's hostname in every hostname group that exists when the
  // Scheduler is built (existingnode.go:64); a group born later only knows the nodes countDomains registered
  for (auto* vec : {&regular, &inverse})
    for (auto& g : *vec)
      if (g.g.key == h.hostname_key && !g.lazy)
        for (int n = 0; n < E; n++)
          if (node_active[n]) g.host_reg.insert(n);
  h.n_regular = (int)regular.size();
  h.cls_lazy_off.assign(1, 0);
  h.cls_lazy.clear();
  for (int x = 0; x < X; x++) {
    for (int gi : cls_lazy[x]) h.cls_lazy.push_back(gi);  // regular groups keep their index in the flattened table
    h.cls_lazy_off.push_back((int)h.cls_lazy.size());
  }
  if (X == 0) h.cls_lazy_off.push_back(0);
  if (h.cls_lazy.empty()) h.cls_lazy.push_back(0);

  // ---- flatten groups: regular first (creation order), then inverse ----
  int G = (int)(regular.size() + inverse.size());
  h.G = G;
  h.groups.resize(std::max(G, 1));
  h.dom_reg.assign(std::max(G, 1), 0);
  h.dom_pop.assign(std::max(G, 1), 0);
  h.g_ndomains.assign(std::max(G, 1), 0);
  h.g_nempty.assign(std::max(G, 1), 0);
  h.dom_cnt.assign((size_t)std::max(G, 1) * 64, 0);
  h.filter_rs.clear();
  int GH = 0;
  std::vector<HGroup*> all;
  for (auto& g : regular) all.push_back(&g);
  for (auto& g : inverse) all.push_back(&g);
  for (int gi = 0; gi < G; gi++) {
    HGroup& g = *all[gi];
    g.g.dom_off = gi * 64;
    g.g.filter_off = (int)h.filter_rs.size();
    g.g.filter_n = (int)g.filter.size();
    for (int r : g.filter) h.filter_rs.push_back(r);
    if (g.g.key == h.hostname_key) {
      g.g.host_row = GH++;
      h.g_ndomains[gi] = (int)g.host_reg.size();
      int pop = 0;
      for (auto& kv : g.host_cnt) pop += kv.second > 0;
      h.g_nempty[gi] = (int)g.host_reg.size() - pop;
    } else {
      h.dom_reg[gi] = g.reg;
      for (int v = 0; v < 64; v++) {
        h.dom_cnt[(size_t)gi * 64 + v] = g.cnt[v];
        if (g.cnt[v] > 0) h.dom_pop[gi] |= 1ull << v;
      }
      h.g_ndomains[gi] = __builtin_popcountll(g.reg);
      int pop = 0;
      for (int v = 0; v < 64; v++) pop += (g.reg >> v & 1) && g.cnt[v] > 0;
      h.g_nempty[gi] = h.g_ndomains[gi] - pop;
    }
    h.groups[gi] = g.g;
  }
  if (h.filter_rs.empty()) h.filter_rs.push_back(0);
  h.GH = GH;
  h.host_cnt_nodes.assign((size_t)std::max(GH, 1) * std::max(E, 1), 0);
  h.g_born.assign(std::max(G, 1), 1);
  h.g_birth.assign(std::max(G, 1), -1);
  for (int gi = 0; gi < G; gi++) {
    if (all[gi]->lazy) h.g_born[gi] = 0;
    if (all[gi]->g.host_row < 0) continue;
    int32_t* row = h.host_cnt_nodes.data() + (size_t)all[gi]->g.host_row * E;
    for (auto& kv : all[gi]->host_cnt) row[kv.first] = kv.second;
  }
  // per-class lists. selects(group, class) only depends on (labelset, namespace): evaluate per distinct pair, and
  // use the first In-expression of a selector to enumerate candidate pairs instead of scanning all of them.
  std::map<std::pair<int, int>, int> pair_id;
  std::vector<std::pair<int, int>> pairs;
  std::vector<int> cls_pair(std::max(X, 1), 0);
  for (int x = 0; x < X; x++) {
    auto key = std::make_pair(p->class_labelset[x], p->class_namespace[x]);
    auto it = pair_id.find(key);
    if (it == pair_id.end()) {
      it = pair_id.emplace(key, (int)pairs.size()).first;
      pairs.push_back(key);
    }
    cls_pair[x] = it->second;
  }
  std::map<std::pair<int, int>, std::vector<int>> label_index;  // (label key, value) -> pairs carrying it
  for (size_t q = 0; q < pairs.size(); q++) {
    int ls = pairs[q].first;
    if (ls < 0) continue;
    for (int i = p->labelset_off[ls]; i < p->labelset_off[ls + 1]; i++)
      label_index[{p->label_key[i], p->label_val[i]}].push_back((int)q);
  }
  std::vector<std::vector<int>> pair_sel(pairs.size());  // groups selecting the pair
  for (int gi = 0; gi < G; gi++) {
    HGroup& g = *all[gi];
    if (g.selector < 0) continue;
    int first_in = -1;
    for (int e = p->selector_off[g.selector]; e < p->selector_off[g.selector + 1] && first_in < 0; e++)
      if (p->selx_op[e] == KP_SEL_IN) first_in = e;
    std::vector<int> cand;
    if (first_in >= 0) {
      for (int i = p->selx_val_off[first_in]; i < p->selx_val_off[first_in + 1]; i++) {
        auto it = label_index.find({p->selx_key[first_in], p->selx_vals[i]});
        if (it != label_index.end()) cand.insert(cand.end(), it->second.begin(), it->second.end());
      }
      std::sort(cand.begin(), cand.end());
      cand.erase(std::unique(cand.begin(), cand.end()), cand.end());
    } else {
      for (size_t q = 0; q < pairs.size(); q++) cand.push_back((int)q);
    }
    for (int q : cand)
      if (c.nsset_has(g.nsset, pairs[q].second) && c.selector_matches(g.selector, pairs[q].first))
        pair_sel[q].push_back(gi);
  }
  std::vector<std::vector<int>> cls_owned(std::max(X, 1));
  for (int gi = 0; gi < G; gi++)
    for (int x : all[gi]->owners) cls_owned[x].push_back(gi);
  h.cls_match_off.assign(X + 1, 0);
  h.cls_rec_off.assign(X + 1, 0);
  h.cls_match.clear();
  h.cls_rec.clear();
  for (int x = 0; x < X; x++) {
    const std::vector<int>& sel = pair_sel[cls_pair[x]];
    auto selects_g = [&](int gi) { return std::binary_search(sel.begin(), sel.end(), gi); };
    // getMatchingTopologies (topology.go:528-541): owned regular groups, then inverse groups that count the pod.
    // bit 30 of an entry == TopologyGroup.selects(pod) ("self-selecting")
    for (int gi : cls_owned[x])
      if (!all[gi]->g.inverse) h.cls_match.push_back(gi | (selects_g(gi) ? (1 << 30) : 0));
    for (int gi : sel)
      if (all[gi]->g.inverse) h.cls_match.push_back(gi | (1 << 30));
    // Record (topology.go:197-220): regular groups that select the pod, inverse groups the pod owns
    for (int gi : sel)
      if (!all[gi]->g.inverse) h.cls_rec.push_back(gi);
    for (int gi : cls_owned[x])
      if (all[gi]->g.inverse) h.cls_rec.push_back(gi);
    h.cls_match_off[x + 1] = (int)h.cls_match.size();
    h.cls_rec_off[x + 1] = (int)h.cls_rec.size();
  }
  if (h.cls_match.empty()) h.cls_match.push_back(0);
  if (h.cls_rec.empty()) h.cls_rec.push_back(0);
  (void)host_to_node;
  plan_classes(c, h);
  return KP_OK;
}

// ---- price lists ----
// Appends one list: the available offerings o of instance type ti with keep(o), by price (stable: ties keep offering order)
template <class Keep>
static void add_list(PriceLists& l, const kp_problem* p, const HostTables& t, int ti, bool dearest_first, Keep keep) {
  std::vector<std::pair<double, int>> ent;
  for (int o = p->it_off_off[ti]; o < p->it_off_off[ti + 1]; o++)
    if (p->off_available[o] && keep(o)) ent.push_back({p->off_price[o], t.off_set[o]});
  std::stable_sort(ent.begin(), ent.end(), [&](const std::pair<double, int>& a, const std::pair<double, int>& b) {
    return dearest_first ? a.first > b.first : a.first < b.first;
  });
  for (auto& e : ent) {
    l.price.push_back(e.first);
    l.set.push_back(e.second);
  }
  l.off.push_back((int32_t)l.set.size());
}
static void pad(PriceLists& l) {
  if (l.set.empty()) {
    l.set.push_back(0);
    l.price.push_back(0);
  }
}

PriceLists order_by_price(const kp_problem* p, const HostTables& t) {
  PriceLists l;
  l.off.assign(1, 0);
  for (int ti = 0; ti < p->n_its; ti++) add_list(l, p, t, ti, false, [](int) { return true; });
  pad(l);
  return l;
}

ConsolPrices consol_prices(const kp_problem* p, const HostTables& t, const kp_consol_input* in) {
  const Ctx c(p, t);
  const int K = t.K;
  ConsolPrices cp;
  cp.node_price.assign(std::max(t.E, 1), -1.0);
  for (int n = 0; n < t.E; n++) {
    const int it = in->node_it[n];
    if (it < 0) continue;
    bool any = false;
    double best = 0;
    for (int o = p->it_off_off[it]; o < p->it_off_off[it + 1]; o++) {
      if (!c.rows_compatible([&](int k) { return c.rs_slot(p->node_reqset[n], k); }, [&](int k) { return c.rs_slot(p->off_reqset[o], k); }, true))
        continue;
      if (!any || p->off_price[o] < best) best = p->off_price[o];
      any = true;
    }
    if (any) cp.node_price[n] = best;
  }
  // bit i of a distinct offering set: compatible with capacity type i, in the order reserved, spot, on-demand
  // (types.go:480-491)
  const int ct_order[3] = {in->ct_reserved, in->ct_spot, in->ct_on_demand};
  std::vector<uint8_t> ctmask(std::max(t.D, 1), 0);
  for (int i = 0; i < 3; i++) {
    if (in->capacity_type_key < 0 || ct_order[i] < 0) continue;
    cp.ct_valid |= 1 << i;
    const Slot ct{SF_PRESENT, 1ull << ct_order[i], 0, 0}, none{0u, 0ull, 0, 0};
    for (int dd = 0; dd < t.D; dd++)
      if (c.rows_compatible([&](int k) { return k == in->capacity_type_key ? ct : none; },
                            [&](int k) { return t.off_slots[(size_t)dd * K + k]; }, true))
        ctmask[dd] |= 1 << i;
  }
  cp.worst.off.assign(1, 0);
  for (int ti = 0; ti < t.T; ti++)
    for (int ci = 0; ci < 3; ci++)
      add_list(cp.worst, p, t, ti, true, [&](int o) { return ((ctmask[t.off_set[o]] >> ci) & 1) != 0; });
  pad(cp.worst);
  return cp;
}
