// kp_prep.hpp -- host-side encoding of a kp_problem into the table layout of kp_tables.hpp.
//
// This is the part of scheduling.NewScheduler / NewTopology that runs once per Solve, not per pod
// (scheduler.go:116-184, topology.go:68-143,162-194,297-426): requirement sets -> slot rows, taint toleration matrix,
// bit-sliced instance-type tables, topology-group construction and initial domain counts.  On top of these it decides
// which shortcuts each class may take (ClassPlan) and builds the price lists of Results.TruncateInstanceTypes and
// consolidation.  libkarpsolve.so encodes the result for the device, where the per-pod hot loop runs (kp_wsolve.cuh);
// oracle/orc_cached.cpp runs the same algorithm over the same tables on one host core.
#pragma once
#include <algorithm>
#include <cstring>
#include <map>
#include <set>
#include <string>
#include <vector>

#include "../../include/karpsolve.h"
#include "kp_slot.hpp"

// a hostname group among a class's match groups: a NodeClaim is exactly one hostname domain (next_candidate)
struct HostCheck {
  int row, type, self, max_skew, g;  // KpGroup::host_row, KpGroup::type, the class selects itself, KpGroup::max_skew, group
};

// Which shortcuts each class may take.  These decide exactness: a shortcut granted to the wrong class gives a wrong
// answer.  Facts of the algorithm only; device limits (staging sizes, mask widths) are applied where they are encoded.
struct ClassPlan {
  int tk_key = -1;                // the topology key of the domain fast path: the non-hostname key most groups sit on
  bool strict_undefined = false;  // no pod can define a new key on an existing node (k_node_cand)
  int n_fsig = 0, n_asig = 0;
  // per class [max(X, 1)]
  std::vector<int32_t> fsig;    // failure signature, -1: none (a failed Compatible may not be permanent)
  std::vector<int32_t> asig;    // accepted signature: id of the class's requirement set, in class order over all classes
  std::vector<uint8_t> chain;   // member of a volume-alternative chain: no signature, no shortcut
  std::vector<uint8_t> fast;    // the accepted-signature fast path: fsig >= 0, counted by no group, no re-check of the types
  std::vector<uint8_t> fp;      // the domain fast path: every group on the hostname key or on tk_key, see plan_classes
  std::vector<uint8_t> has_tk;  // fp and at least one group on tk_key
  std::vector<uint64_t> tok;    // tolerated templates (the first 64)
  std::vector<int32_t> nsig;    // existing-node signature: id of (requirement set, toleration set)
  std::vector<int64_t> rank;    // NewQueue class rank: cpu desc, then memory desc (queue.go:72-108)
  std::vector<int32_t> hchk_off;  // [X + 1] the class's hostname checks in hchk
  std::vector<HostCheck> hchk;
  // per existing-node signature: requirement set (-1: tolerations only, the chain classes) and toleration set
  std::vector<int32_t> nsig_rs, nsig_tolset;
};

struct HostTables {
  int K = 0, R = 0, T = 0, ITW = 0, N = 0, X = 0, G = 0, GH = 0, E = 0, D = 0;
  int n_reqsets = 0, n_taintsets = 0, n_tolsets = 0, has_bounds = 0, hostname_key = -1, nodes_res = -1, n_rv = 0;
  int cpu_res = -1, mem_res = -1;
  std::vector<uint8_t> key_wellknown;
  std::vector<uint64_t> key_univ, val_isint;
  std::vector<int64_t> val_int;
  std::vector<uint8_t> rs_flags;
  std::vector<uint64_t> rs_mask;
  std::vector<int64_t> rs_gte, rs_lte;
  std::vector<uint32_t> rs_keys;
  std::vector<uint8_t> tol_ok;
  std::vector<uint64_t> itv, it_nokey, it_dne, it_nonempty, it_valid;
  std::vector<int64_t> ge_vals;
  std::vector<int32_t> ge_off, itv_off;
  std::vector<Slot> off_slots;
  std::vector<uint32_t> off_keys;
  std::vector<uint64_t> ge_bits;
  std::vector<int32_t> offset_rs;
  std::vector<int32_t> off_set;  // [offerings] index of the offering's distinct requirement set
  // reserved capacity (ReservationManager): reservation id behind a distinct offering set (-1: none), initial capacity
  int n_rsv = 0;
  bool rsv_strict = false;
  std::vector<int32_t> set_rsv, rsv_cap0;
  std::vector<uint64_t> offset_bits;
  std::vector<int64_t> it_capacity, it_alloc;
  std::vector<int32_t> tmpl_rs, tmpl_taintset;
  std::vector<uint64_t> tmpl_its_raw;
  std::vector<int64_t> tmpl_daemon, tmpl_remaining;
  std::vector<uint32_t> tmpl_limit_present;
  std::vector<int64_t> cls_req;
  std::vector<int32_t> cls_relax;  // class after one Preferences.Relax step, -1: none
  std::vector<int32_t> cls_vol_next;  // next volume-topology alternative of a class (kp_problem.class_vol_next), -1: none
  bool has_vol_alts = false;
  std::vector<int32_t> g_born, g_birth, cls_lazy_off, cls_lazy;  // groups born mid-solve (KpDev::g_born)
  int n_regular = 0;                                               // groups [0, n_regular) are regular, the rest inverse
  // minValues: per template a list of (table m, need); per table m the value range [mv_val_off[m], mv_val_off[m+1]) of
  // instance-type bitmaps mv_masks[value * ITW ..]
  bool has_min_values = false, min_values_strict = false;
  std::vector<int32_t> tmpl_mv_off, tmpl_mv_key, tmpl_mv_need, mv_val_off;
  std::vector<uint64_t> mv_masks;
  std::vector<int32_t> cls_rs, cls_strict_rs, cls_tolset, cls_rv, cls_match_off, cls_match, cls_rec_off, cls_rec;
  std::vector<int64_t> cls_sort_cpu, cls_sort_mem;
  std::vector<KpGroup> groups;
  std::vector<int32_t> filter_rs;
  std::vector<int32_t> dom_cnt;
  std::vector<uint64_t> dom_reg, dom_pop;
  std::vector<int32_t> g_ndomains, g_nempty;
  std::vector<int32_t> host_cnt_nodes;  // [GH * E] initial hostname-group counts of existing nodes
  std::vector<int32_t> node_taintset;
  std::vector<uint8_t> node_flags;
  std::vector<int64_t> node_rem;
  std::vector<uint32_t> node_rem_present;
  std::vector<uint8_t> node_sflags;
  std::vector<uint64_t> node_smask;
  std::vector<int64_t> node_sgte, node_slte;
  std::vector<int32_t> group_out_order;  // result order: regular groups (creation order) then inverse groups
  ClassPlan plan;
};

// active: which nodes take part as existing nodes; extra_bound: additional (class,node) pods counted by the topology
int kp_prepare(const kp_problem* p, const std::vector<uint8_t>& node_active,
               const std::vector<std::pair<int, int>>& extra_bound, const std::vector<int32_t>& pending_classes,
               HostTables& h, std::string& err);

// Price lists of offerings: per list, a range [off[i], off[i + 1]) of (price, distinct offering set) entries.  `set` and
// `price` are never empty, so each uploads as a table of at least one element.
struct PriceLists {
  std::vector<int32_t> off, set;
  std::vector<double> price;
};
// OrderByPrice: available offerings per instance type, cheapest first (types.go:238-257)
PriceLists order_by_price(const kp_problem* p, const HostTables& t);

// The price tables of computeConsolidation (consolidation.go:136-337)
struct ConsolPrices {
  std::vector<double> node_price;  // [max(E, 1)] getCandidatePrices: the node's cheapest compatible offering, -1: none
  int ct_valid = 0;                // bit i: capacity type i of (reserved, spot, on-demand) is known
  PriceLists worst;                // WorstLaunchPrice: per (type, capacity type i) list 3 * type + i, dearest first
};
ConsolPrices consol_prices(const kp_problem* p, const HostTables& t, const kp_consol_input* in);
