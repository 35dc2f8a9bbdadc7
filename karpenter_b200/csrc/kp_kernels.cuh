// kp_kernels.cuh -- device code of the solver (sm_90a).
//
//   k_feasibility  (K1)  class x template instance-type feasibility bitmaps: one warp per (class, template) pair,
//                        bit-sliced mask ANDs -- filterInstanceTypesByRequirements (nodeclaim.go:412-480).
//   eval_candidate / topo_record  the exact CanAdd (existingnode.go:70-143, nodeclaim.go:114-202) and Topology.Record
//                        of one pod on one candidate, executed by one warp (used by kp_wsolve.cuh).
//
// Warp layout of an evaluation: lane k owns label key k (requirement slot), lane r owns resource r, lane w owns
// instance-type bitmap word w.
#pragma once
#include <cuda_runtime.h>

#include "../../include/karpsolve.h"
#include "kp_slot.hpp"

#define FULL 0xffffffffu

__device__ __forceinline__ KeyInfo key_info(const KpDev& d, int k) {
  return KeyInfo{d.val_int + (size_t)k * 64, d.val_isint[k], d.key_univ[k]};
}
__device__ __forceinline__ Slot load_slot(const uint8_t* f, const uint64_t* m, const int64_t* g, const int64_t* l,
                                          size_t i, int has_bounds) {
  Slot s;
  s.f = f[i];
  s.m = m[i];
  s.gte = has_bounds ? g[i] : 0;
  s.lte = has_bounds ? l[i] : 0;
  return s;
}
// Taints(taintset).Tolerates(tolset) (pkg/scheduling/taints.go:54-66), precomputed on the host
__device__ __forceinline__ bool tolerated(const KpDev& d, int tolset, int taintset) {
  if (taintset < 0 || d.n_taintsets == 0) return true;
  return d.tol_ok[(size_t)(tolset + 1) * d.n_taintsets + taintset];
}
__device__ __forceinline__ Slot rs_slot(const KpDev& d, int rs, int k) {
  return load_slot(d.rs_flags, d.rs_mask, d.rs_gte, d.rs_lte, (size_t)rs * d.K + k, d.has_bounds);
}

// ---------------------------------------------------------------------------------------------------------------
// Instance-type filter on bit-sliced tables (filterInstanceTypesByRequirements, nodeclaim.go:412-480), one warp:
// lane w owns instance-type bitmap word w, lane r resource r.
//
// fits_word: resources.Fits(total, allocatable) via ">= threshold" bitmaps: lane r ranks q[r] in the sorted distinct
// allocatable values of resource r, the answer is the AND of the R selected rows.
// `j_lane` (lane r): in/out threshold row of resource r (-1: none yet).  Requests of a candidate only grow, so the row
// found for the previous total is a valid starting point and the search usually advances by zero or one step; and
// because `its` already passed the rows of the previous total, only rows that ADVANCED can remove instance types.
// Returns its & Fits.
__device__ __forceinline__ uint64_t fits_word(const KpDev& d, int64_t q_lane, int lane, int* j_lane, uint64_t its) {
  const int R = d.R, ITW = d.ITW;
  int j = 0;
  bool adv = false, fresh = false;
  if (lane < R) {
    const int end = d.ge_off[lane + 1];
    int lo = *j_lane;
    fresh = lo < d.ge_off[lane];
    if (fresh) lo = d.ge_off[lane];
    const int start = lo;
    while (lo < end && d.ge_vals[lo] < q_lane) lo++;
    adv = fresh || lo != start;
    j = lo == end ? -1 : lo;  // -1: the request exceeds every instance type
    *j_lane = lo;
  }
  unsigned advm = __ballot_sync(FULL, adv);
  uint64_t fw = its;
  if (__any_sync(FULL, fresh)) fw &= (lane < ITW) ? d.it_valid[lane] : 0ull;
  while (advm) {
    const int r = __ffs(advm) - 1;
    advm &= advm - 1;
    const int jr = __shfl_sync(FULL, j, r);
    if (lane < ITW) fw &= jr >= 0 ? d.ge_bits[(size_t)jr * ITW + lane] : 0ull;
  }
  return fw;
}
// compat_off_word: word w of compatible(it, S) & hasOffering(it, S) for the requirement slots S (readable by every lane)
__device__ __forceinline__ uint64_t compat_off_word(const KpDev& d, const Slot* S, int lane) {
  const int K = d.K, ITW = d.ITW;
  // hasOffering: lane dd decides Compatible(S, offering set dd, AllowUndefinedWellKnownLabels)
  bool off_ok = false;
  if (lane < d.D) {
    uint32_t keys = d.off_keys[lane];
    off_ok = true;
    while (keys) {
      int k = __ffs(keys) - 1;
      keys &= keys - 1;
      if (!slot_compatible(key_info(d, k), S[k], d.off_slots[(size_t)lane * K + k], d.key_wellknown[k], true))
        off_ok = false;
    }
  }
  uint32_t off_mask = __ballot_sync(FULL, off_ok);
  uint64_t ow = 0, cw = ~0ull;
  if (lane < ITW) {
    while (off_mask) {
      int dd = __ffs(off_mask) - 1;
      off_mask &= off_mask - 1;
      ow |= d.offset_bits[(size_t)dd * ITW + lane];
    }
    // compatible(): InstanceType.Requirements.Intersects(S) -- shared keys only (requirements.go:254-274)
    for (int k = 0; k < K; k++) {
      Slot s = S[k];
      if (!slot_present(s)) continue;
      KeyInfo ki = key_info(d, k);
      uint64_t allowed = slot_allowed(ki, s);
      uint64_t bw = d.it_nokey[(size_t)k * ITW + lane];
      if (allowed == ki.univ) {
        bw |= d.it_nonempty[(size_t)k * ITW + lane];
      } else {
        while (allowed) {
          int v = __ffsll((long long)allowed) - 1;
          allowed &= allowed - 1;
          bw |= d.itv[((size_t)d.itv_off[k] + v) * ITW + lane];
        }
      }
      if (op_is_negative(slot_op(s))) bw |= d.it_dne[(size_t)k * ITW + lane];
      cw &= bw;
    }
  } else {
    cw = 0;
  }
  return cw & ow;
}
// word w of compat & fits & hasOffering (nodeclaim.go:434-445); *fits_out = the resource-only word
__device__ __forceinline__ uint64_t filter_its_word(const KpDev& d, const Slot* S, int64_t q_lane, int lane,
                                                    uint64_t* fits_out) {
  int j0 = -1;
  uint64_t fw = fits_word(d, q_lane, lane, &j0, ~0ull);
  *fits_out = fw;
  return compat_off_word(d, S, lane) & fw;
}

// Where the state of non-hostname group g lives: the on-chip copy of a group on the topology key while the solver CTA
// keeps one (KpDev::tk_slot), else the global tables.
struct GroupState {
  uint64_t *reg, *pop;
  int32_t* cnt;  // counter of value v at cnt[v]
};
__device__ __forceinline__ GroupState tk_state(const KpDev& d, int g, const KpGroup& G) {
  const int s = (d.tk_slot && G.key == d.tk_key) ? d.tk_slot[g] : -1;
  if (s >= 0) return GroupState{d.tk_reg + s, d.tk_pop + s, d.tk_cnt + s * d.tk_nv};
  return GroupState{d.dom_reg + g, d.dom_pop + g, d.dom_cnt + G.dom_off};
}

// ---------------------------------------------------------------------------------------------------------------
// TopologyGroup.Get for a non-hostname key (topologygroup.go:226-428). Runs on the lane that owns the key.
// Returns the `domains` requirement; an empty concrete set means "no eligible domain".
__device__ __forceinline__ Slot topo_domains(const KpDev& d, int g, const KpGroup& G, bool self, const Slot& pod_d,
                                             const Slot& node_d, uint64_t reg, uint64_t pop) {
  KeyInfo ki = key_info(d, G.key);
  const int32_t* cnt = tk_state(d, g, G).cnt;
  uint64_t pod_allowed = slot_allowed(ki, pod_d);
  uint64_t node_allowed = slot_allowed(ki, node_d);
  bool node_in = slot_present(node_d) && slot_op(node_d) == OP_IN;
  Slot out;
  out.f = SF_PRESENT;
  out.m = 0;
  out.gte = 0;
  out.lte = 0;
  if (G.type == KP_TOPO_SPREAD) {
    // domainMinCount (topologygroup.go:289-310)
    uint64_t sup = reg & pod_allowed;
    long long mn = 2147483647LL;
    int nsup = __popcll(sup);
    for (uint64_t s = sup; s;) {
      int v = __ffsll((long long)s) - 1;
      s &= s - 1;
      if (cnt[v] < mn) mn = cnt[v];
    }
    if (G.min_domains >= 0 && nsup < G.min_domains) mn = 0;
    uint64_t cand = node_in ? (node_d.m & reg) : (reg & node_allowed);
    long long best_c = 2147483647LL;
    int best = -1;
    while (cand) {  // ascending value id == the canonical iteration order (SURVEY.md H1)
      int v = __ffsll((long long)cand) - 1;
      cand &= cand - 1;
      long long c = (long long)cnt[v] + (self ? 1 : 0);
      if (c - mn <= (long long)G.max_skew && c < best_c) {
        best = v;
        best_c = c;
      }
    }
    if (best >= 0) out.m = 1ull << best;
    return out;
  }
  if (G.type == KP_TOPO_AFFINITY) {
    uint64_t opts = node_in ? (node_d.m & pod_allowed & reg & pop) : (reg & pod_allowed & pop & node_allowed);
    if (opts) {
      out.m = opts;
      return out;
    }
    bool none_populated = (reg & pop) == 0;
    bool any_compat = (reg & pop & pod_allowed) != 0;
    if (self && (none_populated || !any_compat)) {
      Slot pd = slot_present(pod_d) ? pod_d : slot_exists();
      Slot nd = slot_present(node_d) ? node_d : slot_exists();
      Slot inter = slot_intersection(ki, pd, nd);
      uint64_t a = reg & slot_allowed(ki, inter);
      if (a) out.m |= a & (~a + 1);  // lowest id == the canonical "first random domain"
      uint64_t b = reg & pod_allowed;
      if (b) out.m |= b & (~b + 1);
    }
    return out;
  }
  // anti-affinity: empty domains only
  out.m = reg & ~pop & node_allowed & pod_allowed;
  return out;
}

// TopologyGroup.Record on a hostname group (topologygroup.go:141-155): one more pod of the group on `host`.  Nothing
// here needs to know whether the domain was empty (g_anypop is only ever set), so the record is write-only: two
// fire-and-forget reductions and a store, no load on the solver's chain.  The owning warp is the only writer, and a
// __syncwarp lies between every record and the warp's next read of these tables, which orders the two.
__device__ __forceinline__ void host_record(const KpDev& d, int row, int g, int host) {
  atomicOr(d.host_pop + (size_t)row * d.HW + (host >> 5), 1u << (host & 31));
  atomicAdd(d.host_cnt + (size_t)host * d.GHS + row, 1);
  d.g_anypop[g] = 1;
}
__device__ __forceinline__ void prefetch_l1(const void* p) { asm volatile("prefetch.global.L1 [%0];" ::"l"(p)); }

// One evaluated candidate, kept in the evaluating warp's registers until the winner commits.
struct Eval {
  bool ok;
  bool res_dead;   // no remaining instance type can ever hold these requests again (monotone)
  bool changed;    // the pod tightened at least one requirement slot of the candidate
  bool compat_fail;  // rejected by Requirements.Compatible(pod requirements) alone: independent of requests
  bool pod_noop;   // Compatible passed and the pod's own requirements left every slot of the candidate as it was
  int j;           // lane r: threshold row of the total requests (fits_word)
  Slot F;          // lane k: final requirement slot of key k
  int64_t q;       // lane r: total requests (claims)
  uint64_t its;    // lane w: surviving instance-type word (claims)
};

// The pod being placed, staged once per pod in shared memory (class row of the problem + its requirement slots + the
// descriptors of the topology groups that constrain / count it, so the solver's chain never goes to HBM for them).
#define KP_PG 6              // groups per list staged with the pod; a class with more reads them from HBM
#define TKI_FP 0x100         // tkinfo: the class may take the domain fast path (see wsolve_run)
#define TKI_TK 0x200         // ... and has at least one group on the topology key
#define TKI_FAST 0x400       // topology-free class that may take the accepted-signature fast path
#define TKI_ABIT 0x800       // the class's requirement set has an "adds nothing" bit (asig < 64)
#define TKI_TOPO 0x1000      // some topology group constrains or counts the class
#define TKI_ASIG(t) ((t) & 0xff)  // requirement-set id for the "adds nothing" masks (amask), 0xff: none
struct PodCtx {
  union {
    struct {
      int tolset, rv, moff, mend, roff, rend, fsig, nsig, hoff, hend, cls, pod;
      unsigned long long tmpl_ok;  // bit n: template n's taints are tolerated (taints.go:49-66)
      int relax;                   // class after one Preferences.Relax step, -1: nothing left to relax
      int tkinfo;                  // TKI_*
      unsigned long long ports;      // host ports of the pod (interned entries, hostportusage.go:93-118)
      unsigned long long port_conf;  // every entry that Matches one of them (:50-62)
      int vol_next;                  // class carrying the pod's next volume-topology alternative, -1: none
    };
    int hdr[KP_HDR + 11];  // the class header, then class id, pod id, tmpl_ok (lo, hi), relax, tkinfo, ports, port_conf, vol_next
  };
  int64_t req[KP_MAXR];
  Slot pod_slot[KP_MAXK];
  Slot strict_slot[KP_MAXK];
  int n_mg, n_rg;      // staged entries of cls_match / cls_rec, -1: not staged (more than KP_PG)
  int m_e[KP_PG];      // cls_match entries (group | self << 30)
  int r_g[KP_PG];      // cls_rec entries
  KpGroup mg[KP_PG];
  KpGroup rg[KP_PG];
  int n_hc;            // hostname-group checks among the staged match groups (the scan's per-candidate tests)
  int4 hc[KP_PG];      // {host_row, type | self << 8, max_skew, group}
  // the run of identical pods this one starts in the queue (stager only): entries h .. h + run_n - 1 of the first pass
  // share the class, run_pod[i] is the pod of entry h + i.  The solver may commit a whole run in one step (cohorts).
  int run_n;
  int run_pod[32];
};
// entry i of the pod's match / record list
__device__ __forceinline__ void pod_match(const KpDev& d, const PodCtx& px, int i, int* e, KpGroup* G) {
  if (px.n_mg >= 0) {
    *e = px.m_e[i];
    *G = px.mg[i];
  } else {
    *e = d.cls_match[px.moff + i];
    *G = d.groups[*e & 0x3fffffff];
  }
}
__device__ __forceinline__ void pod_rec(const KpDev& d, const PodCtx& px, int i, int* g, KpGroup* G) {
  if (px.n_rg >= 0) {
    *g = px.r_g[i];
    *G = px.rg[i];
  } else {
    *g = d.cls_rec[px.roff + i];
    *G = d.groups[*g];
  }
}

// Exact CanAdd of the staged pod on one candidate (NodeClaim.CanAdd nodeclaim.go:114-202 when is_claim, else
// ExistingNode.CanAdd existingnode.go:70-143 after the taint / Fits checks of phase 1).
//   base       lane k: the candidate's current requirement slot
//   host       index of the candidate's hostname domain in host_cnt
//   scratch    per-warp shared memory, KP_MAXK slots
// LEAN: the problem has no topology group, no Gt / Lt bound, no minValues and no reservation -- those parts compile away
template <bool LEAN = false>
__device__ __forceinline__ Eval eval_candidate(const KpDev& d, const PodCtx& px, bool is_claim, const Slot& base,
                                               int64_t base_q, uint64_t base_its, int base_j, int host, Slot* scratch,
                                               int lane) {
  Eval ev;
  ev.ok = false;
  ev.res_dead = false;
  ev.changed = false;
  ev.compat_fail = false;
  ev.pod_noop = false;
  ev.j = 0;
  const int K = d.K;
  const bool allow_undef = is_claim;  // ExistingNode.CanAdd passes no compatibility options
  const bool wk = lane < K ? d.key_wellknown[lane] : false;
  KeyInfo ki = lane < K ? key_info(d, lane) : KeyInfo{d.val_int, 0ull, 0ull};
  Slot pod = lane < K ? px.pod_slot[lane] : slot_absent();
  // requirements.Compatible(pod requirements) then Add
  const bool nb = LEAN || !d.has_bounds;
  bool bad = lane < K && !(nb ? slot_compatible_nb(base, pod, wk, allow_undef) : slot_compatible(ki, base, pod, wk, allow_undef));
  if (__any_sync(FULL, bad)) {
    ev.compat_fail = true;
    return ev;
  }
  Slot M = lane < K ? (nb ? slot_add_nb(base, pod) : slot_add(ki, base, pod)) : slot_absent();
  // Topology.AddRequirements (topology.go:226-248)
  const int nm = LEAN ? 0 : px.mend - px.moff;
  if (nm > 0) {
    ev.pod_noop = !__any_sync(FULL, lane < K && !slot_eq(M, base));
    Slot Tt = M;
    bool fail = false;
    Slot strict = lane < K ? px.strict_slot[lane] : slot_absent();
    for (int i = 0; i < nm; i++) {
      int e;
      KpGroup G;
      pod_match(d, px, i, &e, &G);
      int g = e & 0x3fffffff;
      bool self = (e >> 30) & 1;
      if (G.key == d.hostname_key) {
        if (lane == 0) {  // candidates carry exactly one hostname: the fast paths of topologygroup.go:235-247,317-333,402-408
          int cnt = __ldcg(d.host_cnt + (size_t)host * d.GHS + G.host_row);
          bool ok;
          if (G.type == KP_TOPO_SPREAD)
            ok = cnt + (self ? 1 : 0) <= G.max_skew;
          else if (G.type == KP_TOPO_AFFINITY)
            ok = cnt > 0 || (self && d.g_anypop[g] == 0);
          else
            ok = cnt == 0;
          if (!ok) fail = true;
        }
      } else if (lane == G.key) {
        const GroupState st = tk_state(d, g, G);
        Slot dm = topo_domains(d, g, G, self, strict, M, *st.reg, *st.pop);
        if (dm.m == 0)
          fail = true;  // topologyError: domains.Len() == 0
        else
          Tt = slot_add(ki, Tt, dm);
      }
    }
    if (__any_sync(FULL, fail)) return ev;
    bad = lane < K && !slot_compatible(ki, M, Tt, wk, allow_undef);
    if (__any_sync(FULL, bad)) return ev;
    M = lane < K ? slot_add(ki, M, Tt) : slot_absent();
  }
  ev.F = M;
  if (!is_claim) {
    ev.changed = __any_sync(FULL, lane < K && !slot_eq(M, base));
    if (nm <= 0) ev.pod_noop = !ev.changed;
    ev.ok = true;
    return ev;
  }
  // resources.Merge + filterInstanceTypesByRequirements.  base_its already went through the filter with the
  // candidate's current requirements (every NodeClaim.Add stores the filtered list, nodeclaim.go:209; a fresh claim
  // starts from the NewScheduler prefilter, scheduler.go:147), so when the pod leaves every slot unchanged only the
  // resource test can remove instance types.
  const bool changed = __any_sync(FULL, lane < K && !slot_eq(M, base));
  ev.changed = changed;
  if (nm <= 0) ev.pod_noop = !changed;
  int64_t q = base_q + (lane < d.R ? px.req[lane] : 0);
  ev.j = base_j;
  uint64_t fw = fits_word(d, q, lane, &ev.j, base_its);
  uint64_t w = fw;
  if (changed) {
    if (lane < K) scratch[lane] = M;
    __syncwarp();
    w &= compat_off_word(d, scratch, lane);
    __syncwarp();
  }
  ev.q = q;
  ev.its = w;
  ev.ok = __any_sync(FULL, w != 0);
  ev.res_dead = !__any_sync(FULL, fw != 0);
  return ev;
}

// A class row in flight between global memory and the shared PodCtx (one warp; lane k: key k, lane r: resource r,
// lane i < KP_HDR: header word i).
struct ClassRegs {
  int hdr;                // lanes 0..KP_HDR+9: header row, class, pod, tmpl_ok lo / hi, relax, tkinfo, ports, port_conf
  int64_t req;
  Slot pod, strict;
};
__device__ __forceinline__ ClassRegs load_class_regs(const KpDev& d, int X, int pod, int lane) {
  ClassRegs c;
  const uint4* p = reinterpret_cast<const uint4*>(d.cls_lane + ((size_t)X * 32 + lane));
  const uint4 a = p[0], b = p[1];
  c.pod.m = (uint64_t)a.x | ((uint64_t)a.y << 32);
  c.strict.m = (uint64_t)a.z | ((uint64_t)a.w << 32);
  c.req = (int64_t)((uint64_t)b.x | ((uint64_t)b.y << 32));
  c.hdr = lane == KP_HDR ? X : (lane == KP_HDR + 1 ? pod : (int)b.z);
  c.pod.f = b.w & 0xffu;
  c.strict.f = (b.w >> 8) & 0xffu;
  c.pod.gte = c.pod.lte = c.strict.gte = c.strict.lte = 0;
  if (d.has_bounds && lane < d.K) {
    const size_t i = (size_t)X * d.K + lane;
    c.pod.gte = d.cp_g[i];
    c.pod.lte = d.cp_l[i];
    c.strict.gte = d.cs_g[i];
    c.strict.lte = d.cs_l[i];
  }
  return c;
}
__device__ __forceinline__ void store_class_regs(const KpDev& d, PodCtx& px, const ClassRegs& c, int lane) {
  if (lane < KP_HDR + 11) px.hdr[lane] = c.hdr;
  if (lane < d.R) px.req[lane] = c.req;
  if (lane < d.K) {
    px.pod_slot[lane] = c.pod;
    px.strict_slot[lane] = c.strict;
  }
  // the groups that constrain / count the class, parked next to the row (whole warp; lanes 0..11 move one descriptor)
  const int moff = __shfl_sync(FULL, c.hdr, 2), mend = __shfl_sync(FULL, c.hdr, 3);
  const int roff = __shfl_sync(FULL, c.hdr, 4), rend = __shfl_sync(FULL, c.hdr, 5);
  const int nm = mend - moff, nr = rend - roff;
  if (nm == 0 && nr == 0) {  // topology-free class: nothing to park
    if (lane == 0) {
      px.n_mg = 0;
      px.n_rg = 0;
      px.n_hc = 0;
    }
    return;
  }
  const bool sm = nm <= KP_PG, sr = nr <= KP_PG;
  int e = 0, g = 0;
  if (sm && lane < nm) e = d.cls_match[moff + lane];
  if (sr && lane < nr) g = d.cls_rec[roff + lane];
  if (lane == 0) {
    px.n_mg = sm ? nm : -1;
    px.n_rg = sr ? nr : -1;
  }
  if (sm && lane < nm) px.m_e[lane] = e;
  if (sr && lane < nr) px.r_g[lane] = g;
  if (sm)
    for (int i = 0; i < nm; i++) {
      const int gi = __shfl_sync(FULL, e, i) & 0x3fffffff;
      if (lane < (int)(sizeof(KpGroup) / 4)) reinterpret_cast<int*>(&px.mg[i])[lane] = reinterpret_cast<const int*>(&d.groups[gi])[lane];
    }
  if (sr)
    for (int i = 0; i < nr; i++) {
      const int gi = __shfl_sync(FULL, g, i);
      if (lane < (int)(sizeof(KpGroup) / 4)) reinterpret_cast<int*>(&px.rg[i])[lane] = reinterpret_cast<const int*>(&d.groups[gi])[lane];
    }
  __syncwarp();
  bool is_host = false;
  KpGroup G;
  if (sm && lane < nm) {
    G = px.mg[lane];
    is_host = G.key == d.hostname_key;
  }
  const unsigned hm = __ballot_sync(FULL, is_host);
  if (is_host) px.hc[__popc(hm & ((1u << lane) - 1))] = make_int4(G.host_row, G.type | (((e >> 30) & 1) << 8), G.max_skew, e & 0x3fffffff);
  if (lane == 0) px.n_hc = sm ? __popc(hm) : -1;
}

// TopologyNodeFilter.Matches of a filter whose alternatives carry host rules (KpGroup::affinity_policy 3): an alternative
// matches when the placement's requirement slots are compatible with it and its host rule admits `host`.  A branch of its
// own, so that topo_record's loop for every other group stays as it was.
__device__ __forceinline__ bool filter_matches_host_rules(const KpDev& d, const KpGroup& G, const Slot& F, int host, int lane) {
  for (int a = 0; a < G.filter_n; a++) {
    const int rs = d.filter_rs[G.filter_off + a];
    const bool bad = lane < d.K &&
                     !slot_compatible(key_info(d, lane), F, rs_slot(d, rs, lane), d.key_wellknown[lane], false);
    if (!__any_sync(FULL, bad) && host_rule_admits(d.host_rules, d.E, rs, host)) return true;
  }
  return false;
}

// Topology.Record (topology.go:197-220) for the committed placement; executed by one warp.
__device__ __forceinline__ void topo_record(const KpDev& d, const PodCtx& px, const Slot& F, int taintset, int host,
                                            bool allow_undef, int lane) {
  const int K = d.K;
  (void)allow_undef;  // TopologyNodeFilter.Matches never forwards the options (topologynodefilter.go:68-85)
  const int nr = px.rend - px.roff;
  for (int i = 0; i < nr; i++) {
    int g;
    KpGroup G;
    pod_rec(d, px, i, &g, &G);
    if (d.n_lazy && !d.g_born[g]) continue;  // the reference has not created this group yet
    bool counts = true;
    if (!G.inverse) {
      if (G.affinity_policy == 1 && G.filter_n > 0) {
        bool any_alt = false;
        for (int a = 0; a < G.filter_n; a++) {
          int rs = d.filter_rs[G.filter_off + a];
          bool bad = lane < K &&
                     !slot_compatible(key_info(d, lane), F, rs_slot(d, rs, lane), d.key_wellknown[lane], false);
          if (!__any_sync(FULL, bad)) {
            any_alt = true;
            break;
          }
        }
        counts = any_alt;
      } else if (G.affinity_policy == 3) {
        counts = filter_matches_host_rules(d, G, F, host, lane);
      }
      if (counts && G.taint_policy == 1) {
        counts = tolerated(d, G.tolset, taintset);
      }
    }
    if (!counts) continue;
    if (G.key == d.hostname_key) {
      if (lane == 0) host_record(d, G.host_row, g, host);
    } else {
      uint32_t ff = __shfl_sync(FULL, F.f, G.key);
      uint64_t mm = __shfl_sync(FULL, F.m, G.key);
      if (lane == 0 && (ff & SF_PRESENT)) {
        uint64_t rec = 0;
        if (G.inverse || G.type == KP_TOPO_ANTI_AFFINITY)
          rec = mm;  // every value the node may still take
        else if (!(ff & SF_COMPLEMENT) && __popcll(mm) == 1)
          rec = mm;
        uint64_t bits = rec;
        const GroupState st = tk_state(d, g, G);
        while (bits) {
          int v = __ffsll((long long)bits) - 1;
          bits &= bits - 1;
          st.cnt[v]++;
        }
        *st.reg |= rec;
        *st.pop |= rec;
      }
    }
  }
}

// bit dd: Requirements.Compatible(S, offering requirement set dd, AllowUndefinedWellKnownLabels)
__device__ __forceinline__ unsigned offering_ok_mask(const KpDev& d, const Slot* S, int lane) {
  bool ok = false;
  if (lane < d.D) {
    uint32_t keys = d.off_keys[lane];
    ok = true;
    while (keys) {
      const int k = __ffs(keys) - 1;
      keys &= keys - 1;
      if (!slot_compatible(key_info(d, k), S[k], d.off_slots[(size_t)lane * d.K + k], d.key_wellknown[k], true)) ok = false;
    }
  }
  return __ballot_sync(FULL, ok);
}

// offeringsToReserve (nodeclaim.go:240-287) for a candidate NodeClaim whose requirement slots after the pod are in
// `scratch` and whose surviving instance types are `its` (word `lane`).  `held` = reservation ids the claim holds now
// (0 for a fresh one).  Returns the ids to hold afterwards; *error = ReservedOfferingError (strict mode only).
__device__ __forceinline__ unsigned long long offerings_to_reserve(const KpDev& d, const int32_t* rsv_cap, const Slot* scratch,
                                                                    uint64_t its, unsigned long long held, int lane, bool* error) {
  *error = false;
  unsigned sets = offering_ok_mask(d, scratch, lane) & d.rsv_sets;  // reserved offerings compatible with the requirements
  unsigned long long compat = 0;
  while (sets) {
    const int dd = __ffs(sets) - 1;
    sets &= sets - 1;
    const bool hit = lane < d.ITW && (its & d.offset_bits[(size_t)dd * d.ITW + lane]) != 0;  // ... of a surviving, available type
    if (__any_sync(FULL, hit)) compat |= 1ull << d.set_rsv[dd];
  }
  // ReservationManager.CanReserve (reservationmanager.go:55-70): already held by this claim, or capacity left
  const bool c0 = lane < d.n_rsv && rsv_cap[lane] > 0, c1 = lane + 32 < d.n_rsv && rsv_cap[lane + 32] > 0;
  const unsigned long long avail = (unsigned long long)__ballot_sync(FULL, c0) | ((unsigned long long)__ballot_sync(FULL, c1) << 32);
  const unsigned long long take = compat & (held | avail);
  if (d.rsv_strict && take == 0 && (compat != 0 || held != 0)) *error = true;
  return take;
}
// NodeClaim.Add's bookkeeping (nodeclaim.go:216-218): reserve the new ids, release the ones no longer compatible
__device__ __forceinline__ void reservations_commit(const KpDev& d, int32_t* rsv_cap, unsigned long long held,
                                                    unsigned long long take, int lane) {
  const unsigned long long inc = held & ~take, dec = take & ~held;
  if (lane < d.n_rsv) rsv_cap[lane] += (int)((inc >> lane) & 1ull) - (int)((dec >> lane) & 1ull);
  if (lane + 32 < d.n_rsv) rsv_cap[lane + 32] += (int)((inc >> (lane + 32)) & 1ull) - (int)((dec >> (lane + 32)) & 1ull);
  __syncwarp();
}

// FinalizeScheduling (nodeclaim.go:291-307) on the claim rows in global memory: a NodeClaim that holds reservations is
// pinned to capacity-type In [reserved] and reservation-id In [held ids].  One warp, after the solve.
__device__ __forceinline__ void claims_finalize(const KpDev& d, uint8_t* sflags, uint64_t* smask, const unsigned long long* c_rsv,
                                                int nC, int lane) {
  if (!d.n_rsv || d.rsv_ct_key < 0 || d.rsv_id_key < 0) return;
  for (int c = lane; c < nC; c += 32) {
    const unsigned long long held = c_rsv[c];
    if (!held) continue;
    sflags[(size_t)c * d.K + d.rsv_ct_key] = SF_PRESENT;
    smask[(size_t)c * d.K + d.rsv_ct_key] = 1ull << d.rsv_reserved_val;
    uint64_t vals = 0;
    for (unsigned long long h = held; h;) {
      const int id = __ffsll((long long)h) - 1;
      h &= h - 1;
      vals |= d.rsv_val_of[id];
    }
    const size_t i = (size_t)c * d.K + d.rsv_id_key;
    const Slot cur{sflags[i], smask[i], 0, 0};
    const Slot out = slot_add_nb(cur, Slot{SF_PRESENT, vals, 0, 0});  // Requirements.Add: intersect with what is there
    sflags[i] = (uint8_t)out.f;
    smask[i] = out.m;
  }
  __syncwarp();
}

// ---- the domain fast path (classes flagged TKI_FP, see plan_classes in kp_prep.cpp) ------------------------------
// Every topology group of such a class sits on the hostname key or on ONE other key, the problem's "topology key" TK
// (zone in practice).  A NodeClaim that already holds a pod is pinned to a single TK value z (its slot is In{z}); for
// such a claim TopologyGroup.Get (topologygroup.go:226-428) answers either In{z} -- the claim's requirements stay as
// they are -- or nothing, and which of the two depends only on z and the group's counters.  So the verdict for ALL
// single-valued claims is one bit mask over TK's values, computed once per pod:
//   spread         z registered and count(z) + self - min <= maxSkew          (nextDomainTopologySpread :226-287)
//   anti-affinity  z registered, empty, allowed by the pod                      (nextDomainAntiAffinity :393-428)
//   affinity       z registered, populated, allowed by the pod; when the bootstrap rule of :356-374 could fire the
//                  mask cannot tell (*exact = false: no pruning, the full evaluation decides)
// Returns the AND over the pod's TK groups (all ones when it has none).  Warp-uniform.
__device__ __forceinline__ uint64_t domain_mask(const KpDev& d, const PodCtx& px, int lane, bool* exact) {
  uint64_t ez = ~0ull;
  *exact = true;
  const int nm = px.n_mg;
  const Slot strict = px.strict_slot[d.tk_key];
  const uint64_t univ = d.key_univ[d.tk_key];
  const uint64_t pod_allowed = (strict.f & SF_PRESENT) ? (((strict.f & SF_COMPLEMENT) ? ~strict.m : strict.m) & univ) : univ;
  for (int i = 0; i < nm; i++) {
    const KpGroup G = px.mg[i];
    if (G.key != d.tk_key) continue;
    const int e = px.m_e[i], g = e & 0x3fffffff;
    const bool self = (e >> 30) & 1;
    const GroupState st = tk_state(d, g, G);
    const uint64_t reg = *st.reg, pop = *st.pop;
    if (G.type == KP_TOPO_SPREAD) {
      // lane v (and v + 32) reads the counter of value v; min over the domains the pod may use (domainMinCount :289-310)
      const int32_t* cnt = st.cnt;
      const long long c0 = (reg >> lane) & 1ull ? (long long)cnt[lane] : 0, c1 = (reg >> (lane + 32)) & 1ull ? (long long)cnt[lane + 32] : 0;
      const uint64_t sup = reg & pod_allowed;
      long long mn = 2147483647LL;
      if ((sup >> lane) & 1ull) mn = c0;
      if (((sup >> (lane + 32)) & 1ull) && c1 < mn) mn = c1;
      mn = __reduce_min_sync(FULL, (int)mn);  // (counts and the sentinel fit an int: one redux instead of five shuffle rounds)
      if (G.min_domains >= 0 && __popcll(sup) < G.min_domains) mn = 0;
      const long long add = self ? 1 : 0;
      const bool ok0 = ((reg >> lane) & 1ull) && c0 + add - mn <= (long long)G.max_skew;
      const bool ok1 = ((reg >> (lane + 32)) & 1ull) && c1 + add - mn <= (long long)G.max_skew;
      const uint64_t m = (uint64_t)__ballot_sync(FULL, ok0) | ((uint64_t)__ballot_sync(FULL, ok1) << 32);
      ez &= m;
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

// Topology.Record (topology.go:197-220) of a fast-path placement: the claim's requirements are unchanged and its TK
// slot is In{z} (z < 0: the class has no TK group).  The class's record groups are staged and none needs the node
// filter's requirement check (TKI_FP), so every group is one independent read-modify-write: lane i takes group i.
__device__ __forceinline__ void topo_record_fast(const KpDev& d, const PodCtx& px, int z, int taintset, int host, int lane) {
  if (lane < px.n_rg) {
    const KpGroup G = px.rg[lane];
    const int g = px.r_g[lane];
    bool counts = true;
    if (!G.inverse && G.taint_policy == 1) counts = tolerated(d, G.tolset, taintset);
    if (counts) {
      if (G.key == d.hostname_key) {
        host_record(d, G.host_row, g, host);
      } else if (z >= 0) {
        const GroupState st = tk_state(d, g, G);
        st.cnt[z]++;
        const uint64_t bit = 1ull << z;
        if (!(*st.reg & bit)) *st.reg |= bit;
        if (!(*st.pop & bit)) *st.pop |= bit;
      }
    }
  }
  __syncwarp();
}

// InstanceTypes.SatisfiesMinValues (cloudprovider/types.go:301-337) for a NodeClaim of template n whose remaining
// instance types are `its` (word `lane` of the bitmap): every key with minValues must still see that many distinct values.
// One ballot per value, stopping as soon as enough were seen.  Warp-uniform result.
__device__ __forceinline__ bool min_values_ok(const KpDev& d, int n, uint64_t its, int lane) {
  for (int e = d.tmpl_mv_off[n]; e < d.tmpl_mv_off[n + 1]; e++) {
    const int m = d.tmpl_mv_key[e], need = d.tmpl_mv_need[e];
    int seen = 0;
    for (int v = d.mv_val_off[m]; v < d.mv_val_off[m + 1] && seen < need; v++) {
      const bool hit = lane < d.ITW && (its & d.mv_masks[(size_t)v * d.ITW + lane]) != 0;
      seen += __any_sync(FULL, hit) ? 1 : 0;
    }
    if (seen < need) return false;
  }
  return true;
}

// ---------------------------------------------------------------------------------------------------------------
// K1: feasibility of (class, template) pairs without topology. grid-stride over pairs, one warp each.
__global__ void __launch_bounds__(256) k_feasibility(KpDev d, uint64_t* out, int prefilter_only) {
  __shared__ Slot scratch_all[8][KP_MAXK];
  int lane = threadIdx.x & 31, wib = threadIdx.x >> 5;
  Slot* scratch = scratch_all[wib];
  int warps = (gridDim.x * blockDim.x) >> 5;
  int gw = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  int npairs = prefilter_only ? d.N : d.X * d.N;
  for (int pair = gw; pair < npairs; pair += warps) {
    int X = prefilter_only ? -1 : pair / d.N, n = prefilter_only ? pair : pair % d.N;
    Slot base = lane < d.K ? rs_slot(d, d.tmpl_rs[n], lane) : slot_absent();
    uint64_t its = lane < d.ITW ? (prefilter_only ? d.tmpl_its_raw : d.tmpl_its)[(size_t)n * d.ITW + lane] : 0ull;
    uint64_t w = 0;
    if (prefilter_only) {  // scheduler.go:147: filter by the template requirements alone, zero requests
      if (lane < d.K) scratch[lane] = base;
      __syncwarp();
      uint64_t fw;
      w = filter_its_word(d, scratch, 0, lane, &fw) & its;
      __syncwarp();
      if (d.mv_strict && !min_values_ok(d, n, w, lane)) w = 0;  // scheduler.go:147-156: the template is skipped
      if (lane < d.ITW) d.tmpl_its[(size_t)n * d.ITW + lane] = w;
    } else {
      bool tol_ok = tolerated(d, d.cls_tolset[X], d.tmpl_taintset[n]);
      KeyInfo ki = lane < d.K ? key_info(d, lane) : KeyInfo{d.val_int, 0ull, 0ull};
      Slot pod = lane < d.K ? rs_slot(d, d.cls_rs[X], lane) : slot_absent();
      bool bad = lane < d.K && !slot_compatible(ki, base, pod, d.key_wellknown[lane], true);
      bool any_bad = __any_sync(FULL, bad);
      Slot M = lane < d.K ? slot_add(ki, base, pod) : slot_absent();
      if (lane < d.K) scratch[lane] = M;
      __syncwarp();
      int64_t q = lane < d.R ? d.tmpl_daemon[(size_t)n * d.R + lane] + d.cls_req[(size_t)X * d.R + lane] : 0;
      uint64_t fw;
      w = filter_its_word(d, scratch, q, lane, &fw) & its;
      __syncwarp();
      // filterInstanceTypesByRequirements (nodeclaim.go:412-480) keeps nothing when the remaining types fall short of
      // the template's Strict minValues
      if (d.mv_strict && !min_values_ok(d, n, w, lane)) w = 0;
      if (any_bad || !tol_ok) w = 0;
      if (lane < d.ITW) out[((size_t)X * d.N + n) * d.ITW + lane] = w;
    }
  }
}
