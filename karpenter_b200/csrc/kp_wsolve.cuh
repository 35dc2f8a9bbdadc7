// kp_wsolve.cuh -- the Scheduler.Solve loop (scheduler.go:381-684) executed by ONE WARP per Scheduler instance.
//
// First-fit-decreasing with the reference's "fewest pods first" claim order is a serial chain: pod i's placement
// decides the state pod i+1 sees.  A CTA-wide design spends its time in barriers around one working warp, so the
// chain runs inside a single warp with no block-level synchronisation at all:
//
//   lane k  owns label key k      (requirement slot algebra: Compatible / Add)
//   lane r  owns resource r       (requests, Fits)
//   lane w  owns word w of the instance-type bitmap
//   lane i  owns candidate base+i while scanning the claim order / node bitmaps (ballot -> lowest index wins)
//
// The same routine serves the provisioning solve (k_wsolve_batch) and the consolidation search (one instance
// per removal subset, thousands of warps in flight, k_consolidate): an instance is a WInst, a block of pointers to
// its private mutable state.  Existing nodes are found through per-class candidate bitmaps (supersets computed once
// by k_node_cand) and every candidate is re-checked exactly; the consolidation instances share the cluster's base node
// table read-only and keep their few modified nodes in a private overlay.
#pragma once
#include "kp_gosort.cuh"
#include "kp_kernels.cuh"

enum { PERT_NONE = 0, PERT_INC = 1, PERT_APPEND = 2 };

struct WInst {
  // pods: local ids 0..P-1
  int P;
  int32_t* queue;       // [P+1] circular queue of local pod ids, initially byCPUAndMemoryDescending (queue.go:72-108)
  int32_t* qcls;        // [P+1] class of queue[i]
  int32_t* last_len;    // [P]
  int32_t* pod_target;  // [P] or null
  uint8_t* pod_error;   // [P] or null
  const uint8_t* pod_kind;  // [P] or null (all 0): see KpDev::pod_kind
  // NodeClaims
  int Cmax;
  int32_t *c_tmpl, *c_npods;
  int64_t* c_req;
  uint8_t* c_sflags;
  uint64_t* c_smask;
  int64_t *c_sgte, *c_slte;
  uint64_t* c_its;
  int32_t* c_j;             // [Cmax*R] threshold row of the claim's requests per resource (fits_word)
  // rows of the first CR claims are kept in shared memory (0 = none); copied out when the solve ends
  int CR;
  uint8_t* s_sflags;
  uint64_t* s_smask;
  int64_t* s_req;
  int32_t* s_j;
  uint64_t* s_its;
  int32_t *order, *cnt_at;  // s.newNodeClaims: claim id / len(Pods) by position
  // monotone failure cache, one 16-byte entry per claim: x = bit f set when requirement signature f was rejected by
  // Requirements.Compatible, y = bit rv set when no remaining instance type can hold the claim's requests plus request
  // vector rv.  Signatures / vectors with an index >= 64 are simply not cached (exact either way).
  ulonglong2* cmask;
  // amask[c] bit f: requirement signature f adds nothing to claim c's requirements.  Stable for the claim's lifetime
  // (the claim's value sets only shrink, so they stay inside the pod's), which reduces CanAdd for such a pair to the
  // resource test.
  unsigned long long* amask;
  unsigned long long* g_amask;
  // c_dom[c]: the value claim c's slot on the topology key is pinned to, 0xff when it is not a single In value (null: the
  // instance does not use the domain fast path)
  uint8_t *c_dom, *g_c_dom;
  // ReservationManager state of the instance (reservationmanager.go:28-110): remaining capacity per reservation id and
  // the ids each NodeClaim holds (null / unused when the problem has no reserved offerings)
  int32_t* rsv_cap;
  unsigned long long* c_rsv;
  // host ports in use per NodeClaim / per existing node (direct mode) / per overlay entry (consolidation)
  unsigned long long *c_ports, *node_ports, *ov_ports;
  // While the claim order, template ids and failure masks fit, they live in shared memory (CS = claims the shared
  // copies can hold, 0 = not in use); the moment a claim id reaches CS everything migrates to the global arrays below.
  int CS;
  int32_t *g_order, *g_cnt_at, *g_c_tmpl;
  ulonglong2* g_cmask;
  int64_t* tmpl_remaining;  // [N*R]
  // existing nodes
  int64_t* node_rem;
  uint32_t* node_rem_present;
  uint8_t* node_sflags;
  uint64_t* node_smask;
  int64_t *node_sgte, *node_slte;
  int32_t* node_npods;      // direct mode only
  uint32_t *nfit, *nstat;
  const uint32_t* nactive;
  const uint32_t *nfit_sum, *nstat_sum;  // one bit per bitmap word: skip 1024-node chunks nothing can match in
  int n_removed;
  const int32_t* removed;   // overlay mode: nodes taken out of the cluster (the consolidation candidates)
  // overlay (consolidation): entry i shadows node ov_node[i]
  int ov_cap, n_ov;
  int32_t* ov_node;
  int64_t* ov_rem;
  uint32_t* ov_present;
  uint8_t* ov_sflags;
  uint64_t* ov_smask;
  int64_t *ov_sgte, *ov_slte;
  // results
  int n_claims, n_unsched, n_uninit, status;
  long long ev_existing, ev_inflight, ev_tmpl, commits, slow_sorts, scan_chunks, evals, fast_commits;
};

// index of `node` in the overlay, -1 if it is untouched (warp-uniform result)
__device__ __forceinline__ int ov_find(const WInst& I, int node, int lane) {
  for (int b = 0; b < I.n_ov; b += 32) {
    int i = b + lane;
    unsigned m = __ballot_sync(FULL, i < I.n_ov && I.ov_node[i] == node);
    if (m) return b + __ffs(m) - 1;
  }
  return -1;
}

// a NodeClaim's row: requirement slot of key `lane`, requests / threshold row of resource `lane`, instance-type word `lane`
template <bool LEAN = false>
__device__ __forceinline__ void claim_load(const KpDev& d, const WInst& I, int c, int lane, Slot* b, int64_t* q,
                                           uint64_t* its, int* j) {
  const int K = d.K, R = d.R, ITW = d.ITW;
  *b = slot_absent();
  *q = 0;
  *its = 0;
  *j = 0;
  if (c < I.CR) {
    if (lane < K) {
      b->f = I.s_sflags[c * K + lane];
      b->m = I.s_smask[c * K + lane];
    }
    if (lane < R) {
      *q = I.s_req[c * R + lane];
      *j = I.s_j[c * R + lane];
    }
    if (lane < ITW) *its = I.s_its[c * ITW + lane];
  } else {
    if (lane < K) {
      b->f = I.c_sflags[(size_t)c * K + lane];
      b->m = I.c_smask[(size_t)c * K + lane];
    }
    if (lane < R) {
      *q = I.c_req[(size_t)c * R + lane];
      *j = I.c_j[(size_t)c * R + lane];
    }
    if (lane < ITW) *its = I.c_its[(size_t)c * ITW + lane];
  }
  if (!LEAN && d.has_bounds && lane < K) {
    b->gte = I.c_sgte[(size_t)c * K + lane];
    b->lte = I.c_slte[(size_t)c * K + lane];
  }
}
template <bool LEAN = false>
__device__ __forceinline__ void claim_store(const KpDev& d, WInst& I, int c, int lane, const Eval& ev, bool slots) {
  const int K = d.K, R = d.R, ITW = d.ITW;
  if (!LEAN && slots && I.c_dom && lane == d.tk_key)
    I.c_dom[c] = (ev.F.f == SF_PRESENT && __popcll(ev.F.m) == 1) ? (uint8_t)(__ffsll((long long)ev.F.m) - 1) : (uint8_t)0xff;
  if (c < I.CR) {
    if (slots && lane < K) {
      I.s_sflags[c * K + lane] = (uint8_t)ev.F.f;
      I.s_smask[c * K + lane] = ev.F.m;
    }
    if (lane < R) {
      I.s_req[c * R + lane] = ev.q;
      I.s_j[c * R + lane] = ev.j;
    }
    if (lane < ITW) I.s_its[c * ITW + lane] = ev.its;
  } else {
    if (slots && lane < K) {
      I.c_sflags[(size_t)c * K + lane] = (uint8_t)ev.F.f;
      I.c_smask[(size_t)c * K + lane] = ev.F.m;
    }
    if (lane < R) {
      I.c_req[(size_t)c * R + lane] = ev.q;
      I.c_j[(size_t)c * R + lane] = ev.j;
    }
    if (lane < ITW) I.c_its[(size_t)c * ITW + lane] = ev.its;
  }
  if (!LEAN && slots && d.has_bounds && lane < K) {
    I.c_sgte[(size_t)c * K + lane] = ev.F.gte;
    I.c_slte[(size_t)c * K + lane] = ev.F.lte;
  }
}
// requests / threshold rows only (lane r), and the instance-type words only (lane w)
__device__ __forceinline__ void claim_load_rq(const KpDev& d, const WInst& I, int c, int lane, int64_t* q, int* j) {
  *q = 0;
  *j = 0;
  if (lane < d.R) {
    if (c < I.CR) {
      *q = I.s_req[c * d.R + lane];
      *j = I.s_j[c * d.R + lane];
    } else {
      *q = I.c_req[(size_t)c * d.R + lane];
      *j = I.c_j[(size_t)c * d.R + lane];
    }
  }
}
__device__ __forceinline__ uint64_t claim_load_its(const KpDev& d, const WInst& I, int c, int lane) {
  if (lane >= d.ITW) return 0ull;
  return c < I.CR ? I.s_its[c * d.ITW + lane] : I.c_its[(size_t)c * d.ITW + lane];
}
__device__ __forceinline__ void claim_store_rq(const KpDev& d, WInst& I, int c, int lane, int64_t q, int j, bool with_its,
                                               uint64_t its) {
  if (c < I.CR) {
    if (lane < d.R) {
      I.s_req[c * d.R + lane] = q;
      I.s_j[c * d.R + lane] = j;
    }
    if (with_its && lane < d.ITW) I.s_its[c * d.ITW + lane] = its;
  } else {
    if (lane < d.R) {
      I.c_req[(size_t)c * d.R + lane] = q;
      I.c_j[(size_t)c * d.R + lane] = j;
    }
    if (with_its && lane < d.ITW) I.c_its[(size_t)c * d.ITW + lane] = its;
  }
}
// copy the shared-memory claim rows to their global arrays (end of the solve)
__device__ __forceinline__ void claim_rows_flush(const KpDev& d, WInst& I, int nC, int lane) {
  const int n = nC < I.CR ? nC : I.CR;
  for (int i = lane; i < n * d.K; i += 32) {
    I.c_sflags[i] = I.s_sflags[i];
    I.c_smask[i] = I.s_smask[i];
  }
  for (int i = lane; i < n * d.R; i += 32) {
    I.c_req[i] = I.s_req[i];
    I.c_j[i] = I.s_j[i];
  }
  for (int i = lane; i < n * d.ITW; i += 32) I.c_its[i] = I.s_its[i];
  __syncwarp();
}

// ---- in-flight scan: the next position >= `from` in the claim order whose claim can still pass the cheap tests
struct ScanCtx {
  unsigned long long fbit, rbit, tok;  // failure bits to test, tolerated templates
  bool all_tmpl;
  int hoff, hend;                      // hostname-group checks of the class
  int first_clear, first_rclear;       // first position (>= the scan start) whose signature / request-vector bit is clear
  bool use_ez;                         // prune claims pinned to a topology-key value outside `ez` (domain_mask)
  uint64_t ez;
  const int4* hc;                      // the hostname checks: staged with the pod, or cls_hchk + hoff
};
// U sub-chunks of 32 positions per step: their loads are independent, so a step costs one memory latency, not U.
template <int U, bool LEAN = false>
__device__ __forceinline__ int next_candidate(const KpDev& d, const WInst& I, const int32_t* ord, int nC, int from,
                                              ScanCtx& sc, int lane, int E, int* cc_out, int limit = 0x7fffffff) {
  const ulonglong2* cm = I.cmask;
  if (limit > nC) limit = nC;  // positions at and above `limit` are not looked at: the caller continues there
  for (int base = from; base < limit; base += 32 * U) {  // (unaligned: a step always looks at 32 * U fresh positions)
    bool pass[U], fclear[U], rclear[U];
    int c[U];
#pragma unroll
    for (int u = 0; u < U; u++) {
      const int pos = base + u * 32 + lane;
      c[u] = -1;
      pass[u] = fclear[u] = rclear[u] = false;
      if (pos < limit && pos >= from) {
        c[u] = ord[pos];
        const ulonglong2 mk = cm[c[u]];
        fclear[u] = !(mk.x & sc.fbit);
        rclear[u] = !(mk.y & sc.rbit);
        pass[u] = fclear[u] && rclear[u];
        if (pass[u] && !sc.all_tmpl) pass[u] = (sc.tok >> I.c_tmpl[c[u]]) & 1ull;
      }
    }
    if (!LEAN && sc.use_ez) {
#pragma unroll
      for (int u = 0; u < U; u++)
        if (pass[u]) {
          const int z = I.c_dom[c[u]];
          if (z != 0xff) pass[u] = (sc.ez >> z) & 1ull;
        }
    }
    // hostname groups: a NodeClaim is exactly one hostname domain (topologygroup.go:235-247,317-333,402-408).  Two
    // groups per round, so that all their counter loads are in flight together (one L2 latency, not one per group).
    for (int i = sc.hoff; !LEAN && i < sc.hend; i += 2) {
      const bool two = i + 1 < sc.hend;
      const int4 ha = sc.hc[i], hb = two ? sc.hc[i + 1] : ha;
      // anti-affinity / affinity only ask "is the domain populated": one bit of host_pop (L1: the stager prefetched the
      // row); a hostname spread needs the count
      const bool cnt_a = (ha.y & 0xff) == KP_TOPO_SPREAD, cnt_b = (hb.y & 0xff) == KP_TOPO_SPREAD;
      int ca[U], cb[U];
#pragma unroll
      for (int u = 0; u < U; u++) {
        const int hi = E + c[u];
        ca[u] = cb[u] = 0;
        if (pass[u]) {
          ca[u] = cnt_a ? __ldcg(d.host_cnt + (size_t)hi * d.GHS + ha.x)
                        : (int)((d.host_pop[(size_t)ha.x * d.HW + (hi >> 5)] >> (hi & 31)) & 1u);
          if (two)
            cb[u] = cnt_b ? __ldcg(d.host_cnt + (size_t)hi * d.GHS + hb.x)
                          : (int)((d.host_pop[(size_t)hb.x * d.HW + (hi >> 5)] >> (hi & 31)) & 1u);
        }
      }
#pragma unroll
      for (int r = 0; r < 2; r++) {
        if (r == 1 && !two) break;
        const int4 hc = r == 0 ? ha : hb;
        const int type = hc.y & 0xff, self = hc.y >> 8;
#pragma unroll
        for (int u = 0; u < U; u++) {
          if (!pass[u]) continue;
          const int hcnt = r == 0 ? ca[u] : cb[u];
          if (type == KP_TOPO_SPREAD)
            pass[u] = hcnt + self <= hc.z;
          else if (type == KP_TOPO_AFFINITY)
            pass[u] = hcnt > 0 || (self && (d.g_ndomains[hc.w] - d.g_nempty[hc.w]) == 0);
          else
            pass[u] = hcnt == 0;
        }
      }
    }
#pragma unroll
    for (int u = 0; u < U; u++) {
      if (sc.fbit && sc.first_clear < 0) {
        const unsigned fm = __ballot_sync(FULL, fclear[u]);
        if (fm) sc.first_clear = base + u * 32 + __ffs(fm) - 1;
      }
      if (sc.rbit && sc.first_rclear < 0) {
        const unsigned rm = __ballot_sync(FULL, rclear[u]);
        if (rm) sc.first_rclear = base + u * 32 + __ffs(rm) - 1;
      }
      const unsigned m = __ballot_sync(FULL, pass[u]);
      if (m) {
        const int l = __ffs(m) - 1;
        *cc_out = __shfl_sync(FULL, c[u], l);
        return base + u * 32 + l;
      }
    }
  }
  return -1;
}

// The cheap tests of next_candidate for ONE claim per lane, without the topology-key mask (which changes from pod to pod
// of a cohort): failure bits, tolerated template, hostname groups.
template <bool LEAN>
__device__ __forceinline__ bool cheap_pass(const KpDev& d, const WInst& I, const ScanCtx& sc, int c, int E) {
  const ulonglong2 mk = I.cmask[c];
  bool pass = !(mk.x & sc.fbit) && !(mk.y & sc.rbit);
  if (pass && !sc.all_tmpl) pass = (sc.tok >> I.c_tmpl[c]) & 1ull;
  for (int i = sc.hoff; !LEAN && pass && i < sc.hend; i++) {
    const int4 hc = sc.hc[i];
    const int type = hc.y & 0xff, self = hc.y >> 8, hi = E + c;
    const int hcnt = type == KP_TOPO_SPREAD ? __ldcg(d.host_cnt + (size_t)hi * d.GHS + hc.x)
                                            : (int)((d.host_pop[(size_t)hc.x * d.HW + (hi >> 5)] >> (hi & 31)) & 1u);
    if (type == KP_TOPO_SPREAD)
      pass = hcnt + self <= hc.z;
    else if (type == KP_TOPO_AFFINITY)
      pass = hcnt > 0 || (self && (d.g_ndomains[hc.w] - d.g_nempty[hc.w]) == 0);
    else
      pass = hcnt == 0;
  }
  return pass;
}

// CanAdd of k more pods of the staged class on a claim whose requirements they leave as they are (the "adds nothing" fast
// path): do the merged requests still fit a remaining instance type?  The stored list only changes when a threshold row
// advances.  Monotone in k.  Outputs (lane r: requests / threshold row; lane w: instance-type word when *any_adv).
__device__ __forceinline__ bool fp_fit(const KpDev& d, const WInst& I, const PodCtx& px, int cc, int k, int lane, int64_t* q_out,
                                       int* lo_out, bool* any_adv_out, uint64_t* its_out) {
  int64_t q;
  int j;
  claim_load_rq(d, I, cc, lane, &q, &j);
  int lo = j;
  bool adv = false;
  if (lane < d.R) {
    q += px.req[lane] * (int64_t)k;
    const int end = d.ge_off[lane + 1];
    while (lo < end && d.ge_vals[lo] < q) lo++;
    adv = lo != j;
  }
  unsigned advm = __ballot_sync(FULL, adv);
  const bool any_adv = advm != 0;
  uint64_t its = 0;
  bool ok = true;
  if (any_adv) {
    its = claim_load_its(d, I, cc, lane);
    const int jj = (lane < d.R && lo == d.ge_off[lane + 1]) ? -1 : lo;
    while (advm) {
      const int r = __ffs(advm) - 1;
      advm &= advm - 1;
      const int jr = __shfl_sync(FULL, jj, r);
      if (lane < d.ITW) its &= jr >= 0 ? d.ge_bits[(size_t)jr * d.ITW + lane] : 0ull;
    }
    ok = __any_sync(FULL, its != 0);
  }
  *q_out = q;
  *lo_out = lo;
  *any_adv_out = any_adv;
  *its_out = its;
  return ok;
}

// shared -> global migration of the small per-claim arrays (see WInst::CS); executed once, by the whole warp
__device__ __forceinline__ void migrate_small(const KpDev& d, WInst& I, int nC, int lane) {
  for (int i = lane; i < nC; i += 32) {
    I.g_order[i] = I.order[i];
    I.g_cnt_at[i] = I.cnt_at[i];
    I.g_c_tmpl[i] = I.c_tmpl[i];
    I.g_cmask[i] = I.cmask[i];
    I.g_amask[i] = I.amask[i];
    if (I.c_dom) I.g_c_dom[i] = I.c_dom[i];
  }
  __syncwarp();
  if (lane == 0) {
    I.order = I.g_order;
    I.cnt_at = I.g_cnt_at;
    I.c_tmpl = I.g_c_tmpl;
    I.cmask = I.g_cmask;
    I.amask = I.g_amask;
    if (I.c_dom) I.c_dom = I.g_c_dom;
    I.CS = 0;
  }
  __syncwarp();
}

// Pod staging ring between a stager warp and the solver warp of one CTA (k_wsolve_batch): the stager walks the queue a few
// pods ahead and parks each pod's class row (header, requests, requirement slots) in shared memory, so the solver's
// dependence chain never waits on -- or spends instructions for -- the L2 loads of the next pod.
#define KP_RING 8
struct StageRing {
  volatile int produced;  // pods staged so far (stager)
  volatile int consumed;  // pods the solver is done with (solver)
  volatile int tail_pub;  // queue entries below this index are valid (solver; grows with every requeue)
  volatile int done;
  volatile int skip_to;   // queue entries below this index were committed as part of a cohort: nothing to stage (solver)
  PodCtx slot[KP_RING];
};

template <bool COHORT>
__device__ void stager_run(const KpDev& d, const WInst& I, StageRing* ring, const int lane) {
  const int cap = I.P + 1;
  // The queue is read 32 entries at a time (one coalesced load; entries below tail_pub never change), and the class row
  // of pod i+1 is requested before pod i is parked, so the stager pays one L2 latency per pod at most -- it has to stay
  // ahead of a solver that needs under 2 us per pod.
  for (int base = 0;;) {
    int avail;
    for (;;) {
      if (ring->done) return;
      const int sk = __shfl_sync(FULL, (int)ring->skip_to, 0);
      if (sk > base) base = sk;
      avail = __shfl_sync(FULL, (int)ring->tail_pub, 0) - base;
      if (avail > 0) break;
      __nanosleep(64);
    }
    __threadfence_block();
    if (avail > 32) avail = 32;
    int li = 0, X = -1;
    if (lane < avail) {
      const int qi = (base + lane) % cap;
      li = __ldcg(I.queue + qi);
      X = __ldcg(I.qcls + qi);
    }
    ClassRegs nxt = load_class_regs(d, __shfl_sync(FULL, X, 0), __shfl_sync(FULL, li, 0), lane);
    bool rebased = false;
    for (int i = 0; i < avail; i++) {
      const int idx = base + i;
      const ClassRegs c = nxt;
      if (i + 1 < avail) nxt = load_class_regs(d, __shfl_sync(FULL, X, i + 1), __shfl_sync(FULL, li, i + 1), lane);
      int sk = 0;
      for (;;) {
        if (ring->done) return;
        sk = ring->skip_to;
        if (sk > idx || idx - ring->consumed < KP_RING) break;
        __nanosleep(32);
      }
      sk = __shfl_sync(FULL, sk, 0);
      if (sk > idx) {  // the solver committed this entry with a cohort: restart the block at the first entry it still needs
        base = sk;
        rebased = true;
        break;
      }
      PodCtx& slot = ring->slot[idx & (KP_RING - 1)];
      store_class_regs(d, slot, c, lane);
      // the run of identical pods starting here (first pass only: requeued pods are tried one at a time)
      if (COHORT) {
        const int Xi = __shfl_sync(FULL, X, i);
        const unsigned same = __ballot_sync(FULL, lane >= i && lane < avail && X == Xi && base + lane < I.P);
        const unsigned tail_m = same >> i;  // bit t: entry idx + t is in the block and of the same class
        const int run = tail_m == FULL ? 32 : __ffs(~tail_m) - 1;
        const int rp = __shfl_sync(FULL, li, (i + lane) & 31);
        slot.run_pod[lane] = rp;
        if (lane == 0) slot.run_n = run;
      }
      __syncwarp();
      // pull what the solver will read for this pod into L1 now: the presence rows of its hostname groups (the part
      // that covers the NodeClaims: 8 lines == 8 192 claims) and the counter rows of its topology-key groups
      if (slot.n_hc > 0) {
        const int g8 = lane >> 3, l8 = lane & 7;  // four groups at a time, eight lines each
        for (int k = g8; k < slot.n_hc; k += 4) {
          const int w = (d.E >> 5) + l8 * 32;
          if (w < d.HW) prefetch_l1(d.host_pop + (size_t)slot.hc[k].x * d.HW + w);
        }
      }
      if (slot.n_mg > 0 && lane < 2 * slot.n_mg) {
        const KpGroup& G = slot.mg[lane >> 1];
        if (G.key == d.tk_key) prefetch_l1(d.dom_cnt + G.dom_off + (lane & 1) * 32);
      }
      __threadfence_block();
      __syncwarp();
      if (lane == 0) ring->produced = idx + 1;
    }
    if (!rebased) base += avail;
  }
}

// ---- cohorts -----------------------------------------------------------------------------------------------------
// The stager reports the run of identical pods a queue entry starts (PodCtx::run_n).  When the class takes the fast path
// (requirements implied by the claim's, domain = the claim's pinned value), the targets of the next pods follow from the
// claim order alone, so a run commits in one step:
//   one claim, alone in its tie group of the order (nobody else has its pod count): the next pods land on it again until
//     it is full or its count passes the next claim's -- k pods with ONE resource test (fp_fit is monotone in k);
//   a tie group of several claims: every commit moves its claim to the end of the group (the stable result of
//     sort.Slice(len(Pods)), see the sort stage of wsolve_run), so the following pods take the following claims of the
//     group, each at most once; the moves are applied in closed form.
// Everything else -- a candidate that needs the full evaluation, a sort Go would not do stably, the end of the 32-claim
// window -- ends the cohort and the next pod takes the ordinary path: the result is the reference's, pod for pod.  The
// last pick is never moved here: the reference sorts at the start of the NEXT pod's in-flight stage (scheduler.go:504),
// which may never come (end of the queue, a pod an existing node takes); it is left to the sort stage as PERT_INC.
// Kept out of line: the ordinary path's instruction footprint (one warp, no latency hiding) must not grow with it.
struct CohortOut {
  int state;          // 0: not attempted (take the ordinary path)  1: the candidate was tried, failed and is marked  2: committed
  int npods;          // pods committed (state 2)
  int nevals;
  long long ev_sum;   // sum of (position + 1) over the commits: what the reference evaluated
  int pert, pert_pos;
  unsigned moved;     // window lanes whose claim moved to the end of the group; the group is [w0, gE]
  int w0, gE;
};
template <bool LEAN>
__device__ __noinline__ CohortOut cohort_try(const KpDev& d, WInst& I, const PodCtx& px, const ScanCtx sc, int32_t* ord, int32_t* cnt,
                                             const int nC, const int lb, const int cpos, const int cc, const int E, const int lane,
                                             const unsigned long long abit, const unsigned long long rbit, const bool fast_ok,
                                             const bool has_tk) {
  CohortOut out;
  out.state = 0;
  out.npods = 0;
  out.nevals = 0;
  out.ev_sum = 0;
  out.pert = PERT_NONE;
  out.pert_pos = 0;
  out.moved = 0;
  out.w0 = 0;
  out.gE = 0;
  bool fp0 = (I.amask[cc] & abit) != 0;
  if (fp0 && !fast_ok && has_tk) fp0 = I.c_dom[cc] != 0xff;
  if (!fp0) return out;
  // the window: 32 positions from the first one that passes every test that does not depend on the pod's domain mask
  // (claims pinned to a value this pod may not use can be the next pod's target)
  int w0 = cpos;
  if (!LEAN && sc.use_ez) {
    ScanCtx st = sc;
    st.use_ez = false;
    st.first_clear = 0;
    st.first_rclear = 0;
    int c2;
    w0 = st.hend > st.hoff ? next_candidate<4, LEAN>(d, I, ord, nC, lb, st, lane, E, &c2)
                           : next_candidate<1, LEAN>(d, I, ord, nC, lb, st, lane, E, &c2);
    if (w0 < 0 || w0 > cpos) w0 = cpos;
  }
  const int pw = w0 + lane;
  int wc = -1, wn = -1;
  if (pw < nC) {
    wc = ord[pw];
    wn = cnt[pw];
  }
  const int c0 = __shfl_sync(FULL, wn, 0);
  const unsigned gmask = __ballot_sync(FULL, pw < nC && wn == c0);
  const int gsz = gmask == FULL ? 32 : __ffs(~gmask) - 1;  // the tie group is contiguous: the order is sorted
  const int L = px.run_n;
  if (fast_ok && gsz == 1) {
    // ---- one claim, k pods
    const int nxt = __shfl_sync(FULL, wn, 1);
    int kcap = L;
    if (w0 + 1 < nC && (long long)nxt - c0 + 1 < kcap) kcap = nxt - c0 + 1;  // the count may pass the next one only once
    int64_t q, qb;
    int lo, lob;
    bool adv, advb;
    uint64_t its, itsb;
    int k = kcap;
    out.nevals = 1;
    if (!fp_fit(d, I, px, cc, k, lane, &q, &lo, &adv, &its)) {
      int good = 0, bad = kcap;
      while (bad - good > 1) {
        const int mid = (good + bad) >> 1;
        if (fp_fit(d, I, px, cc, mid, lane, &qb, &lob, &advb, &itsb)) {
          good = mid;
          q = qb;
          lo = lob;
          adv = advb;
          its = itsb;
        } else {
          bad = mid;
        }
      }
      k = good;
    }
    if (k == 0) {  // not even one: permanent for this request vector
      if (lane == 0) I.cmask[cc].y |= rbit;
      __syncwarp();
      out.state = 1;
      return out;
    }
    claim_store_rq(d, I, cc, lane, q, lo, adv, its);
    if (lane == 0) cnt[cpos] += k;
    if (I.pod_target && lane < k) {
      I.pod_target[px.run_pod[lane]] = KP_TARGET_CLAIM(cc);
      I.pod_error[px.run_pod[lane]] = KP_PODERR_NONE;
    }
    __syncwarp();
    out.state = 2;
    out.npods = k;
    out.ev_sum = (long long)k * (cpos + 1);
    out.pert = PERT_INC;
    out.pert_pos = cpos;
    return out;
  }
  if (!(gsz >= 2 && cpos < w0 + gsz && (d.stable_order || nC <= 12 || nC >= 50))) return out;
  // ---- a tie group: the static verdict of every window claim, then one pick per pod
  bool wpass = false, wfp = false;
  int wz = -1;
  if (lane < gsz) {
    wpass = cheap_pass<LEAN>(d, I, sc, wc, E);
    if (wpass) {
      wfp = (I.amask[wc] & abit) != 0;
      if (wfp && !fast_ok && has_tk) {
        wz = I.c_dom[wc];
        wfp = wz != 0xff;
      }
    }
  }
  unsigned avail = __ballot_sync(FULL, wpass && wfp);
  const unsigned bar = __ballot_sync(FULL, wpass && !wfp);  // would need the full evaluation: nothing beyond it
  if (bar) avail &= (1u << (__ffs(bar) - 1)) - 1;
  if (!((avail >> (cpos - w0)) & 1u)) return out;
  const bool gend_known = gsz < 32 || w0 + 32 >= nC;
  unsigned picked = 0;  // claims whose move is settled (every pick but the last)
  int npick = 0, nmoved = 0, my_t = -1, j = 0;
  int prev_l = -1, prev_pj = 0;
  bool prev_inv = false;
  while (j < L) {
    if (prev_l >= 0) {
      // pod j reaches the in-flight stage (its class fails on the existing nodes): the reference sorts now.  An inversion
      // exists iff a claim of the old count still follows the previous pick; Go repairs it stably unless the pick stands at
      // one of the positions choosePivot samples (see the sort stage)
      bool stable = true;
      if (prev_inv && !d.stable_order && nC > 12) {
        const int q4 = nC / 4, pj = prev_pj;
        stable = !(pj == q4 - 1 || pj == q4 || pj == 2 * q4 - 1 || pj == 2 * q4 || pj == 3 * q4 - 1 || pj == 3 * q4);
      }
      if (!stable) break;  // the real pdqsort decides: the sort stage runs it
      if (lane == prev_l) my_t = nmoved;
      nmoved++;
      picked |= 1u << prev_l;
      prev_l = -1;
    }
    unsigned allowed = avail;
    if (!LEAN && has_tk) {
      uint64_t ez = sc.ez;
      if (j > 0) {
        bool exact;
        ez = domain_mask(d, px, lane, &exact);
        if (!exact) break;
      }
      allowed &= __ballot_sync(FULL, wz >= 0 && ((ez >> wz) & 1ull));
    }
    if (!allowed) break;
    const int l = __ffs(allowed) - 1;
    const int cl = __shfl_sync(FULL, wc, l);
    int64_t q;
    int lo;
    bool adv;
    uint64_t its;
    out.nevals++;
    avail &= ~(1u << l);
    if (!fp_fit(d, I, px, cl, 1, lane, &q, &lo, &adv, &its)) {  // full: the same pod takes the next claim
      if (lane == 0) I.cmask[cl].y |= rbit;
      __syncwarp();
      continue;
    }
    claim_store_rq(d, I, cl, lane, q, lo, adv, its);
    const int pj = w0 + l - __popc(picked & ((1u << l) - 1));  // where the claim stands right now
    out.ev_sum += pj + 1;
    if (lane == 0 && I.pod_target) {
      I.pod_target[px.run_pod[j]] = KP_TARGET_CLAIM(cl);
      I.pod_error[px.run_pod[j]] = KP_PODERR_NONE;
    }
    if (!LEAN && !fast_ok) topo_record_fast(d, px, __shfl_sync(FULL, wz, l), d.tmpl_taintset[I.c_tmpl[cl]], E + cl, lane);
    __syncwarp();
    const unsigned rest = gmask & ~picked & ~(1u << l);
    prev_inv = !gend_known || (rest & ~((2u << l) - 1u)) != 0;
    prev_l = l;
    prev_pj = pj;
    j++;
    npick++;
  }
  if (npick == 0) {  // (every tried claim was full and is marked)
    out.state = 1;
    return out;
  }
  // ---- the settled moves in closed form.  Every stable move takes its claim (count c0 + 1 now) right behind the last
  // claim that still has c0 pods: the group ends up as [not moved, in order][moved, LAST one first].
  const int m = nmoved;
  int gE = w0 + gsz - 1;  // last position of the tie group
  if (gsz == 32 && m > 0) {  // it may go on behind the window: those claims close up by m
    for (int s0 = w0 + 32;; s0 += 32) {
      const int i = s0 + lane;
      const bool in = i < nC && cnt[i] == c0;
      const int vo = in ? ord[i] : 0;
      const unsigned gk = __ballot_sync(FULL, in);
      const int n = gk == FULL ? 32 : __ffs(~gk) - 1;
      __syncwarp();
      if (lane < n) {
        ord[i - m] = vo;
        cnt[i - m] = c0;
      }
      __syncwarp();
      gE = s0 + n - 1;
      if (n < 32) break;
    }
  }
  const bool mv = (picked >> lane) & 1u;
  const int rank = __popc(~picked & ((1u << lane) - 1));  // claims below me that stay
  __syncwarp();
  if (lane < gsz) {
    if (mv) {
      ord[gE - my_t] = wc;
      cnt[gE - my_t] = c0 + 1;
    } else {
      ord[w0 + rank] = wc;
      cnt[w0 + rank] = lane == prev_l ? c0 + 1 : c0;
    }
  }
  __syncwarp();
  out.state = 2;
  out.npods = npick;
  out.moved = picked;
  out.w0 = w0;
  out.gE = gE;
  if (prev_l >= 0) {
    out.pert = PERT_INC;
    out.pert_pos = w0 + __popc(~picked & ((1u << prev_l) - 1));
  }
  return out;
}

// The pod's next volume-topology alternative (nodeclaim.go:136-153): the requirement slots of class `alt` replace the staged
// ones -- everything else of the row is the same pod.  next_alt: the class after `alt` in the chain, -1 at its end.
__device__ __forceinline__ void load_alt_slots(const KpDev& d, PodCtx& px, int alt, int lane) {
  if (lane < d.K) {
    const ClsLane c = d.cls_lane[(size_t)alt * 32 + lane];
    Slot sl;
    sl.f = c.pod_f;
    sl.m = c.pod_m;
    sl.gte = 0;
    sl.lte = 0;
    if (d.has_bounds) {
      sl.gte = d.cp_g[(size_t)alt * d.K + lane];
      sl.lte = d.cp_l[(size_t)alt * d.K + lane];
    }
    px.pod_slot[lane] = sl;
  }
  __syncwarp();
}
__device__ __forceinline__ int next_alt(const KpDev& d, int alt) { return d.cls_lane[(size_t)alt * 32 + KP_HDR + 10].hdr; }

// One Scheduler.Solve over the instance's queue.  OVERLAY: existing-node state = shared base + private overlay.
// STAGED: pods arrive through a StageRing filled by a second warp instead of being staged inline.
// COHORT: runs of identical pods may commit in one step (cohort_try); instantiated separately because the mere call site
// costs the ordinary path 7 % (register allocation of a 250-register loop) -- the host picks it when the queue has runs.
// VOL: some pod has several volume-topology alternatives (kp_problem.class_vol_next): every candidate evaluation walks the
// pod's chain of alternative requirement rows; compiled into an instantiation of its own for the same reason as COHORT.
// LEAN: no topology group, Gt / Lt bound, minValues or reservation anywhere in the problem (the host decides): the code for
// them is not even compiled into that instance, which keeps the serial chain's instruction footprint small.
template <bool OVERLAY, bool STAGED, bool LEAN = false, bool COHORT = false, bool VOL = false>
__device__ void wsolve_run(const KpDev& d, WInst& I, PodCtx& ctx, Slot* scratch, const int lane, StageRing* ring = nullptr) {
  const int K = d.K, R = d.R, ITW = d.ITW, E = d.E, EW = d.EW;
  const int P = I.P;
  int head = 0, tail = P;
  const int cap = P + 1;
  int hq = 0, tq = P;  // head / tail modulo cap (cap > P, so the initial tail index is P)
  const long long watchdog_limit = 4ll * P + 1024;
  int nC = 0;
  int pert = PERT_NONE, pert_pos = 0;
  long long ev_existing = 0, ev_inflight = 0, ev_tmpl = 0, commits = 0, slow_sorts = 0, scan_chunks = 0, evals = 0, fast_commits = 0;
  int n_unsched = 0, n_uninit = 0, status = KP_OK, n_born = 0;
  int32_t* ord = I.order;
  int32_t* cnt = I.cnt_at;
  // templates NewScheduler kept (scheduler.go:147-160)
  int alive_tmpl = 0;
  for (int n = 0; n < d.N; n++) {
    uint64_t w = lane < ITW ? d.tmpl_its[(size_t)n * ITW + lane] : 0ull;
    alive_tmpl += __any_sync(FULL, w != 0) ? 1 : 0;
  }
  int n_active_nodes = 0;
  for (int w = lane; w < EW; w += 32) n_active_nodes += __popc(I.nactive[w]);
  for (int o = 16; o; o >>= 1) n_active_nodes += __shfl_xor_sync(FULL, n_active_nodes, o);
  if (OVERLAY) n_active_nodes -= I.n_removed;

  // software pipeline of the class-row staging: `pf` holds the class row of queue index pf_idx (loads issued one
  // iteration ahead), `ids` the (class, pod) of queue index ids_idx (two iterations ahead)
  ClassRegs pf;
  int pf_idx = -1, ids_idx = -1, ids_cls = 0, ids_pod = 0;
  pf.hdr = 0;
  pf.req = 0;
  pf.pod = slot_absent();
  pf.strict = slot_absent();

  // lb0 / lb1 (lane f): every claim at a position below this bound has rejected requirement signature f (resp. f+32)
  // for good, so the in-flight scan of a pod with that signature starts there.  Maintained under every reordering.
  int lb0 = 0, lb1 = 0;
  // lr0 / lr1 (lane v): the same for request vector v (resp. v+32): every claim below can never fit it again
  int lr0 = 0, lr1 = 0;
  long long watchdog = 0;
  unsigned long long t_start = 0;
  if (d.deadline_ns > 0) asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t_start));
  for (;;) {
    // ---- Queue.Pop (queue.go:46-60)
    const int len = tail - head;
    if (len == 0) break;
    if (d.deadline_ns > 0 && (watchdog & 63) == 0) {  // context deadline (scheduler.go:411-414): partial results stay valid
      unsigned long long now;
      asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(now));
      now = __shfl_sync(FULL, now, 0);
      if ((long long)(now - t_start) > d.deadline_ns) {
        status = KP_DEADLINE;
        break;
      }
    }
    if (++watchdog > watchdog_limit) {  // cannot happen: every requeue cycle needs progress (queue.go:54-58)
      status = KP_ERR_INVALID;
      break;
    }
    const int h = head;
    const int hq1 = hq + 1 >= cap ? hq + 1 - cap : hq + 1, hq2 = hq1 + 1 >= cap ? hq1 + 1 - cap : hq1 + 1;
    int li, X;
    if (STAGED) {
      if (lane == 0) ring->consumed = h;  // every slot below h is free again
      while (ring->produced <= h) {
      }
      __threadfence_block();
      __syncwarp();
      const PodCtx& sx = ring->slot[h & (KP_RING - 1)];
      li = sx.pod;
      X = sx.cls;
    } else if (ids_idx == h) {
      li = ids_pod;
      X = ids_cls;
    } else {
      li = I.queue[hq];
      X = I.qcls[hq];
    }
    if (h >= P && I.last_len[li] == len) break;  // a full cycle without progress
    head = h + 1;
    hq = hq1;
    if (!STAGED) {
      {
        ClassRegs cur = pf_idx == h ? pf : load_class_regs(d, X, li, lane);
        __syncwarp();
        store_class_regs(d, ctx, cur, lane);
        __syncwarp();
      }
      // issue the loads for the next two pods; nothing below waits on them
      pf_idx = -1;
      if (h + 1 < tail) {
        int nli, nX;
        if (ids_idx == h + 1) {
          nli = ids_pod;
          nX = ids_cls;
        } else {
          nli = I.queue[hq1];
          nX = I.qcls[hq1];
        }
        pf = load_class_regs(d, nX, nli, lane);
        pf_idx = h + 1;
      }
      ids_idx = -1;
      if (h + 2 < tail) {
        ids_pod = I.queue[hq2];
        ids_cls = I.qcls[hq2];
        ids_idx = h + 2;
      }
    }
    PodCtx& pxw = STAGED ? ring->slot[h & (KP_RING - 1)] : ctx;
    int Xc = X;  // class the pod is tried as: X, then its relaxations (trySchedule, scheduler.go:438-469)
  try_pod:
    const PodCtx& px = pxw;
    const int rv = px.rv, fsig = px.fsig;
    const unsigned long long fbit = (fsig >= 0 && fsig < 64) ? 1ull << fsig : 0ull;
    const unsigned long long rbit = (rv < 64 && !(VOL && px.vol_next >= 0)) ? 1ull << rv : 0ull;
    bool found = false;

    // ================= addToExistingNode (scheduler.go:520-555) =================
    if (E > 0 && px.nsig >= 0) {
      const uint32_t* fitrow = I.nfit + (size_t)rv * EW;
      const uint32_t* strow = I.nstat + (size_t)px.nsig * EW;
      int seen = 0;
      // chunks of 32 bitmap words (1024 nodes) that can hold a candidate at all, from the word-level summaries: one
      // parallel load for up to 32 chunks (32 768 nodes); clusters beyond that scan every chunk
      unsigned live = 0xffffffffu;
      if (d.ESW <= 32) {
        const uint32_t sw = lane < d.ESW ? (I.nfit_sum[(size_t)rv * d.ESW + lane] & I.nstat_sum[(size_t)px.nsig * d.ESW + lane]) : 0u;
        live = __ballot_sync(FULL, sw != 0);
      }
      for (int w0 = 0; w0 < EW && !found; w0 += 32) {
        if (d.ESW <= 32 && !((live >> (w0 >> 5)) & 1u)) continue;
        const int w = w0 + lane;
        uint32_t bits = w < EW ? (fitrow[w] & strow[w] & I.nactive[w]) : 0u;
        if (OVERLAY)
          for (int i = 0; i < I.n_removed; i++)
            if ((I.removed[i] >> 5) == w) bits &= ~(1u << (I.removed[i] & 31));
        unsigned has = __ballot_sync(FULL, bits != 0);
        while (has && !found) {
          const int src = __ffs(has) - 1;
          has &= has - 1;
          uint32_t bw = __shfl_sync(FULL, bits, src);
          while (bw && !found) {
            const int b = __ffs(bw) - 1;
            bw &= bw - 1;
            const int node = (w0 + src) * 32 + b;
            seen++;
            // current state of the node
            int oi = -1;
            if (OVERLAY) oi = ov_find(I, node, lane);
            Slot nb = slot_absent();
            int64_t rem = 0;
            uint32_t pr;
            if (OVERLAY && oi >= 0) {
              if (lane < K) nb = load_slot(I.ov_sflags, I.ov_smask, I.ov_sgte, I.ov_slte, (size_t)oi * K + lane, (!LEAN && d.has_bounds));
              if (lane < R) rem = I.ov_rem[(size_t)oi * R + lane];
              pr = I.ov_present[oi];
            } else {
              if (lane < K)
                nb = load_slot(I.node_sflags, I.node_smask, I.node_sgte, I.node_slte, (size_t)node * K + lane, (!LEAN && d.has_bounds));
              if (lane < R) rem = I.node_rem[(size_t)node * R + lane];
              pr = I.node_rem_present[node];
            }
            // HostPortUsage.Conflicts (existingnode.go:76-82)
            if (!LEAN && px.port_conf) {
              const unsigned long long used = (OVERLAY && oi >= 0) ? I.ov_ports[oi] : I.node_ports[node];
              if (used & px.port_conf) continue;
            }
            // resources.Fits(pod requests, remaining) (resources.go:150-163)
            bool bad = false;
            if (lane < R) {
              const bool present = (pr >> lane) & 1;
              if (present && rem < 0) bad = true;
              if (px.req[lane] > (present ? rem : 0)) bad = true;
            }
            if (__any_sync(FULL, bad)) {
              if (!OVERLAY && lane == 0) I.nfit[(size_t)rv * EW + (node >> 5)] &= ~(1u << (node & 31));  // monotone
              continue;
            }
            Eval ev = eval_candidate<LEAN>(d, px, false, nb, 0, 0, 0, node, scratch, lane);
            if (VOL && !ev.ok && px.vol_next >= 0) {  // the other volume-topology alternatives (existingnode.go:98-113)
              for (int alt = px.vol_next; alt >= 0 && !ev.ok; alt = next_alt(d, alt)) {
                load_alt_slots(d, pxw, alt, lane);
                ev = eval_candidate<LEAN>(d, px, false, nb, 0, 0, 0, node, scratch, lane);
              }
              if (!ev.ok) load_alt_slots(d, pxw, Xc, lane);  // the next candidate starts with the first alternative again
            }
            if (!ev.ok) continue;
            // ExistingNode.Add (existingnode.go:147-155)
            if (OVERLAY) {
              const bool oi_new = oi < 0;
              if (oi < 0) {
                oi = I.n_ov;
                if (oi >= I.ov_cap) {
                  status = KP_ERR_CAPACITY;
                  break;
                }
                if (lane == 0) {
                  I.ov_node[oi] = node;
                  I.n_ov = oi + 1;
                }
              }
              if (lane < K) {
                const size_t i = (size_t)oi * K + lane;
                I.ov_sflags[i] = (uint8_t)ev.F.f;
                I.ov_smask[i] = ev.F.m;
                if ((!LEAN && d.has_bounds)) {
                  I.ov_sgte[i] = ev.F.gte;
                  I.ov_slte[i] = ev.F.lte;
                }
              }
              if (lane < R) I.ov_rem[(size_t)oi * R + lane] = rem - px.req[lane];
              if (lane == 0) I.ov_present[oi] = pr | ((1u << R) - 1);
              if (!LEAN && d.n_hostports && lane == 0) I.ov_ports[oi] = (oi_new ? I.node_ports[node] : I.ov_ports[oi]) | px.ports;
              __syncwarp();
            } else {
              if (ev.changed && lane < K) {
                const size_t i = (size_t)node * K + lane;
                I.node_sflags[i] = (uint8_t)ev.F.f;
                I.node_smask[i] = ev.F.m;
                if ((!LEAN && d.has_bounds)) {
                  I.node_sgte[i] = ev.F.gte;
                  I.node_slte[i] = ev.F.lte;
                }
              }
              if (lane < R) I.node_rem[(size_t)node * R + lane] = rem - px.req[lane];
              if (lane == 0) {
                I.node_rem_present[node] = pr | ((1u << R) - 1);
                I.node_npods[node]++;
                if (!LEAN && px.ports) I.node_ports[node] |= px.ports;
              }
            }
            if (lane == 0) {
              if (I.pod_target) {
                I.pod_target[li] = node;
                I.pod_error[li] = KP_PODERR_NONE;
              }
            }
            // helpers.go:121-140: an uninitialized target is an error for a candidate's pod only
            if (!(d.node_flags[node] & KP_NODE_INITIALIZED) && (!I.pod_kind || I.pod_kind[li] == 0)) n_uninit++;
            if (!LEAN) topo_record(d, px, ev.F, d.node_taintset[node], node, false, lane);
            ev_existing += node + 1;
            found = true;
          }
          if (status != KP_OK) break;
        }
        if (status != KP_OK) break;
      }
      if (status != KP_OK) break;
      if (found) {
        commits++;
        continue;
      }
      ev_existing += n_active_nodes;
    } else if (E > 0) {
      ev_existing += n_active_nodes;
    }

    // ================= sort.Slice(newNodeClaims, len(Pods) asc) (scheduler.go:504) =================
    if (pert != PERT_NONE) {
      const int p = pert_pos;
      const bool inversion = pert == PERT_INC ? (p + 1 < nC && cnt[p + 1] < cnt[p]) : (nC >= 2 && cnt[nC - 1] < cnt[nC - 2]);
      if (inversion) {
        // When does Go's pdqsort leave the stable result?  n <= 12: insertion sort (stable).  n >= 50: choosePivot
        // samples the triples around n/4, n/2, 3n/4; the slice is sorted except for the one pair (p, p+1), so it
        // reports "increasing" -- and partialInsertionSort then repairs the pair by shifting the elevated element
        // right, i.e. the stable move -- exactly when p is not the first or middle element of a sampled triple.  (An
        // appended claim sits at n-1, never sampled.)  Everything else runs the real pdqsort.
        bool stable = d.stable_order || nC <= 12;
        if (!stable && nC >= 50) {
          const int q4 = nC / 4;
          stable = pert == PERT_APPEND || !(p == q4 - 1 || p == q4 || p == 2 * q4 - 1 || p == 2 * q4 || p == 3 * q4 - 1 || p == 3 * q4);
        }
        if (stable) {
          if (pert == PERT_INC) {  // elevated count: shift smaller successors left until one is not smaller
            const int ec = cnt[p], eo = ord[p];
            int i0 = p;
            for (;;) {
              const int i = i0 + lane;
              const bool in = i + 1 < nC;
              const int vc = in ? cnt[i + 1] : 0x7fffffff, vo = in ? ord[i + 1] : 0;
              const unsigned stop = __ballot_sync(FULL, vc >= ec);
              const int nmove = stop ? __ffs(stop) - 1 : 32;
              __syncwarp();
              if (lane < nmove) {
                cnt[i] = vc;
                ord[i] = vo;
              }
              __syncwarp();
              i0 += nmove;
              if (nmove < 32) break;
            }
            if (lane == 0) {
              cnt[i0] = ec;
              ord[i0] = eo;
            }
            // positions (p, i0] moved one to the left: a bound inside that range follows its elements
            if (p < lb0 && lb0 <= i0) lb0--;
            if (p < lb1 && lb1 <= i0) lb1--;
            if (p < lr0 && lr0 <= i0) lr0--;
            if (p < lr1 && lr1 <= i0) lr1--;
          } else {  // new claim appended: shift larger predecessors right until one is not larger
            const int ec = cnt[nC - 1], eo = ord[nC - 1];
            int i0 = nC - 1;
            for (;;) {
              const int i = i0 - lane;
              const bool in = i - 1 >= 0;
              const int vc = in ? cnt[i - 1] : -0x7fffffff, vo = in ? ord[i - 1] : 0;
              const unsigned stop = __ballot_sync(FULL, vc <= ec);
              const int nmove = stop ? __ffs(stop) - 1 : 32;
              __syncwarp();
              if (lane < nmove) {
                cnt[i] = vc;
                ord[i] = vo;
              }
              __syncwarp();
              i0 -= nmove;
              if (nmove < 32) break;
            }
            if (lane == 0) {
              cnt[i0] = ec;
              ord[i0] = eo;
            }
            // the new claim (untested by every signature) now sits at i0
            if (lb0 > i0) lb0 = i0;
            if (lb1 > i0) lb1 = i0;
            if (lr0 > i0) lr0 = i0;
            if (lr1 > i0) lr1 = i0;
          }
        } else {
          // exact pdqsort emulation (rare: ties scrambled by Go's unstable partition), warp-cooperative
          WarpSorter s{cnt, ord, lane};
          s.pdqsort(0, nC, WarpSorter::bits_len((unsigned long long)nC));
          slow_sorts++;
          lb0 = 0;  // ties were permuted arbitrarily: the bounds restart
          lb1 = 0;
          lr0 = 0;
          lr1 = 0;
        }
        __syncwarp();
      } else if (pert == PERT_APPEND) {  // the new claim stays last
        if (lb0 > nC - 1) lb0 = nC - 1;
        if (lb1 > nC - 1) lb1 = nC - 1;
        if (lr0 > nC - 1) lr0 = nC - 1;
        if (lr1 > nC - 1) lr1 = nC - 1;
      }
      pert = PERT_NONE;
    }

    // ================= addToInflightNode (scheduler.go:557-589) =================
    {
      ScanCtx sc;
      sc.fbit = fbit;
      sc.rbit = rbit;
      sc.tok = px.tmpl_ok;
      sc.all_tmpl = (sc.tok & d.tmpl_all) == d.tmpl_all;
      sc.first_clear = -1;
      sc.first_rclear = -1;
      sc.use_ez = false;
      sc.ez = ~0ull;
      // tkinfo (host-computed per class, kp_prep.cpp plan_classes): which shortcuts the class may take
      const int tki = px.tkinfo;
      // bit of the pod's requirement set in the claims' "adds nothing" masks
      const unsigned long long abit = (tki & TKI_ABIT) ? 1ull << (tki & 63) : 0ull;
      // topology-free and counted by no topology group (no minValues / reservations to re-check on the shrinking type list)
      const bool fast_ok = tki & TKI_FAST;
      // the domain fast path: topology on the hostname key and / or the topology key only (kp_kernels.cuh domain_mask)
      bool dom_fp = false, has_tk = false;
      if (!LEAN && (tki & TKI_TOPO)) {
        if (px.n_hc >= 0) {  // hostname checks staged with the pod
          sc.hc = px.hc;
          sc.hoff = 0;
          sc.hend = px.n_hc;
        } else {
          sc.hc = d.cls_hchk;
          sc.hoff = px.hoff;
          sc.hend = px.hend;
        }
        dom_fp = (tki & TKI_FP) && I.c_dom != nullptr;
        has_tk = tki & TKI_TK;
        if (dom_fp && has_tk) {
          bool exact;
          sc.ez = domain_mask(d, px, lane, &exact);
          sc.use_ez = exact;
          dom_fp = exact;
        }
        dom_fp = dom_fp && abit != 0;
      } else {
        sc.hc = nullptr;
        sc.hoff = 0;
        sc.hend = 0;
      }
      int lbf = 0, lbr = 0;
      if (fbit) lbf = __shfl_sync(FULL, fsig < 32 ? lb0 : lb1, fsig & 31);
      if (rbit) lbr = __shfl_sync(FULL, rv < 32 ? lr0 : lr1, rv & 31);
      const int lb = lbf > lbr ? lbf : lbr;  // below either bound a claim fails for one of the two reasons
      const bool scanned = (sc.tok & d.tmpl_all) != 0;
      int from = lb;
      // ---- cohorts (cohort_try): a run of identical fast-path pods may commit in one step
      unsigned coh_moved = 0;
      int coh_w0 = 0, coh_gE = 0, coh_extra = 0;
      bool coh_ok = COHORT && STAGED && !OVERLAY && d.cohort && Xc == X && px.run_n >= 2 && abit != 0 && (fast_ok || dom_fp) &&
                    (LEAN || (px.ports == 0 && px.port_conf == 0)) && (fast_ok || !has_tk || n_active_nodes == 0);
      for (int i = sc.hoff; !LEAN && coh_ok && i < sc.hend; i++)
        if ((sc.hc[i].y & 0xff) == KP_TOPO_AFFINITY) coh_ok = false;  // "is any domain populated" changes with every record
      while (scanned && !found) {
        int cc;
        // classes with hostname checks read presence words / counters per candidate: 128 positions per step there (their
        // loads overlap) -- after ONE 32-wide step: most pods find their claim among the first positions of the scan
        int cpos;
        if (sc.hend > sc.hoff) {
          const int lim = from + 32;
          cpos = next_candidate<1, LEAN>(d, I, ord, nC, from, sc, lane, E, &cc, lim);
          if (cpos < 0 && lim < nC) cpos = next_candidate<4, LEAN>(d, I, ord, nC, lim, sc, lane, E, &cc);
        } else {
          cpos = next_candidate<1, LEAN>(d, I, ord, nC, from, sc, lane, E, &cc);
        }
        if (cpos < 0) break;
        from = cpos + 1;
        {
          if (!LEAN && px.port_conf && (I.c_ports[cc] & px.port_conf)) continue;  // host ports (nodeclaim.go:120-124)
          if (COHORT && coh_ok) {
            const CohortOut co = cohort_try<LEAN>(d, I, px, sc, ord, cnt, nC, lb, cpos, cc, E, lane, abit, rbit, fast_ok, has_tk);
            evals += co.nevals;
            if (co.state == 2) {
              fast_commits += co.npods;
              ev_inflight += co.ev_sum;
              coh_extra = co.npods - 1;
              coh_moved = co.moved;
              coh_w0 = co.w0;
              coh_gE = co.gE;
              pert = co.pert;
              pert_pos = co.pert_pos;
              found = true;
              continue;
            }
            if (co.state == 1) continue;  // the candidate was tried and is marked: go on scanning
          }
          int zdom = -1;  // fast-path candidates of a class with topology-key groups: the claim's pinned value
          bool fp = false;
          if ((fast_ok || dom_fp) && (I.amask[cc] & abit)) {
            fp = true;
            if (!fast_ok && has_tk) {
              zdom = I.c_dom[cc];
              fp = zdom != 0xff;  // (the scan already tested the value against the domain mask)
            }
          }
          if (fp) {
            // ---- the pod's requirements are already implied by the claim's (and, for a fast-path topology class, the
            // domain choice is the value the claim is pinned to): CanAdd == "do the merged requests still fit a
            // remaining instance type", and the stored list only changes when a threshold row advances
            int64_t q;
            int lo;
            bool any_adv;
            uint64_t its;
            const bool ok = fp_fit(d, I, px, cc, 1, lane, &q, &lo, &any_adv, &its);
            evals++;
            if (!ok) {  // nothing left that holds the merged requests: permanent for this request vector
              if (lane == 0) I.cmask[cc].y |= rbit;
              __syncwarp();
              continue;
            }
            claim_store_rq(d, I, cc, lane, q, lo, any_adv, its);
            if (lane == 0) {
              if (!LEAN && px.ports) I.c_ports[cc] |= px.ports;
              cnt[cpos]++;
              if (I.pod_target) {
                I.pod_target[li] = KP_TARGET_CLAIM(cc);
                I.pod_error[li] = KP_PODERR_NONE;
              }
            }
            if (!LEAN && !fast_ok) topo_record_fast(d, px, zdom, d.tmpl_taintset[I.c_tmpl[cc]], E + cc, lane);
            fast_commits++;
            __syncwarp();
            pert = PERT_INC;
            pert_pos = cpos;
            ev_inflight += cpos + 1;
            found = true;
            continue;
          }
          Slot b;
          int64_t bq;
          uint64_t bi;
          int bj;
          claim_load<LEAN>(d, I, cc, lane, &b, &bq, &bi, &bj);
          evals++;
          Eval ev;
          unsigned long long held = 0, take = 0;
          bool alt_loaded = false;
          for (int alt = -1;;) {
            ev = eval_candidate<LEAN>(d, px, true, b, bq, bi, bj, E + cc, scratch, lane);
            // Strict minValues (nodeclaim.go:464-475): the surviving types must still span enough distinct values
            if (!LEAN && d.mv_strict && ev.ok && !min_values_ok(d, I.c_tmpl[cc], ev.its, lane)) ev.ok = false;
            if (abit && ev.pod_noop && lane == 0) I.amask[cc] |= abit;
            held = 0;
            take = 0;
            if (!LEAN && d.n_rsv && ev.ok) {  // offeringsToReserve (nodeclaim.go:197-200): a ReservedOfferingError is just "next claim" here
              if (lane < K) scratch[lane] = ev.F;
              __syncwarp();
              held = I.c_rsv[cc];
              bool rerr;
              take = offerings_to_reserve(d, I.rsv_cap, scratch, ev.its, held, lane, &rerr);
              __syncwarp();
              if (rerr) ev.ok = false;
            }
            if (!VOL || ev.ok) break;
            alt = alt < 0 ? px.vol_next : next_alt(d, alt);  // the other volume-topology alternatives (nodeclaim.go:136-153)
            if (alt < 0) break;
            load_alt_slots(d, pxw, alt, lane);
            alt_loaded = true;
          }
          if (VOL && alt_loaded && !ev.ok) load_alt_slots(d, pxw, Xc, lane);  // the next candidate starts with the first alternative
          if (!ev.ok) {
            if (lane == 0) {
              ulonglong2 mk = I.cmask[cc];
              if (ev.res_dead) mk.y |= rbit;
              if (ev.compat_fail) mk.x |= fbit;
              I.cmask[cc] = mk;
            }
            __syncwarp();
            continue;
          }
          // NodeClaim.Add (nodeclaim.go:207-219)
          claim_store<LEAN>(d, I, cc, lane, ev, ev.changed);
          if (!LEAN && d.n_rsv) {
            reservations_commit(d, I.rsv_cap, held, take, lane);
            if (lane == 0) I.c_rsv[cc] = take;
          }
          if (lane == 0) {
            if (!LEAN && px.ports) I.c_ports[cc] |= px.ports;
            cnt[cpos]++;
            if (I.pod_target) {
              I.pod_target[li] = KP_TARGET_CLAIM(cc);
              I.pod_error[li] = KP_PODERR_NONE;
            }
          }
          if (!LEAN) topo_record(d, px, ev.F, d.tmpl_taintset[I.c_tmpl[cc]], E + cc, true, lane);
          __syncwarp();
          pert = PERT_INC;
          pert_pos = cpos;
          ev_inflight += cpos + 1;  // claims 0..cpos were evaluated by the reference
          found = true;
        }
      }
      // a bound may only advance when the scan really started at it (positions below `lb` were not looked at)
      if (fbit && scanned && lbf == lb) {  // all positions below the first clear bit rejected the signature
        const int nb = sc.first_clear >= 0 ? sc.first_clear : nC;
        if (lane == (fsig & 31)) {
          if (fsig < 32)
            lb0 = nb;
          else
            lb1 = nb;
        }
      }
      if (rbit && scanned && lbr == lb) {
        const int nb = sc.first_rclear >= 0 ? sc.first_rclear : nC;
        if (lane == (rv & 31)) {
          if (rv < 32)
            lr0 = nb;
          else
            lr1 = nb;
        }
      }
      if (found && coh_moved) {
        // the cohort rearranged [coh_w0, coh_gE]: a bound inside follows the claims that stayed (all of them rejected its
        // signature before; the ones that moved went behind them)
        const int w0 = coh_w0, gE = coh_gE;
#define KP_COH_ADJ(b)                                                          \
  if ((b) > w0 && (b) <= gE) {                                                 \
    const int nb_ = (b) - w0;                                                  \
    (b) -= __popc(coh_moved & (nb_ >= 32 ? FULL : (1u << nb_) - 1u));          \
  }
        KP_COH_ADJ(lb0)
        KP_COH_ADJ(lb1)
        KP_COH_ADJ(lr0)
        KP_COH_ADJ(lr1)
#undef KP_COH_ADJ
      }
      if (found && coh_extra > 0) {  // the rest of the cohort left the queue together with its first pod
        commits += coh_extra;
        watchdog += coh_extra;
        scan_chunks += coh_extra + 1;  // (reported as cohort_pods)
        if (E > 0) ev_existing += (long long)coh_extra * n_active_nodes;
        head += coh_extra;
        hq += coh_extra;
        if (hq >= cap) hq -= cap;
        if (STAGED) {
          if (lane == 0) ring->skip_to = head;
        }
      }
      if (found) {
        commits++;
        continue;
      }
      ev_inflight += nC;
    }

    // ================= addToNewNodeClaim (scheduler.go:592-684) =================
    int err = alive_tmpl ? KP_PODERR_INCOMPATIBLE : KP_PODERR_NO_TEMPLATES;
    for (int n = 0; n < d.N && !found; n++) {
      uint64_t tw = lane < ITW ? d.tmpl_its[(size_t)n * ITW + lane] : 0ull;
      const bool alive = __any_sync(FULL, tw != 0);  // NewScheduler drops templates whose prefilter is empty
      if (!alive) continue;
      ev_tmpl++;
      const uint32_t lp = d.tmpl_limit_present[n];
      if (lp) {  // limits: scheduler.go:605-623, filterByRemainingResources :860-876
        if (d.nodes_res >= 0 && (lp >> d.nodes_res & 1) && I.tmpl_remaining[(size_t)n * R + d.nodes_res] == 0) continue;
        if (lane < ITW) {
          uint64_t keep = 0;
          for (uint64_t bits = tw; bits;) {
            const int b = __ffsll((long long)bits) - 1;
            bits &= bits - 1;
            const int t = lane * 64 + b;
            bool viable = true;
            for (int r = 0; r < R; r++)
              if ((lp >> r & 1) && d.it_capacity[(size_t)t * R + r] > I.tmpl_remaining[(size_t)n * R + r]) viable = false;
            if (viable) keep |= 1ull << b;
          }
          tw = keep;
        }
        if (!__any_sync(FULL, tw != 0)) continue;
      }
      const int cnew = nC;
      if (cnew >= I.Cmax) {
        status = KP_ERR_CAPACITY;
        break;
      }
      if (!((px.tmpl_ok >> n) & 1ull)) continue;
      if (!LEAN && px.port_conf && (d.tmpl_ports[n] & px.port_conf)) continue;  // the daemons' ports (scheduler.go:794-811)
      if (I.CS && cnew >= I.CS) {  // the shared-memory copies are full: continue on the global arrays
        migrate_small(d, I, nC, lane);
        ord = I.order;
        cnt = I.cnt_at;
      }
      Slot b = lane < K ? rs_slot(d, d.tmpl_rs[n], lane) : slot_absent();
      const int64_t bq = lane < R ? d.tmpl_daemon[(size_t)n * R + lane] : 0;
      Eval ev;
      unsigned long long take = 0;
      bool rerr = false, alt_loaded = false;
      for (int alt = -1;;) {
        ev = eval_candidate<LEAN>(d, px, true, b, bq, tw, -1, E + cnew, scratch, lane);
        if (!LEAN && d.mv_strict && ev.ok && !min_values_ok(d, n, ev.its, lane)) ev.ok = false;
        take = 0;
        rerr = false;
        if (!LEAN && d.n_rsv && ev.ok) {
          if (lane < K) scratch[lane] = ev.F;
          __syncwarp();
          take = offerings_to_reserve(d, I.rsv_cap, scratch, ev.its, 0ull, lane, &rerr);
          __syncwarp();
          if (rerr) ev.ok = false;
        }
        if (!VOL || ev.ok) break;
        alt = alt < 0 ? px.vol_next : next_alt(d, alt);  // the other volume-topology alternatives: the last one's error counts
        if (alt < 0) break;
        load_alt_slots(d, pxw, alt, lane);
        alt_loaded = true;
      }
      if (VOL && alt_loaded && !ev.ok) load_alt_slots(d, pxw, Xc, lane);
      if (rerr) {
        // compatible reserved capacity of this NodePool is taken: no NodePool of lower weight may take the pod
        // (scheduler.go:632-646), and the pod is not relaxed either (:447-453)
        err = KP_PODERR_RESERVED;
        break;
      }
      if (!ev.ok) continue;
      // NewNodeClaim + Add
      claim_store<LEAN>(d, I, cnew, lane, ev, true);
      if (lane == 0) {
        I.c_tmpl[cnew] = n;
        ord[cnew] = cnew;
        cnt[cnew] = 1;
        if (I.pod_target) {
          I.pod_target[li] = KP_TARGET_CLAIM(cnew);
          I.pod_error[li] = KP_PODERR_NONE;
        }
      }
      // a recycled instance must not inherit failure bits of an earlier claim with this id
      if (lane == 0) {
        I.cmask[cnew] = make_ulonglong2(0ull, 0ull);
        I.amask[cnew] = ((px.tkinfo & TKI_ABIT) && ev.pod_noop) ? 1ull << (px.tkinfo & 63) : 0ull;
        if (!LEAN && d.n_rsv) I.c_rsv[cnew] = take;
        if (!LEAN && d.n_hostports) I.c_ports[cnew] = d.tmpl_ports[n] | px.ports;
      }
      if (!LEAN && d.n_rsv) reservations_commit(d, I.rsv_cap, 0ull, take, lane);
      // subtractMax (scheduler.go:840-857): remaining -= max capacity over the claim's instance types
      if (lp) {
        for (int r = 0; r < R; r++) {
          if (!(lp >> r & 1)) continue;
          long long mx = 0;
          if (lane < ITW)
            for (uint64_t bits = ev.its; bits;) {
              const int bb = __ffsll((long long)bits) - 1;
              bits &= bits - 1;
              const long long capv = d.it_capacity[(size_t)(lane * 64 + bb) * R + r];
              if (capv > mx) mx = capv;
            }
          for (int o = 16; o; o >>= 1) {
            const long long other = __shfl_xor_sync(FULL, mx, o);
            if (other > mx) mx = other;
          }
          if (lane == 0) I.tmpl_remaining[(size_t)n * R + r] -= mx;
        }
      }
      // Topology.Register(hostname) (nodeclaim.go:213): every hostname group learns the new, empty domain
      if (!LEAN && d.GH > 0) {
        for (int g = lane; g < d.G; g += 32)
          if (d.groups[g].key == d.hostname_key) {
            d.g_ndomains[g]++;
            d.g_nempty[g]++;
          }
        __syncwarp();
      }
      if (!LEAN) topo_record(d, px, ev.F, d.tmpl_taintset[n], E + cnew, true, lane);
      __syncwarp();
      nC = cnew + 1;
      pert = PERT_APPEND;
      pert_pos = cnew;
      found = true;
      commits++;
    }
    if (status != KP_OK) break;
    if (!found) {
      const int nx = err == KP_PODERR_RESERVED ? -1 : px.relax;  // staged with the class row: cls_relax[Xc]
      if (nx >= 0) {  // Preferences.Relax dropped one soft constraint (preferences.go:38-57): same pod, next class row
        Xc = nx;
        // Topology.Update of the relaxed pod (scheduler.go:462): groups only relaxed pods own come into being now
        for (int i = d.cls_lazy_off[nx]; !LEAN && i < d.cls_lazy_off[nx + 1]; i++) {
          const int g = d.cls_lazy[i];
          if (d.g_born[g]) continue;
          if (lane == 0) {
            d.g_born[g] = 1;
            d.g_birth[g] = n_born;
          }
          n_born++;
          __syncwarp();
        }
        ClassRegs cur = load_class_regs(d, Xc, li, lane);
        __syncwarp();
        store_class_regs(d, pxw, cur, lane);
        __syncwarp();
        goto try_pod;
      }
      // scheduler.go:415-421: record the error and requeue the ORIGINAL pod
      if (lane == 0) {
        if (I.pod_target) {
          I.pod_error[li] = (uint8_t)err;
          I.pod_target[li] = KP_TARGET_UNSCHEDULED;
        }
        I.queue[tq] = li;
        I.qcls[tq] = X;
        I.last_len[li] = tail + 1 - head;
      }
      tail++;
      tq = tq + 1 >= cap ? tq + 1 - cap : tq + 1;
      if (STAGED) {
        __threadfence_block();
        if (lane == 0) ring->tail_pub = tail;
      }
      __syncwarp();
    }
  }
  if (STAGED) {
    __syncwarp();
    if (lane == 0) ring->done = 1;
  }
  // len(Pods) of every claim is the count stored next to it in the claim order
  for (int i = lane; i < nC; i += 32) I.c_npods[ord[i]] = cnt[i];
  // pods still queued when the loop ends are the PodErrors (scheduler.go:415-423); a simulation ignores the errors of
  // provisionable pending pods (AllNonPendingPodsScheduled, scheduler.go:330-334)
  n_unsched = tail - head;
  if (I.pod_kind && n_unsched > 0) {
    int keep = 0;
    for (int i = head + lane; i < tail; i += 32) keep += I.pod_kind[I.queue[i % cap]] != KP_EXTRA_PENDING;
    for (int o = 16; o; o >>= 1) keep += __shfl_xor_sync(FULL, keep, o);
    n_unsched = keep;
  }
  if (lane == 0) {
    I.n_claims = nC;
    I.n_unsched = n_unsched;
    I.n_uninit = n_uninit;
    I.status = status;
    I.ev_existing = ev_existing;
    I.ev_inflight = ev_inflight;
    I.ev_tmpl = ev_tmpl;
    I.commits = commits;
    I.slow_sorts = slow_sorts;
    I.scan_chunks = scan_chunks;
    I.evals = evals;
    I.fast_commits = fast_commits;
  }
  __syncwarp();
}
