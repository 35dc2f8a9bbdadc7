// kp_consolidate.cuh -- launchable kernels around the warp solver (kp_wsolve.cuh):
//
//   k_node_cand     existing-node candidate bitmaps: for every (class signature | request vector) x node one bit.
//                   Streams the node table once per signature tile -- the HBM-bound, embarrassingly parallel part.
//   k_wsolve_batch  Scheduler.Solve: one CTA per instance (n >= 1); order / failure bitmaps / staged tables in shared
//                   memory.
//   k_consolidate   disruption.SimulateScheduling + computeConsolidation (helpers.go:51-142, consolidation.go:136-229)
//                   for every candidate subset: one warp per subset pulled from a global counter, 8 warps per CTA, all
//                   SMs busy; the cluster's node table is shared read-only, each warp keeps the nodes its simulation
//                   touched in a private overlay.
//
// Each memory layout a host sizes and a kernel carves is written out once, here: the staged read-only tables
// (KP_STAGED_TABLES), the solver CTA's shared memory (SolveSmem) and k_consolidate's per-warp scratch
// (KP_CONSOL_SCRATCH).
#pragma once
#include "kp_wsolve.cuh"

#define KP_ALIGN16(x) (((x) + 15) & ~(size_t)15)

// The read-only tables a kernel stages in shared memory, in order: field, element type, element count in the
// dimensions of the KpDev `d`.  Each table starts 16-byte aligned.  kp_tab_bytes sizes them, stage_tables copies them.
#define KP_STAGED_TABLES(X, d)                                    \
  X(key_wellknown, uint8_t, d.K)                                  \
  X(key_univ, uint64_t, d.K)                                      \
  X(val_isint, uint64_t, d.K)                                     \
  X(ge_off, int32_t, (size_t)d.R + 1)                             \
  X(ge_vals, int64_t, d.n_ge)                                     \
  X(ge_bits, uint64_t, (size_t)d.n_ge * d.ITW)                    \
  X(itv_off, int32_t, (size_t)d.K + 1)                            \
  X(itv, uint64_t, (size_t)d.n_itv * d.ITW)                       \
  X(it_nokey, uint64_t, (size_t)d.K * d.ITW)                      \
  X(it_dne, uint64_t, (size_t)d.K * d.ITW)                        \
  X(it_nonempty, uint64_t, (size_t)d.K * d.ITW)                   \
  X(it_valid, uint64_t, d.ITW)                                    \
  X(off_slots, Slot, (size_t)(d.D > 0 ? d.D : 1) * d.K)           \
  X(off_keys, uint32_t, d.D > 0 ? d.D : 1)                        \
  X(offset_bits, uint64_t, (size_t)(d.D > 0 ? d.D : 1) * d.ITW)   \
  X(tmpl_taintset, int32_t, d.N > 0 ? d.N : 1)                    \
  X(nfit_sum, uint32_t, (size_t)d.n_rv * d.ESW)                   \
  X(nstat_sum, uint32_t, (size_t)d.n_nsig * d.ESW)

// bytes of the staged tables
__host__ __device__ inline size_t kp_tab_bytes(const KpDev& d) {
  size_t b = 0;
#define KP_TAB_BYTES(field, type, count) b += KP_ALIGN16(sizeof(type) * (size_t)(count));
  KP_STAGED_TABLES(KP_TAB_BYTES, d)
#undef KP_TAB_BYTES
  return b;
}

// Copy the pointer block to shared memory and, when they fit, the staged tables next to it; patches the pointers.  All
// threads of the CTA.
__device__ __forceinline__ void stage_tables(const KpDev& d_in, KpDev* ds, unsigned char* tab) {
  const int tid = threadIdx.x, nt = blockDim.x;
  {
    const int* src = reinterpret_cast<const int*>(&d_in);
    int* dst = reinterpret_cast<int*>(ds);
    for (int i = tid; i < (int)(sizeof(KpDev) / 4); i += nt) dst[i] = src[i];
  }
  __syncthreads();
  if (d_in.tab_bytes > 0) {
    size_t off = 0;
#define KP_STAGE(field, type, count)                                     \
  {                                                                      \
    size_t n_ = (size_t)(count);                                         \
    type* dst_ = reinterpret_cast<type*>(tab + off);                     \
    const type* src_ = d_in.field;                                       \
    for (size_t i_ = tid; i_ < n_; i_ += nt) dst_[i_] = src_[i_];        \
    if (tid == 0) ds->field = dst_;                                      \
    off += KP_ALIGN16(sizeof(type) * n_);                                \
  }
    KP_STAGED_TABLES(KP_STAGE, d_in)
#undef KP_STAGE
  }
  __syncthreads();
}

// ---------------------------------------------------------------------------------------------------------------
// Candidate bitmaps over existing nodes.  Row y < n_nsig: class signature (requirements, tolerations) -- taints
// tolerated (taints.go:49-66) and no key the node defines has an empty intersection with the pod's requirement
// (requirements.go:254-274); an undefined key passes unless `strict_undefined` (no pod can ever define a key on a
// node, so the strict Compatible of existingnode.go:89 would fail forever).  Row n_nsig + rv: resources.Fits of the
// request vector (resources.go:150-163).  Both are monotone supersets of "CanAdd succeeds".
__global__ void __launch_bounds__(256) k_node_cand(KpDev d, const int32_t* nsig_rs, const int32_t* nsig_tolset,
                                                    const int64_t* rv_req, int strict_undefined) {
  const int n = blockIdx.x * blockDim.x + threadIdx.x, row = blockIdx.y, lane = threadIdx.x & 31;
  bool bit = false;
  if (n < d.E) {
    if (row < d.n_nsig) {
      bit = tolerated(d, nsig_tolset[row], d.node_taintset[n]);
      const int rs = nsig_rs[row];  // -1: a class with volume-topology alternatives -- every tolerated node is a candidate
      if (rs >= 0 && bit) bit = host_rule_admits(d.host_rules, d.E, rs, n);  // exact on the hostname key
      for (int k = 0; rs >= 0 && k < d.K && bit; k++) {
        Slot pod = rs_slot(d, rs, k);
        if (!slot_present(pod)) continue;
        Slot nd = load_slot(d.node_sflags, d.node_smask, d.node_sgte, d.node_slte, (size_t)n * d.K + k, d.has_bounds);
        if (!slot_present(nd)) {
          if (strict_undefined && !op_is_negative(slot_op(pod))) bit = false;
        } else if (!slot_has_intersection(key_info(d, k), nd, pod) &&
                   !(op_is_negative(slot_op(pod)) && op_is_negative(slot_op(nd)))) {
          bit = false;
        }
      }
    } else {
      const int rv = row - d.n_nsig;
      const uint32_t pr = d.node_rem_present[n];
      bit = true;
      for (int r = 0; r < d.R; r++) {
        const int64_t rem = d.node_rem[(size_t)n * d.R + r];
        const bool present = (pr >> r) & 1;
        if (present && rem < 0) bit = false;
        if (rv_req[(size_t)rv * d.R + r] > (present ? rem : 0)) bit = false;
      }
    }
  }
  const unsigned m = __ballot_sync(FULL, bit);
  const int w = n >> 5;
  if (lane == 0 && w < d.EW) {
    if (row < d.n_nsig)
      d.nstat[(size_t)row * d.EW + w] = m;
    else
      d.nfit[(size_t)(row - d.n_nsig) * d.EW + w] = m;
  }
}

// word-level summaries of the candidate bitmaps: bit w of summary word s <=> bitmap word 32*s+w (masked by nactive for
// the Fits rows) is non-zero.  One thread per summary word.
__global__ void __launch_bounds__(256) k_node_sum(KpDev d) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x, rows = d.n_rv + d.n_nsig;
  if (i >= rows * d.ESW) return;
  const int row = i / d.ESW, s = i % d.ESW;
  const uint32_t* src = row < d.n_rv ? d.nfit + (size_t)row * d.EW : d.nstat + (size_t)(row - d.n_rv) * d.EW;
  uint32_t out = 0;
  for (int w = 0; w < 32; w++) {
    const int idx = s * 32 + w;
    if (idx < d.EW && (src[idx] & d.nactive[idx])) out |= 1u << w;
  }
  if (row < d.n_rv)
    d.nfit_sum[(size_t)row * d.ESW + s] = out;
  else
    d.nstat_sum[(size_t)(row - d.n_rv) * d.ESW + s] = out;
}

// ---------------------------------------------------------------------------------------------------------------
// Scheduler.Solve, one instance.
struct WSolveShared {
  KpDev ds;
  WInst inst;
  StageRing ring;
  Slot scratch[KP_MAXK];
};

// The solver CTA's dynamic shared memory: byte offset of every region and the total.  In order: the WSolveShared block;
// the staged tables (tab_bytes); the state of the `ntk` groups on tk_key (slot map over all groups, registered /
// populated masks, counters with a stride of tk_nv); the hot rows of the first CQ claims (requests, threshold rows); the
// cold rows of the first CR (requirement masks, instance-type words, slot flags); the small arrays of the first CS
// (failure masks, order, counts, template ids, c_dom).  An absent region takes no bytes.  plan_solve sizes the plan
// with it, wsolve_cta carves its shared memory with it.
struct SolveSmem {
  size_t tab, tk_slot, tk_reg, tk_pop, tk_cnt, s_req, s_j, s_smask, s_its, s_sflags, pmask, amask, order, cnt_at, c_tmpl,
      c_dom, total;
  __host__ __device__ SolveSmem(const KpDev& d, size_t tab_bytes, int CS, int CQ, int CR, int ntk) {
    size_t o = KP_ALIGN16(sizeof(WSolveShared));
    auto at = [&o](size_t& r, size_t bytes) {
      r = o;
      o += bytes;
    };
    at(tab, tab_bytes);
    const size_t tk = ntk > 0 ? ntk : 0, q = CQ > 0 ? CQ : 0, c = CR > 0 ? CR : 0, s = CS > 0 ? CS : 0;
    at(tk_slot, tk ? KP_ALIGN16((size_t)d.G * 4) : 0);
    at(tk_reg, KP_ALIGN16(tk * 8));
    at(tk_pop, KP_ALIGN16(tk * 8));
    at(tk_cnt, KP_ALIGN16(tk * d.tk_nv * 4));
    at(s_req, KP_ALIGN16(q * d.R * 8));
    at(s_j, KP_ALIGN16(q * d.R * 4));
    at(s_smask, KP_ALIGN16(c * d.K * 8));
    at(s_its, KP_ALIGN16(c * d.ITW * 8));
    at(s_sflags, KP_ALIGN16(c * d.K));
    at(pmask, s * 16);
    at(amask, s * 8);
    at(order, s * 4);
    at(cnt_at, s * 4);
    at(c_tmpl, s * 4);
    at(c_dom, s);
    total = o + 64;
  }
};

// warp 0: the solver; warp 1: the pod stager (see StageRing)
template <bool LEAN, bool COHORT, bool VOL>
__device__ __forceinline__ void wsolve_cta(const KpDev& d_in, int CS, int CQ, int CR, int ntk) {
  extern __shared__ __align__(16) unsigned char smem_raw[];
  WSolveShared& sh = *reinterpret_cast<WSolveShared*>(smem_raw);
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  stage_tables(d_in, &sh.ds, smem_raw + SolveSmem(d_in, 0, 0, 0, 0, 0).tab);
  const KpDev& d = sh.ds;
  WInst& I = sh.inst;
  const SolveSmem L(d, d.tab_bytes, CS, CQ, CR, ntk);
  int32_t* s_slot = nullptr;
  uint64_t *s_reg = nullptr, *s_pop = nullptr;
  int32_t* s_cnt = nullptr;
  if (ntk > 0) {  // the state of the groups on the topology key, numbered in group order (warp 0)
    const int nv = d_in.tk_nv;
    s_slot = reinterpret_cast<int32_t*>(smem_raw + L.tk_slot);
    s_reg = reinterpret_cast<uint64_t*>(smem_raw + L.tk_reg);
    s_pop = reinterpret_cast<uint64_t*>(smem_raw + L.tk_pop);
    s_cnt = reinterpret_cast<int32_t*>(smem_raw + L.tk_cnt);
    if (warp == 0) {
      for (int base = 0, n = 0; base < d_in.G; base += 32) {
        const int g = base + lane;
        const KpGroup* G_ = g < d_in.G ? d_in.groups + g : nullptr;
        const bool on = G_ && G_->key == d_in.tk_key;
        const unsigned m = __ballot_sync(FULL, on);
        const int s = n + __popc(m & ((1u << lane) - 1));
        if (g < d_in.G) s_slot[g] = on ? s : -1;
        if (on) {
          s_reg[s] = d_in.dom_reg[g];
          s_pop[s] = d_in.dom_pop[g];
          for (int v = 0; v < nv; v++) s_cnt[s * nv + v] = d_in.dom_cnt[G_->dom_off + v];
        }
        n += __popc(m);
      }
    }
  }
  const int Cmax = d.Cmax;
  if (threadIdx.x == 0) {
    sh.ring.produced = 0;
    sh.ring.consumed = 0;
    sh.ring.tail_pub = (int)d.P;
    sh.ring.done = 0;
    sh.ring.skip_to = 0;
    I.P = (int)d.P;
    I.queue = d.queue;
    I.qcls = d.qcls;
    I.last_len = d.last_len;
    I.pod_target = d.pod_target;
    I.pod_error = d.pod_error;
    I.pod_kind = d.pod_kind;
    I.Cmax = Cmax;
    I.c_tmpl = d.c_tmpl;
    I.c_npods = d.c_npods;
    I.c_req = d.c_req;
    I.c_sflags = d.c_sflags;
    I.c_smask = d.c_smask;
    I.c_sgte = d.c_sgte;
    I.c_slte = d.c_slte;
    I.c_its = d.c_its;
    I.c_j = d.c_j;
    I.order = d.order;
    I.cnt_at = d.cnt_at;
    I.pmask = d.pmask;
    I.amask = d.amask;
    I.tmpl_remaining = d.tmpl_remaining;
    I.n_removed = 0;
    I.removed = nullptr;
    I.ov_cap = 0;
    I.n_ov = 0;
    I.CS = 0;
    I.c_dom = d.c_dom;
    I.rsv_cap = d.rsv_cap;
    I.c_rsv = d.c_rsv;
    I.c_ports = d.c_ports;
    I.ov_ports = nullptr;
    I.CQ = 0;
    I.CR = 0;
    if (ntk > 0) {
      sh.ds.tk_slot = s_slot;
      sh.ds.tk_reg = s_reg;
      sh.ds.tk_pop = s_pop;
      sh.ds.tk_cnt = s_cnt;
    }
    if (CQ > 0) {  // hot rows of the first CQ claims
      I.s_req = reinterpret_cast<int64_t*>(smem_raw + L.s_req);
      I.s_j = reinterpret_cast<int32_t*>(smem_raw + L.s_j);
      I.CQ = CQ;
    }
    if (CR > 0) {  // cold rows of the first CR claims
      I.s_smask = reinterpret_cast<uint64_t*>(smem_raw + L.s_smask);
      I.s_its = reinterpret_cast<uint64_t*>(smem_raw + L.s_its);
      I.s_sflags = reinterpret_cast<uint8_t*>(smem_raw + L.s_sflags);
      I.CR = CR;
    }
    if (CS > 0) {  // claim order, template ids and the failure masks of the first CS claims live in shared memory
      I.pmask = reinterpret_cast<ulonglong2*>(smem_raw + L.pmask);
      I.amask = reinterpret_cast<unsigned long long*>(smem_raw + L.amask);
      I.order = reinterpret_cast<int32_t*>(smem_raw + L.order);
      I.cnt_at = reinterpret_cast<int32_t*>(smem_raw + L.cnt_at);
      I.c_tmpl = reinterpret_cast<int32_t*>(smem_raw + L.c_tmpl);
      I.c_dom = reinterpret_cast<uint8_t*>(smem_raw + L.c_dom);
      I.CS = CS;
    }
  }
  __syncthreads();
  if (warp == 1) {
    stager_run<COHORT>(d, I, &sh.ring, lane);
    return;
  }
  wsolve_run<false, LEAN, COHORT, VOL>(d, I, sh.ring.slot[0], sh.scratch, lane, &sh.ring);
  const int nC = I.n_claims;
  claim_rows_flush(d, I, nC, lane);
  if (ntk > 0) {  // before k_scatter_counts, the counter all-reduce and the download read them
    for (int g = lane; g < d.G; g += 32) {
      const int s = s_slot[g];
      if (s < 0) continue;
      d_in.dom_reg[g] = s_reg[s];
      d_in.dom_pop[g] = s_pop[s];
      for (int v = 0; v < d.tk_nv; v++) d_in.dom_cnt[d_in.groups[g].dom_off + v] = s_cnt[s * d.tk_nv + v];
    }
    __syncwarp();
  }
  if (!LEAN) claims_finalize(d, I.c_sflags, I.c_smask, I.c_rsv, nC, lane);
  if (I.CS > 0) {  // the host reads the final order (claim_rank) and template ids from global memory
    for (int i = lane; i < nC; i += 32) {
      d_in.order[i] = I.order[i];
      d_in.cnt_at[i] = I.cnt_at[i];
      d_in.c_tmpl[i] = I.c_tmpl[i];
    }
  }
  if (lane == 0) {
    *d.n_claims = nC;
    *d.status = I.status;
    d.counters[0] = I.ev_existing;
    d.counters[1] = I.ev_inflight;
    d.counters[2] = I.ev_tmpl;
    d.counters[3] = I.commits;
    d.counters[4] = I.slow_sorts;
    d.counters[5] = I.scan_chunks;
    d.counters[6] = I.evals;
    d.counters[7] = I.n_unsched;
    d.counters[8] = I.n_uninit;
    d.counters[9] = I.fast_commits;
#ifdef KP_PHASE_PROF
    for (int p = 0; p < KP_NPHASE; p++) d.counters[KP_PROF_AT + p] = I.prof[p];
    d.counters[KP_PROF_AT + KP_NPHASE] = I.prof_total;
    d.counters[KP_PROF_AT + KP_NPHASE + 1] = I.scan_steps;
    d.counters[KP_PROF_AT + KP_NPHASE + 2] = I.scan_pos;
    d.counters[KP_PROF_AT + KP_NPHASE + 3] = I.scan_first_cyc;
#endif
  }
}
// Scheduler instances in one launch, one CTA (== one SM) each: a single provisioning solve (a batch of one), NodePool
// shards of a provisioning pass, or the candidate sets of a consolidation pass whose pods carry topology constraints
// (SimulateScheduling, helpers.go:51-142).  Instances share nothing but the device; plan[b] = {CS, CQ, CR, groups on the
// topology key whose state is on chip (0: none)} of instance b.
template <bool LEAN, bool COHORT, bool VOL = false>
__global__ void __launch_bounds__(64, 1) k_wsolve_batch(const KpDev* __restrict__ devs, const int4* __restrict__ plan) {
  const int4 pl = plan[blockIdx.x];
  // (the lean and cohort instantiations leave the topology-key state in global memory: the code to stage it costs their
  // register allocation more than it saves)
  wsolve_cta<LEAN, COHORT, VOL>(devs[blockIdx.x], pl.x, pl.y, pl.z, LEAN || COHORT ? 0 : pl.w);
}

// ---------------------------------------------------------------------------------------------------------------
// Consolidation.

// k_consolidate's per-warp scratch, in allocation order: field, element type, elements per warp slot in the dimensions
// of the KpDev `d` and the KpConsol `q`, whether the pass needs it.  The host allocates slots x count of each field it
// needs (one array per field); consol_slot points warp `slot` at elements [slot * count, (slot + 1) * count) of each,
// null where the pass lacks the field.  KP_SORT_SCRATCH is what consol_decide uses: the instance types of the single new
// NodeClaim in price order (sort keys / ids) and a bitmap; the general path allocates it alone, one slot per instance.
#define KP_SORT_SCRATCH(X, d, q)                                     \
  X(sort_key, double, q.T, true)                                     \
  X(sort_val, int32_t, q.T, true)                                    \
  X(sort_bits, unsigned long long, d.ITW, true)
#define KP_CONSOL_SCRATCH(X, d, q)                                   \
  X(queue, int32_t, (size_t)q.capq + 1, true)                        \
  X(qcls, int32_t, (size_t)q.capq + 1, true)                         \
  X(last_len, int32_t, q.capq, true)                                 \
  X(clsl, int32_t, q.capq, true)                                     \
  X(rk, int32_t, q.capq, true)                                       \
  X(kindl, uint8_t, q.capq, q.n_extra > 0) /* kind of local pod i, 0: candidate pod */ \
  X(rsv_cap, int32_t, d.n_rsv, d.n_rsv > 0) /* the simulation's own ReservationManager */ \
  X(c_rsv, unsigned long long, q.capq, d.n_rsv > 0)                  \
  X(c_ports, unsigned long long, q.capq, d.n_hostports > 0) /* host ports of the claims / touched nodes */ \
  X(ov_ports, unsigned long long, q.capq, d.n_hostports > 0)         \
  X(c_tmpl, int32_t, q.capq, true)                                   \
  X(c_npods, int32_t, q.capq, true)                                  \
  X(order, int32_t, q.capq, true)                                    \
  X(cnt_at, int32_t, q.capq, true)                                   \
  X(c_req, int64_t, (size_t)q.capq * d.R, true)                      \
  X(c_sflags, uint8_t, (size_t)q.capq * d.K, true)                   \
  X(c_smask, uint64_t, (size_t)q.capq * d.K, true)                   \
  X(c_its, uint64_t, (size_t)q.capq * d.ITW, true)                   \
  X(c_j, int32_t, (size_t)q.capq * d.R, true)                        \
  KP_SORT_SCRATCH(X, d, q)                                           \
  X(pmask, ulonglong2, q.capq, true)                                 \
  X(amask, unsigned long long, q.capq, true)                         \
  X(tmpl_remaining, int64_t, (size_t)(d.N > 0 ? d.N : 1) * d.R, true) \
  X(ov_node, int32_t, q.capq, true)                                  \
  X(ov_rem, int64_t, (size_t)q.capq * d.R, true)                     \
  X(ov_present, uint32_t, q.capq, true)                              \
  X(ov_sflags, uint8_t, (size_t)q.capq * d.K, true)                  \
  X(ov_smask, uint64_t, (size_t)q.capq * d.K, true)                  \
  X(c_sgte, int64_t, (size_t)q.capq * d.K, d.has_bounds)             \
  X(c_slte, int64_t, (size_t)q.capq * d.K, d.has_bounds)             \
  X(ov_sgte, int64_t, (size_t)q.capq * d.K, d.has_bounds)            \
  X(ov_slte, int64_t, (size_t)q.capq * d.K, d.has_bounds)
struct ConsolScratch {
#define KP_SCRATCH_FIELD(f, type, count, present) type* f;
  KP_CONSOL_SCRATCH(KP_SCRATCH_FIELD, , )
#undef KP_SCRATCH_FIELD
};

struct KpConsol {
  // inputs
  int n_subsets;
  const int32_t* subset_off;
  const int32_t* subset_nodes;
  const int32_t* node_pod_off;   // [E+1] rows of the cluster's pod table bound to node i
  const int32_t* pod_class;      // [rows]
  const int32_t* pod_rank;       // [rows] position in byCPUAndMemoryDescending order over all rows
  const double* node_price;      // [E] cheapest compatible offering of the node's instance type, < 0: none
  const uint8_t* node_is_spot;   // [E]
  const int32_t* node_it;        // [E] instance type of the node, -1 unknown
  int filter_same_type;          // apply filterOutSameInstanceType to replacements of >= 2 nodes
  const int32_t* node_tmpl;      // [E] NodePool of the node, -1 unmanaged
  const int64_t* node_capacity;  // [E*R]
  const int64_t* tmpl_remaining0;// [N*R] limits minus capacity of ALL nodes
  // WorstLaunchPrice lists: for instance type t and capacity type i (reserved, spot, on-demand) the AVAILABLE offerings
  // whose requirement set admits that capacity type, most expensive first -- the first entry whose set is compatible
  // with the claim's requirements is the answer (types.go:480-491)
  const int32_t* wl_off;         // [T*3+1]
  const int32_t* wl_set;         // distinct offering requirement set of the entry
  const double* wl_price;
  // OrderByPrice lists (types.go:238-257): the AVAILABLE offerings of instance type t, cheapest first -- the first entry
  // whose set is compatible with the requirements is the sort key
  const int32_t* ml_off;         // [T+1]
  const int32_t* ml_set;
  const double* ml_price;
  int T;
  int ct_key, ct_spot, ct_od, ct_order_valid;  // bit i of ct_order_valid: ct_order[i] is interned
  int spot_to_spot_enabled;
  // pods every simulation schedules besides the candidates' (helpers.go:65-91): rows extra_row0 .. extra_row0+n_extra-1
  int n_extra, extra_row0;
  const uint8_t* extra_kind;     // [n_extra] KP_EXTRA_*
  // context deadline: the first warp to start stamps t_start; a warp that finds deadline_ns used up stops pulling work
  long long deadline_ns;
  unsigned long long* t_start;
  int capq;                      // pods / claims / overlay entries an instance can hold
  ConsolScratch ws;              // per warp slot scratch (KP_CONSOL_SCRATCH): the arrays of all slots
  // outputs
  uint8_t* decision;             // [n_subsets] KP_DECISION_*, 255 = needs a feature that is not built
  uint64_t* replacement_its;     // [n_subsets * ITW]
  int32_t* n_new_claims;
  int32_t* n_unscheduled;
  // the replacement NodeClaim of a REPLACE: template, requests, requirement slots after the capacity-type pins
  int32_t* repl_tmpl;            // [n_subsets]
  int64_t* repl_req;             // [n_subsets * R]
  uint8_t* repl_sflags;          // [n_subsets * K]
  uint64_t* repl_smask;
  int64_t *repl_sgte, *repl_slte;
  int export_order;              // also write the price order of the replacement's instance types
  int32_t* repl_order;           // [n_subsets * order_cap] (order_cap = min(T, 600)), repl_order_n[s] entries used
  int32_t* repl_order_n;
  int order_cap;
  int32_t* next;                 // work counter
  int32_t* status;
};

// warp slot `slot`'s share of the per-warp scratch
__device__ __forceinline__ ConsolScratch consol_slot(const KpDev& d, const KpConsol& q, size_t slot) {
  ConsolScratch w;
#define KP_SCRATCH_SLOT(f, type, count, present) w.f = (present) ? q.ws.f + slot * (size_t)(count) : nullptr;
  KP_CONSOL_SCRATCH(KP_SCRATCH_SLOT, d, q)
#undef KP_SCRATCH_SLOT
  return w;
}

// computeConsolidation (consolidation.go:136-229) for one simulated candidate set: `unscheduled` pods could not be
// placed (or only on uninitialized nodes), `n_new` NodeClaims were opened; claim 0's row (requirement slots, instance
// types) is read through the c_* pointers.  One warp; `slot` selects the warp's sort scratch in q; result row `s`.
// OrderByPrice lists of the catalog: the available offerings of every instance type, cheapest first, with the offering
// requirement set each belongs to (host-built; shared by the consolidation decision and Results.TruncateInstanceTypes)
struct PriceTabs {
  const int32_t* ml_off;   // [T+1]
  const int32_t* ml_set;
  const double* ml_price;
};
// InstanceTypes.OrderByPrice (types.go:238-257) of the types in `cur` (lane w: word w of the bitmap; n_its of them) under
// the requirements whose compatible offering sets are `okmask`: sk / sv receive (price, type) in the order Go's sort.Slice
// leaves them, starting from the provider order (ascending type index).
__device__ __forceinline__ void order_by_price(const PriceTabs& pt, uint64_t cur, int n_its, unsigned okmask, double* sk,
                                               int32_t* sv, int ITW, int lane) {
  const int cw = lane < ITW ? __popcll(cur) : 0;
  int pre = cw;
  for (int o = 1; o < 32; o <<= 1) {
    const int t = __shfl_up_sync(FULL, pre, o);
    if (lane >= o) pre += t;
  }
  int at = pre - cw;
  for (uint64_t bits = lane < ITW ? cur : 0ull; bits;) {
    const int b = __ffsll((long long)bits) - 1;
    bits &= bits - 1;
    const int t = lane * 64 + b;
    double mp = 1.7976931348623157e308;
    for (int e = pt.ml_off[t]; e < pt.ml_off[t + 1]; e++)
      if ((okmask >> pt.ml_set[e]) & 1u) {
        mp = pt.ml_price[e];
        break;
      }
    sk[at] = mp;
    sv[at] = t;
    at++;
  }
  __syncwarp();
  WarpSorterT<double> srt{sk, sv, lane};
  srt.pdqsort(0, n_its, WarpSorterT<double>::bits_len((unsigned long long)n_its));
}
// the first n entries of sv as a bitmap (sb: ITW words of scratch); lane w returns word w
__device__ __forceinline__ uint64_t first_types_bitmap(const int32_t* sv, int n, unsigned long long* sb, int ITW, int lane) {
  if (lane < ITW) sb[lane] = 0ull;
  __syncwarp();
  for (int i = lane; i < n; i += 32) atomicOr(&sb[sv[i] >> 6], 1ull << (sv[i] & 63));
  __syncwarp();
  return lane < ITW ? sb[lane] : 0ull;
}

__device__ __forceinline__ void consol_decide(const KpDev& d, const KpConsol& q, size_t slot, Slot* scratch,
                                              const uint8_t* c_sflags, const uint64_t* c_smask, const int64_t* c_sgte,
                                              const int64_t* c_slte, const uint64_t* c_its, int c_tmpl0, const int64_t* c_req0,
                                              int c_npods0, int sn, const int32_t* snodes, int unscheduled, int n_new, int s,
                                              int lane) {
  const int K = d.K, ITW = d.ITW;
  int decision = KP_DECISION_NOOP;
  uint64_t rep = 0;  // lane w: word w of the replacement instance types
  bool have_slots = false;  // scratch[] holds the claim's requirement slots (with the spot pin when it applied)
  bool spot_pinned = false, mv_dropped = false;
  int n_ord_out = 0;
  if (!unscheduled) {
    if (n_new == 0) {
      decision = KP_DECISION_DELETE;
    } else if (n_new == 1) {
      // the single new NodeClaim: requirements (hostname already dropped), instance types
      Slot S = lane < K ? load_slot(c_sflags, c_smask, c_sgte, c_slte, (size_t)lane, d.has_bounds) : slot_absent();
      const uint64_t its = lane < ITW ? c_its[lane] : 0ull;
      int n_its = lane < ITW ? __popcll(its) : 0;
      for (int o = 16; o; o >>= 1) n_its += __shfl_xor_sync(FULL, n_its, o);
      // getCandidatePrices (consolidation.go:319-337)
      double price = 0;
      bool zero = false, all_spot = true;
      for (int i = 0; i < sn; i++) {
        const double np = q.node_price[snodes[i]];
        if (np < 0) zero = true;
        price += np;
        if (!q.node_is_spot[snodes[i]]) all_spot = false;
      }
      if (zero) price = 0.0;
      bool spot_ok = false;
      if (q.ct_key >= 0 && q.ct_spot >= 0) {
        const uint32_t f = __shfl_sync(FULL, S.f, q.ct_key);
        const uint64_t m = __shfl_sync(FULL, S.m, q.ct_key);
        const int64_t g = __shfl_sync(FULL, S.gte, q.ct_key), l = __shfl_sync(FULL, S.lte, q.ct_key);
        spot_ok = slot_has(key_info(d, q.ct_key), Slot{f, m, g, l}, q.ct_spot);
      }
      if (lane < K) scratch[lane] = S;
      __syncwarp();
      have_slots = true;
      unsigned okmask = offering_ok_mask(d, scratch, lane);
      const bool spot_path = all_spot && spot_ok;
      uint64_t cur = its;  // lane w: word w of the NodeClaim's instance types as they go through the steps below
      // ---- OrderByPrice + Truncate(600) (helpers.go:120, scheduler.go:361-379, types.go:238-257,339-351).  The order
      // only matters when it truncates, or for the 15-cheapest rule of single-node spot-to-spot consolidation.
      const ConsolScratch w = consol_slot(d, q, slot);
      double* sk = w.sort_key;
      int32_t* sv = w.sort_val;
      unsigned long long* sb = w.sort_bits;
      int n_ord = 0;
      const bool need_order = n_its > 600 || (spot_path && q.spot_to_spot_enabled) || q.export_order;
      if (need_order) {
        order_by_price(PriceTabs{q.ml_off, q.ml_set, q.ml_price}, cur, n_its, okmask, sk, sv, ITW, lane);
        n_ord = n_its;
        if (n_ord > 600) {
          n_ord = 600;
          cur = first_types_bitmap(sv, n_ord, sb, ITW, lane);
          // Truncate (types.go:339-351): the 600 cheapest must still satisfy minValues, else TruncateInstanceTypes drops the
          // NodeClaim and its pods become PodErrors (scheduler.go:361-379): not all pods scheduled, nothing to do
          if (d.mv_strict && !min_values_ok(d, c_tmpl0, cur, lane)) {
            mv_dropped = true;
            unscheduled = c_npods0;
          }
        }
      }
      if (mv_dropped) {
        decision = KP_DECISION_NOOP;
      } else if (spot_path && !q.spot_to_spot_enabled) {
        decision = KP_DECISION_NOOP;  // computeSpotToSpotConsolidation needs the feature gate (consolidation.go:239)
      } else {
        if (spot_path) {  // restrict the claim to spot (consolidation.go:252-257) and drop types without such an offering
          if (lane == q.ct_key)
            scratch[lane] = slot_add(key_info(d, lane), scratch[lane], Slot{SF_PRESENT, 1ull << q.ct_spot, 0, 0});
          spot_pinned = true;
          __syncwarp();
          okmask = offering_ok_mask(d, scratch, lane);
          uint64_t keep = 0;
          for (uint64_t bits = lane < ITW ? cur : 0ull; bits;) {
            const int b = __ffsll((long long)bits) - 1;
            bits &= bits - 1;
            const int t = lane * 64 + b;
            for (int e = q.ml_off[t]; e < q.ml_off[t + 1]; e++)
              if ((okmask >> q.ml_set[e]) & 1u) {
                keep |= 1ull << b;
                break;
              }
          }
          cur = keep;
        }
        // RemoveInstanceTypeOptionsByPriceAndMinValues (nodeclaim.go:309-318): keep WorstLaunchPrice < price
        if (lane < ITW) {
          for (uint64_t bits = cur; bits;) {
            const int b = __ffsll((long long)bits) - 1;
            bits &= bits - 1;
            const int t = lane * 64 + b;
            double worst = 1.7976931348623157e308;
            for (int ci = 0; ci < 3 && worst > 1e308; ci++) {  // reserved -> spot -> on-demand (types.go:480-491)
              if (q.ct_key < 0 || !((q.ct_order_valid >> ci) & 1)) continue;
              for (int e = q.wl_off[t * 3 + ci]; e < q.wl_off[t * 3 + ci + 1]; e++)
                if ((okmask >> q.wl_set[e]) & 1u) {
                  worst = q.wl_price[e];
                  break;
                }
            }
            if (worst < price) rep |= 1ull << b;
          }
        }
        bool any = __any_sync(FULL, rep != 0);
        // ... and SatisfiesMinValues of what is left (nodeclaim.go:314-316): an error is "Filtering by price", no command
        if (any && d.mv_strict && !min_values_ok(d, c_tmpl0, rep, lane)) any = false;
        if (any && spot_path && sn == 1) {
          // single-node spot-to-spot: at least 15 cheaper types, and only the 15 cheapest go out (consolidation.go:283-312)
          int total = lane < ITW ? __popcll(rep) : 0;
          for (int o = 16; o; o >>= 1) total += __shfl_xor_sync(FULL, total, o);
          if (total < 15) {
            any = false;
          } else {
            if (lane < ITW) sb[lane] = rep;
            __syncwarp();
            // the first n of the surviving types in price order, as a bitmap (lane w: word w)
            auto prefix_bits = [&](int n) {
              uint64_t acc = 0;
              int taken = 0;
              for (int b0 = 0; b0 < n_ord && taken < n; b0 += 32) {
                const int i = b0 + lane;
                const int t = i < n_ord ? sv[i] : 0;
                const bool in = i < n_ord && ((sb[t >> 6] >> (t & 63)) & 1ull);
                const unsigned m = __ballot_sync(FULL, in);
                const int rank = taken + __popc(m & ((1u << lane) - 1));
                const bool take = in && rank < n;
                for (int l = 0; l < 32; l++) {  // hand each taken type to the lane that owns its word
                  const int tt = __shfl_sync(FULL, take ? t : -1, l);
                  if (tt >= 0 && (tt >> 6) == lane) acc |= 1ull << (tt & 63);
                }
                taken += __popc(m);
              }
              return acc;
            };
            // 15, or as many as minValues needs if that is more: the shortest prefix of the price order that satisfies every
            // key (consolidation.go:296-312, types.go:301-337).  All `total` types satisfy them (checked above).
            uint64_t first = prefix_bits(15);
            if (d.mv_strict && !min_values_ok(d, c_tmpl0, first, lane)) {
              int bad = 15, good = total;
              while (good - bad > 1) {
                const int mid = (good + bad) >> 1;
                if (min_values_ok(d, c_tmpl0, prefix_bits(mid), lane))
                  good = mid;
                else
                  bad = mid;
              }
              first = prefix_bits(good);
            }
            rep = first;
          }
        }
        if (any && q.filter_same_type && sn >= 2) {
          // filterOutSameInstanceType (multinodeconsolidation.go:189-226): if an option is a type that is being removed,
          // only options cheaper than the cheapest such node are worth a replacement
          double max_price = 1.7976931348623157e308;
          for (int i = 0; i < sn; i++) {
            const int t = q.node_it[snodes[i]];
            if (t < 0) continue;
            const bool in_rep = (__shfl_sync(FULL, rep, t >> 6) >> (t & 63)) & 1ull;
            if (!in_rep) continue;
            double mine = 1.7976931348623157e308;  // cheapest removed node of this type; none priced: 0 (Go map miss)
            for (int j = 0; j < sn; j++)
              if (q.node_it[snodes[j]] == t && q.node_price[snodes[j]] >= 0 && q.node_price[snodes[j]] < mine)
                mine = q.node_price[snodes[j]];
            if (mine > 1e308) mine = 0.0;
            if (mine < max_price) max_price = mine;
          }
          if (max_price < 1e308) {
            uint64_t keep = 0;
            if (lane < ITW)
              for (uint64_t bits = rep; bits;) {
                const int b = __ffsll((long long)bits) - 1;
                bits &= bits - 1;
                const int t = lane * 64 + b;
                double worst = 1.7976931348623157e308;
                for (int ci = 0; ci < 3 && worst > 1e308; ci++) {
                  if (q.ct_key < 0 || !((q.ct_order_valid >> ci) & 1)) continue;
                  for (int e = q.wl_off[t * 3 + ci]; e < q.wl_off[t * 3 + ci + 1]; e++)
                    if ((okmask >> q.wl_set[e]) & 1u) {
                      worst = q.wl_price[e];
                      break;
                    }
                }
                if (worst < max_price) keep |= 1ull << b;
              }
            rep = keep;
            any = __any_sync(FULL, rep != 0);
            // RemoveInstanceTypeOptionsByPriceAndMinValues again (multinodeconsolidation.go:220-224)
            if (any && d.mv_strict && !min_values_ok(d, c_tmpl0, rep, lane)) any = false;
          }
        }
        if (any) decision = KP_DECISION_REPLACE;
        if (any && q.export_order && q.repl_order) {
          // the surviving types in OrderByPrice order (sv[] holds the claim's types by price; ties as Go leaves them)
          if (lane < ITW) sb[lane] = rep;
          __syncwarp();
          int32_t* dst = q.repl_order + (size_t)s * q.order_cap;
          for (int b0 = 0; b0 < n_ord; b0 += 32) {
            const int i = b0 + lane;
            const int t = i < n_ord ? sv[i] : 0;
            const bool in = i < n_ord && ((sb[t >> 6] >> (t & 63)) & 1ull);
            const unsigned m = __ballot_sync(FULL, in);
            const int at = n_ord_out + __popc(m & ((1u << lane) - 1));
            if (in && at < q.order_cap) dst[at] = t;
            n_ord_out += __popc(m);
          }
          if (n_ord_out > q.order_cap) n_ord_out = q.order_cap;
        }
      }
    }
  }
  if (decision != KP_DECISION_REPLACE) rep = 0;
  if (lane < ITW) q.replacement_its[(size_t)s * ITW + lane] = rep;
  if (q.repl_tmpl) {  // Command.Replacements: the NodeClaim itself (consolidation.go:206-229)
    const bool repl = decision == KP_DECISION_REPLACE && have_slots;
    Slot F = slot_absent();
    if (repl && lane < K) {
      F = scratch[lane];
      // OD -> [OD, spot]: the price filter assumed the spot variant launches, so the claim is pinned to spot (:211-214)
      if (!spot_pinned && lane == q.ct_key && q.ct_spot >= 0 && q.ct_od >= 0) {
        const KeyInfo ki = key_info(d, lane);
        if (slot_has(ki, F, q.ct_spot) && slot_has(ki, F, q.ct_od)) F = slot_add(ki, F, Slot{SF_PRESENT, 1ull << q.ct_spot, 0, 0});
      }
    }
    if (lane < K) {
      const size_t i = (size_t)s * K + lane;
      q.repl_sflags[i] = (uint8_t)F.f;
      q.repl_smask[i] = F.m;
      if (q.repl_sgte) {
        q.repl_sgte[i] = F.gte;
        q.repl_slte[i] = F.lte;
      }
    }
    if (lane < d.R) q.repl_req[(size_t)s * d.R + lane] = repl ? c_req0[lane] : 0;
    if (lane == 0) {
      q.repl_tmpl[s] = repl ? c_tmpl0 : -1;
      if (q.repl_order_n) q.repl_order_n[s] = repl ? n_ord_out : 0;
    }
  }
  if (lane == 0) {
    q.decision[s] = (uint8_t)decision;
    q.n_new_claims[s] = n_new;
    q.n_unscheduled[s] = unscheduled;
  }
  __syncwarp();
}

#define CONSOL_WARPS 8
struct ConsolWarp {
  WInst inst;
  PodCtx ctx;
  Slot scratch[KP_MAXK];
};
struct ConsolShared {
  KpDev ds;
  ConsolWarp w[CONSOL_WARPS];
};

// Two CTAs per SM (<= 128 registers, a few spills): the chain of one subset is latency-bound, so resident warps are what
// fills the issue slots.  Pinned because ptxas otherwise flips between 128 and 248 registers on unrelated edits.
#ifndef CONSOL_MIN_CTAS
#define CONSOL_MIN_CTAS 2
#endif
// VOL: some pod of the cluster has several volume-topology alternatives (kp_problem.class_vol_next); the host launches that
// instantiation only then, so the other two compile to what they did before it existed.
template <bool LEAN, bool VOL = false>
__global__ void __launch_bounds__(CONSOL_WARPS * 32, CONSOL_MIN_CTAS) k_consolidate(const __grid_constant__ KpDev d_in,
                                                                    const __grid_constant__ KpConsol q) {
  extern __shared__ __align__(16) unsigned char smem_raw[];
  ConsolShared& sh = *reinterpret_cast<ConsolShared*>(smem_raw);
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  stage_tables(d_in, &sh.ds, smem_raw + KP_ALIGN16(sizeof(ConsolShared)));
  const KpDev& d = sh.ds;
  ConsolWarp& W = sh.w[warp];
  WInst& I = W.inst;
  const int R = d.R, N = d.N;
  const size_t slot = (size_t)blockIdx.x * CONSOL_WARPS + warp;
  const int capq = q.capq;
  const ConsolScratch w = consol_slot(d, q, slot);
  if (lane == 0) {
    I.queue = w.queue;
    I.qcls = w.qcls;
    I.last_len = w.last_len;
    I.pod_target = nullptr;
    I.pod_error = nullptr;
    I.Cmax = capq;
    I.c_tmpl = w.c_tmpl;
    I.c_npods = w.c_npods;
    I.c_req = w.c_req;
    I.c_sflags = w.c_sflags;
    I.c_smask = w.c_smask;
    I.c_sgte = w.c_sgte;
    I.c_slte = w.c_slte;
    I.c_its = w.c_its;
    I.c_j = w.c_j;
    I.order = w.order;
    I.cnt_at = w.cnt_at;
    I.pmask = w.pmask;
    I.amask = w.amask;
    I.tmpl_remaining = w.tmpl_remaining;
    I.CS = 0;
    I.CQ = 0;
    I.CR = 0;
    I.c_dom = nullptr;  // candidate sets with topology take the batch path (k_wsolve_batch)
    I.rsv_cap = w.rsv_cap;
    I.c_rsv = w.c_rsv;
    I.c_ports = w.c_ports;
    I.ov_ports = w.ov_ports;
    I.ov_cap = capq;
    I.ov_node = w.ov_node;
    I.ov_rem = w.ov_rem;
    I.ov_present = w.ov_present;
    I.ov_sflags = w.ov_sflags;
    I.ov_smask = w.ov_smask;
    I.ov_sgte = w.ov_sgte;
    I.ov_slte = w.ov_slte;
  }
  __syncwarp();
  int32_t* clsl = w.clsl;
  int32_t* rk = w.rk;
  uint8_t* kindl = w.kindl;
  if (lane == 0) I.pod_kind = kindl;
  unsigned long long t0 = 0;
  if (q.deadline_ns > 0) {
    if (lane == 0) {
      unsigned long long now;
      asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(now));
      t0 = atomicCAS(q.t_start, 0ull, now);
      if (t0 == 0) t0 = now;
    }
    t0 = __shfl_sync(FULL, t0, 0);
  }

  for (;;) {
    if (q.deadline_ns > 0) {  // context deadline (helpers.go / consolidation timeouts): finished subsets stay valid
      unsigned long long now;
      asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(now));
      now = __shfl_sync(FULL, now, 0);
      if ((long long)(now - t0) > q.deadline_ns) break;
    }
    int s = 0;
    if (lane == 0) s = atomicAdd(q.next, 1);
    s = __shfl_sync(FULL, s, 0);
    if (s >= q.n_subsets) break;
    const int so = q.subset_off[s], sn = q.subset_off[s + 1] - so;
    const int32_t* snodes = q.subset_nodes + so;
    // ---- pods = the candidates' reschedulable pods (helpers.go:60-75), sorted like NewQueue (queue.go:37-43)
    int n = 0;
    for (int i = 0; i < sn; i++) {
      const int node = snodes[i];
      const int a = q.node_pod_off[node], b = q.node_pod_off[node + 1];
      for (int j = a + lane; j < b; j += 32) {
        const int o = n + (j - a);
        if (o < capq) {
          clsl[o] = q.pod_class[j];
          rk[o] = q.pod_rank[j];
        }
      }
      n += b - a;
    }
    const int n_cand_pods = n;
    for (int j = lane; j < q.n_extra; j += 32) {  // pending pods + pods of deleting nodes (helpers.go:65-91)
      const int o = n + j;
      if (o < capq) {
        clsl[o] = q.pod_class[q.extra_row0 + j];
        rk[o] = q.pod_rank[q.extra_row0 + j];
      }
    }
    n += q.n_extra;
    if (kindl)
      for (int i = lane; i < n && i < capq; i += 32) kindl[i] = i < n_cand_pods ? 0 : q.extra_kind[i - n_cand_pods];
    if (n > capq) {
      if (lane == 0) *q.status = KP_ERR_CAPACITY;
      break;
    }
    __syncwarp();
    for (int i = lane; i < n; i += 32) {
      const int my = rk[i];
      int pos = 0;
      for (int j = 0; j < n; j++) pos += rk[j] < my ? 1 : 0;
      I.queue[pos] = i;
      I.qcls[pos] = clsl[i];
    }
    // ---- per-instance state
    if (lane == 0) {
      I.P = n;
      I.n_ov = 0;
      I.n_removed = sn;
      I.removed = snodes;
    }
    for (int i = lane; i < d.n_rsv; i += 32) I.rsv_cap[i] = d.rsv_cap[i];  // NewReservationManager: a fresh one per simulation
    for (int i = lane; i < N * R; i += 32) {  // updateRemainingResources over stateNodes minus candidates
      const int t = i / R, r = i % R;
      int64_t rem = q.tmpl_remaining0[i];
      if ((d.tmpl_limit_present[t] >> r) & 1)
        for (int c = 0; c < sn; c++)
          if (q.node_tmpl[snodes[c]] == t) rem += q.node_capacity[(size_t)snodes[c] * R + r];
      I.tmpl_remaining[i] = rem;
    }
    __syncwarp();
    wsolve_run<true, LEAN, false, VOL>(d, I, W.ctx, W.scratch, lane);
    if (I.status != KP_OK) {
      if (lane == 0) *q.status = I.status;
      break;
    }
    if (!LEAN) claims_finalize(d, I.c_sflags, I.c_smask, I.c_rsv, I.n_claims, lane);
    // ---- computeConsolidation (consolidation.go:136-229)
    consol_decide(d, q, slot, W.scratch, I.c_sflags, I.c_smask, I.c_sgte, I.c_slte, I.c_its, I.n_claims > 0 ? I.c_tmpl[0] : -1,
                  I.c_req, I.n_claims > 0 ? I.c_npods[0] : 0, sn, snodes, I.n_unsched + I.n_uninit, I.n_claims, s, lane);
  }
}

// The general consolidation path (evicted pods carry topology constraints): every candidate set is a full
// Scheduler.Solve of its own (fresh NewTopology) -- all sets of a chunk run as ONE k_wsolve_batch launch, one CTA each --
// and this kernel then applies computeConsolidation to every instance: block b = instance b = result row b.
__global__ void __launch_bounds__(32) k_decide_batch(const KpDev* __restrict__ devs, KpConsol q, const int32_t* __restrict__ soff,
                                                     const int32_t* __restrict__ snodes) {
  __shared__ Slot scratch[KP_MAXK];
  const int lane = threadIdx.x, b = blockIdx.x;
  const KpDev& d = devs[b];
  const int unscheduled = (int)(d.counters[7] + d.counters[8]);
  const int n_new = *d.n_claims;
  consol_decide(d, q, (size_t)b, scratch, d.c_sflags, d.c_smask, d.c_sgte, d.c_slte, d.c_its, n_new > 0 ? d.c_tmpl[0] : -1,
                d.c_req, n_new > 0 ? d.c_npods[0] : 0, soff[b + 1] - soff[b], snodes + soff[b], unscheduled, n_new, b, lane);
}

// ---------------------------------------------------------------------------------------------------------------
// Results.TruncateInstanceTypes (scheduler.go:361-379; provisioner.go:380 calls it right after Solve): every new NodeClaim
// keeps its `max_n` cheapest instance types (Truncate, types.go:339-351: OrderByPrice over the claim's requirements); a
// truncated list that breaks the NodePool's minValues (Strict) drops the claim.  One warp per claim, grid-stride; slot w of
// the scratch arrays belongs to warp w.
__global__ void __launch_bounds__(128) k_truncate_claims(KpDev d, PriceTabs pt, int max_n, double* sort_key, int32_t* sort_val,
                                                         unsigned long long* sort_bits, uint8_t* dropped) {
  __shared__ Slot scratch[4][KP_MAXK];
  const int lane = threadIdx.x & 31, wi = threadIdx.x >> 5, warp = blockIdx.x * 4 + wi, nw = gridDim.x * 4;
  const int K = d.K, ITW = d.ITW, nC = *d.n_claims;
  double* sk = sort_key + (size_t)warp * d.T;
  int32_t* sv = sort_val + (size_t)warp * d.T;
  unsigned long long* sb = sort_bits + (size_t)warp * ITW;
  for (int c = warp; c < nC; c += nw) {
    const uint64_t its = lane < ITW ? d.c_its[(size_t)c * ITW + lane] : 0ull;
    int n_its = lane < ITW ? __popcll(its) : 0;
    for (int o = 16; o; o >>= 1) n_its += __shfl_xor_sync(FULL, n_its, o);
    if (n_its <= max_n) continue;  // (the order itself is not part of the result)
    if (lane < K) scratch[wi][lane] = load_slot(d.c_sflags, d.c_smask, d.c_sgte, d.c_slte, (size_t)c * K + lane, d.has_bounds);
    __syncwarp();
    const unsigned okmask = offering_ok_mask(d, scratch[wi], lane);
    order_by_price(pt, its, n_its, okmask, sk, sv, ITW, lane);
    const uint64_t cur = first_types_bitmap(sv, max_n, sb, ITW, lane);
    if (lane < ITW) d.c_its[(size_t)c * ITW + lane] = cur;
    const bool ok = !d.mv_strict || min_values_ok(d, d.c_tmpl[c], cur, lane);
    if (lane == 0 && !ok) dropped[c] = 1;
    __syncwarp();
  }
}
// ... and the pods of a dropped claim become PodErrors (scheduler.go:368-373)
__global__ void __launch_bounds__(256) k_mark_dropped(const int32_t* pod_target, uint8_t* pod_error, const uint8_t* dropped, int64_t P) {
  const int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
  if (i >= P) return;
  const int t = pod_target[i];
  if (t <= -2 && dropped[-2 - t]) pod_error[i] = KP_PODERR_MINVALUES_TRUNCATED;
}
