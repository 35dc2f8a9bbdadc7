// kp_tables.hpp -- the HBM-resident layout of a scheduling problem (shared between host prep and the kernels).
//
// Requirements (pkg/scheduling/requirements.go:36) become fixed-width rows: one slot per label key, each slot a flag
// byte + one 64-bit value mask (+ optional integer bounds).  Instance-type side data is bit-sliced: for every
// (key, value) a bitmap over instance types, for every resource a table of ">= threshold" bitmaps, for every distinct
// offering requirement set a bitmap of the types that sell it.  filterInstanceTypesByRequirements
// (nodeclaim.go:412-480) then is a handful of coalesced 64-bit ANDs/ORs per instance-type word.
#pragma once
#include <cstdint>
#ifndef __CUDACC__
struct int4 { int x, y, z, w; };
struct ulonglong2 { unsigned long long x, y; };
#endif

#define KP_MAXK 32          // label keys (one warp lane per key)
#define KP_MAXR 8           // resources
#define KP_MAX_ITW 32       // instance-type bitmap words (<= 2048 types, one lane per word)
#define KP_MAX_OFFSETS 32   // distinct offering requirement sets
#define KP_HDR 10            // ints of a class header: tolset, rv, moff, mend, roff, rend, fsig, nsig, hoff, hend

// slot flags
#define SF_COMPLEMENT 0x01u
#define SF_HAS_GTE 0x02u
#define SF_HAS_LTE 0x04u
#define SF_PRESENT 0x10u

// operators of a slot (requirement.go:282-293)
#define OP_IN 0
#define OP_NOT_IN 1
#define OP_EXISTS 2
#define OP_DNE 3

// one scheduling.Requirement on a 64-value universe: {complement, values, gte, lte} (requirement.go:36-43)
struct Slot {
  uint32_t f;   // SF_*
  uint64_t m;   // values
  int64_t gte, lte;
};

// One lane's share of a class row: lane k carries the class's requirement slots on key k, lane r its request for
// resource r, lane i < KP_HDR header word i (lanes KP_HDR+2, +3: the tolerated-template mask, KP_HDR+4: cls_relax, KP_HDR+5: tkinfo).  32 bytes, so staging a
// pod is two 16-byte loads per lane.
struct ClsLane {
  uint64_t pod_m, strict_m;
  int64_t req;
  int32_t hdr;
  uint8_t pod_f, strict_f, pad[2];
};
static_assert(sizeof(ClsLane) == 32, "ClsLane is loaded as two 16-byte vectors");

struct KpGroup {
  int32_t key;          // label key, or -1 for the hostname key
  int32_t type;         // KP_TOPO_*
  int32_t max_skew;
  int32_t min_domains;  // -1 == nil
  int32_t inverse;
  int32_t dom_off;      // offset into dom_cnt (non-hostname groups); hostname groups: row in host_cnt
  int32_t filter_off, filter_n;   // TopologyNodeFilter.Requirements alternatives (reqset ids)
  int32_t taint_policy;
  int32_t affinity_policy;  // 0 ignore 1 honor 2 unset; 3 honor, and some filter alternative carries a host rule (bit 0: honor)
  int32_t tolset;
  int32_t host_row;     // row index among hostname groups, -1 otherwise
};
static_assert(sizeof(KpGroup) == 48, "KpGroup is read by value on the solver's critical path: three 16-byte loads");


// pointers into device memory; filled by the host, passed by value to kernels
struct KpDev {
  int K, R, T, ITW, N, X, G, GH, E, D;  // keys, resources, types, words, templates, classes, groups, hostname groups, nodes, offering sets
  int n_reqsets, n_taintsets, n_tolsets;
  int has_bounds;
  int hostname_key;  // index in the ORIGINAL key numbering (slots use compact ids without hostname)
  // key universe
  const uint8_t* key_wellknown;   // [K]
  const uint64_t* key_univ;       // [K] mask of valid value bits
  const int64_t* val_int;         // [K*64]
  const uint64_t* val_isint;      // [K] bitmask
  // requirement sets as slot rows
  const uint8_t* rs_flags;        // [n_reqsets*K]
  const uint64_t* rs_mask;        // [n_reqsets*K]
  const int64_t* rs_gte;          // [n_reqsets*K] (has_bounds)
  const int64_t* rs_lte;
  // taints
  const uint8_t* tol_ok;          // [(n_tolsets+1) * n_taintsets], row tolset+1 (row 0 == no tolerations)
  // instance types (bit-sliced)
  const int32_t* itv_off;         // [K+1] prefix of value counts: row of (k, v) is itv_off[k] + v
  const uint64_t* itv;            // [itv_off[K]*ITW] types whose In-set on key k contains value v
  const uint64_t* it_nokey;       // [K*ITW] types that do not define key k
  const uint64_t* it_dne;         // [K*ITW] types whose slot on k is the empty concrete set
  const uint64_t* it_nonempty;    // [K*ITW] types with a non-empty In-set on k
  const uint64_t* it_valid;       // [ITW] types without a negative allocatable entry
  const int32_t* ge_off;          // [R+1] rows of resource r are ge_off[r] .. ge_off[r+1]
  const int64_t* ge_vals;         // [ge_off[R]] ascending distinct allocatable values per resource
  const uint64_t* ge_bits;        // [ge_off[R]*ITW] row j = types with alloc[r] >= ge_vals[j]
  const Slot* off_slots;          // [D*K] requirement slots of the distinct offering requirement sets
  const uint32_t* off_keys;       // [D] keys present in each set
  const uint64_t* offset_bits;    // [D*ITW] types with an AVAILABLE offering of that set
  int tab_bytes;                  // shared-memory bytes of the staged read-only tables (k_solve); 0 = not staged
  int n_ge, n_itv;                // rows of ge_vals / itv
  int nodes_res;                  // resource index of "pods" (limits), -1: none
  const int64_t* it_capacity;     // [T*R] (limits)
  // templates
  const int32_t* tmpl_rs;         // [N]
  const int32_t* tmpl_taintset;   // [N]
  const uint64_t* tmpl_its_raw;   // [N*ITW] instanceTypes[np] before the prefilter
  uint64_t* tmpl_its;             // [N*ITW] after the NewScheduler prefilter (scheduler.go:147)
  const int64_t* tmpl_daemon;     // [N*R]
  int64_t* tmpl_remaining;        // [N*R] remainingResources (limits)
  const uint32_t* tmpl_limit_present;  // [N]
  // Host rules (kp_prep.cpp build_host_rules): the folded kubernetes.io/hostname requirement of a requirement set, as an
  // admission test of candidates (host_rule_admits).  [n_reqsets] offset of the set's record, -1: no rule; a record is
  // {admits NodeClaims, ceil(E/32) words of admitted existing nodes}.
  const int32_t* host_rules;
  // classes
  const int64_t* cls_req;         // [X*R]
  const int32_t* cls_rs;          // [X]
  const int32_t* cls_tolset;      // [X]
  const int32_t* cls_relax;       // [X] class after one Preferences.Relax step (preferences.go:38-57), -1: none
  // minValues, Strict policy (cloudprovider/types.go:301-337): template n must keep, for each e in
  // [tmpl_mv_off[n], tmpl_mv_off[n+1]), tmpl_mv_need[e] distinct values of table tmpl_mv_key[e]
  // Topology groups the reference creates mid-solve (Topology.Update of a relaxed pod, topology.go:162-194, when the
  // relaxation changed the group's identity: the node filter holds the pod's tolerations and node-affinity terms,
  // topologynodefilter.go:30-64).  Until a pod is first tried as the relaxed class the group does not exist: it records
  // nothing.  (Only spreads can be lazy -- affinity groups have no node filter -- and a spread reads an unregistered
  // hostname as count 0, topologygroup.go:235-247, so hostnames registered before the birth need no bookkeeping.)
  int n_lazy;                     // number of such groups (0: nothing below is ever read)
  int32_t* g_born;                // [G] 1 once the group exists (all but lazy groups: from the start)
  int32_t* g_birth;               // [G] birth order of lazy groups (-1: never born), for the result's group table
  const int32_t* cls_lazy_off;    // [X+1] lazy groups of a class, in constraint order
  const int32_t* cls_lazy;
  int mv_strict;                  // 0: no template carries minValues (or BestEffort): nothing is checked
  const int32_t* tmpl_mv_off;     // [N+1]
  const int32_t* tmpl_mv_key;
  const int32_t* tmpl_mv_need;
  const int32_t* mv_val_off;      // [M+2]
  const uint64_t* mv_masks;       // [values * ITW] instance types that offer the value
  int n_rv;
  const int32_t* cls_match;       // groups that constrain a class (owned + inverse selecting it); bit 30 = selects(pod)
  const int32_t* cls_rec;         // groups that may count a class on Record (select it / inverse owned)
  const ClsLane* cls_lane;        // [X*32] class rows, lane-major (see ClsLane): header, requests, requirement slots
  const int4* cls_hchk;           // hostname-group checks of a class {host_row, type | self << 8, max_skew, group}
  const int64_t* cp_g;            // [X*K] Gt / Lt bounds of PodData.Requirements (has_bounds only)
  const int64_t* cp_l;
  const int64_t* cs_g;            // [X*K] ... of PodData.StrictRequirements
  const int64_t* cs_l;
  // topology groups
  const KpGroup* groups;          // [G]
  const int32_t* filter_rs;       // filter alternatives
  int32_t* dom_cnt;               // [sum over non-hostname groups of 64]
  uint64_t* dom_reg;              // [G] registered-domain mask (t.domains keys)
  uint64_t* dom_pop;              // [G] domains with count > 0 (complement of t.emptyDomains within dom_reg)
  // Null, or while a k_wsolve_batch CTA keeps them on chip: the state of the groups on tk_key.  tk_slot[g] = index s of
  // group g among them (-1: other key); its registered / populated masks are tk_reg[s] / tk_pop[s], its counter of
  // value v is tk_cnt[s * tk_nv + v].  Every reader and writer goes through tk_state (kp_kernels.cuh).
  int32_t* tk_slot;
  uint64_t *tk_reg, *tk_pop;
  int32_t* tk_cnt;
  int tk_nv;                      // value ids of tk_key lie below this
  // the domain fast path (kp_kernels.cuh domain_mask): the one non-hostname key topology groups of fast-path classes
  // use (-1: none), and per claim the value its slot on that key is pinned to (0xff: not a single In value)
  int tk_key;
  uint8_t* c_dom;                 // [Cmax]
  int32_t* g_anypop;              // [G] hostname groups: some domain is populated (len(t.domains) > len(t.emptyDomains)).
                                  // Only ever set during a solve (Record populates, Register adds empty domains, nothing
                                  // unregisters), so a record sets it with a plain store and reads nothing
  // (tk_key and c_dom sit here so that every field below stays 16-byte aligned as it is: k_wsolve_batch reads this block
  // from shared memory in 16-byte pairs, and its register count moves with that pairing)
  int32_t* host_cnt;              // [H * GHS] HOST-major (existing nodes then claims), GHS = max(GH, 1) ints per host: only
                                  // the rows of hosts that exist are ever touched, so the footprint (and the TLB reach it
                                  // needs) follows the NodeClaims opened, not the capacity provisioned for them.
                                  // Updated with RED, read with ld.cg (never through L1)
  int GHS;
  uint32_t* host_pop;             // [GH * HW] bit (group, host): count > 0 -- what anti-affinity / affinity checks read;
                                  // two cache lines per group and 1 000 NodeClaims, prefetched by the stager warp
  int HW;                         // words per host_pop row = ceil(H / 32)
  int H;                          // E + claim capacity
  // existing nodes (dynamic)
  const int32_t* node_taintset;   // [E]
  const uint8_t* node_flags;      // [E] KP_NODE_*
  int64_t* node_rem;              // [E*R]
  uint32_t* node_rem_present;     // [E]
  uint8_t* node_sflags;           // [E*K]
  uint64_t* node_smask;           // [E*K]
  int64_t* node_sgte;             // [E*K]
  int64_t* node_slte;
  int32_t* node_npods;            // [E]
  // claims (dynamic)
  int Cmax;
  int32_t* c_tmpl;                // [Cmax]
  int32_t* c_npods;
  int64_t* c_req;                 // [Cmax*R]
  uint8_t* c_sflags;              // [Cmax*K]
  uint64_t* c_smask;
  int64_t* c_sgte;
  int64_t* c_slte;
  uint64_t* c_its;                // [Cmax*ITW]
  int32_t* c_j;                   // [Cmax*R] threshold rows of the claim's requests (fits_word)
  int32_t* order;                 // [Cmax] s.newNodeClaims as claim ids
  int32_t* cnt_at;                // [Cmax] len(Pods) by position
  // monotone failure cache: for a topology-free class whose keys can never be "undefined" on a NodeClaim, CanAdd only
  // ever flips from true to false (requirements tighten, requests grow, instance types shrink: nodeclaim.go:207-219)
  int n_fsig;                     // distinct requirement sets of such classes
  ulonglong2* pmask;              // [Cmax] per claim, by position in `order`: x = rejected requirement signatures, y = request
                                  // vectors that can never fit again (bit index = signature / vector id, ids >= 64 are not cached)
  unsigned long long* amask;      // [Cmax] per claim: signatures that add nothing to the claim's requirements
  unsigned long long tmpl_all;    // bit n: template n survived the NewScheduler prefilter input (n < N)
  // existing-node candidate bitmaps (supersets; the exact CanAdd runs on every candidate)
  int n_nsig, EW;                 // distinct (requirements, tolerations) signatures; words per row = ceil(E/32)
  uint32_t* nfit;                 // [n_rv * EW] resources.Fits(request vector, remaining) held when last checked
  uint32_t* nstat;                // [n_nsig * EW] taints tolerated and no defined key has an empty intersection
  uint32_t* nactive;              // [EW] schedulable nodes
  int ESW;                        // summary words per row = ceil(EW/32)
  uint32_t* nfit_sum;             // [n_rv * ESW] bit w of word s: nfit word 32*s+w (and nactive) is non-zero
  uint32_t* nstat_sum;            // [n_nsig * ESW] the same for nstat
  // pods
  int64_t P;
  const int32_t* pod_class;       // [P]
  int32_t* queue;                 // [P+1] circular queue of pod rows, initially byCPUAndMemoryDescending
  int32_t* qcls;                  // [P+1] class of queue[i]
  int32_t* last_len;              // [P]
  int32_t* pod_target;            // [P]
  uint8_t* pod_error;             // [P]
  const uint8_t* pod_kind;        // [P] or null: 0 candidate pod, KP_EXTRA_* (consolidation simulations, helpers.go:65-140)
  // scalars out
  int32_t* n_claims;              // [1]
  int64_t* counters;              // [8] existing evals, inflight evals, template evals, commits, slow sorts, ...
  int32_t* status;                // [1] 0 ok, 4 capacity
  int stable_order;
  // host ports (hostportusage.go:35-108): interned <ip, port, protocol> entries in use per NodeClaim / existing node; a
  // class row carries the pod's own entries and everything that Matches them
  int n_hostports;
  int cohort;  // cohort commits of identical pods allowed (kp_wsolve.cuh), 0 with KP_NO_COHORT
  unsigned long long* c_ports;        // [Cmax]
  unsigned long long* node_ports;     // [E]
  const unsigned long long* tmpl_ports;  // [N]
  // reserved capacity (reservationmanager.go:28-110, nodeclaim.go:240-287): reservation id behind each distinct offering
  // set (-1: not reserved), remaining capacity per id, ids held per NodeClaim (bit set)
  int n_rsv, rsv_strict;
  unsigned rsv_sets;              // bit dd: offering set dd is a reserved one
  const int32_t* set_rsv;         // [D]
  int32_t* rsv_cap;               // [n_rsv]
  unsigned long long* c_rsv;      // [Cmax]
  int rsv_ct_key, rsv_reserved_val, rsv_id_key;  // FinalizeScheduling's pins (nodeclaim.go:291-307)
  unsigned long long rsv_val_of[64];             // value bit (in rsv_id_key) of reservation id i
  long long deadline_ns;          // 0 = none; the solve stops with KP_DEADLINE once this much device time has passed
};
// The block is copied to every solver CTA's shared memory, whose plan (kp_api.cu plan_solve) is sized around it: a new
// field takes a padding word (the int fields fill the holes before pointers) rather than growing it.
static_assert(sizeof(KpDev) == 1600, "KpDev's size is part of the solver's shared-memory plan");
