/* karpsolve.h -- C ABI of libkarpsolve.so: the H100 solver behind Karpenter's
 * provisioning hot path.
 *
 * What this boundary replaces (all paths relative to the reference tree,
 * kubernetes-sigs/karpenter @ 7e9d4269):
 *
 *   kp_solve        <-> (*Scheduler).Solve            pkg/controllers/provisioning/scheduling/scheduler.go:381-436
 *                       incl. NewScheduler prefilter   scheduler.go:116-184 and NewTopology topology.go:68-103
 *   kp_consolidate  <-> consolidation.computeConsolidation   pkg/controllers/disruption/consolidation.go:136-229
 *                       over SimulateScheduling               pkg/controllers/disruption/helpers.go:51-142
 *   kp_problem      <-> the arguments of NewScheduler (nodePools, stateNodes, instanceTypes, daemonSetPods) and
 *                       Solve (pods), with cloudprovider.InstanceType / Offering (pkg/cloudprovider/types.go:122-138,
 *                       372-379) flattened to interned integer tables. Strings never cross: the caller (the cgo shim,
 *                       see INTEGRATION.md) interns label keys/values and keeps the tables.
 *   kp_result       <-> scheduling.Results             scheduler.go:237-241 (NewNodeClaims / ExistingNodes / PodErrors)
 *
 * Conventions: plain pointers + counts, no ownership transfer of inputs (the library copies what it needs during the
 * call and retains no caller pointer after return -- the cgo pointer rule).  Outputs are owned by the library until
 * kp_result_free / kp_consol_result_free.  Every entry point returns a kp_status.  There is NO CPU fallback: if no CUDA
 * device is usable the call fails with KP_ERR_CUDA.
 */
#ifndef KARPSOLVE_H
#define KARPSOLVE_H

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define KP_ABI_VERSION 4

typedef enum kp_status {
  KP_OK = 0,
  KP_DEADLINE = 1,         /* partial results valid; maps to context.DeadlineExceeded (scheduler.go:411-414) */
  KP_ERR_INVALID = 2,      /* malformed problem */
  KP_ERR_CUDA = 3,         /* device / driver failure; message via kp_last_error */
  KP_ERR_CAPACITY = 4,     /* a compiled limit was exceeded (e.g. > KP_MAX_RESOURCES) */
  KP_ERR_UNSUPPORTED = 5   /* feature of the reference not built yet (CSI volume limits, BestEffort minValues in kp_consolidate,
                              kubernetes.io/hostname on a NodePool / instance type / offering, with Gt / Lt / minValues, or
                              together with hostname-key pod affinity) */
} kp_status;

/* ---- requirement encoding --------------------------------------------------------------------------------------
 * One entry == one scheduling.Requirement in its canonical form (pkg/scheduling/requirement.go:36-43):
 * {Key, complement, values, gte, lte, MinValues}.  The operator -> canonical mapping of NewRequirementWithFlexibility
 * (requirement.go:48-102: NotIn/Exists -> complement, Gt N -> gte N+1, Lt N -> lte N-1) is applied by the caller.
 * A requirement set (scheduling.Requirements, requirements.go:36) is a CSR row of entries; entries that repeat a key
 * are folded with Requirements.Add (requirements.go:133-140), i.e. intersected, in row order.
 */
#define KP_REQ_COMPLEMENT 0x01u
#define KP_REQ_HAS_GTE 0x02u
#define KP_REQ_HAS_LTE 0x04u
#define KP_REQ_HAS_MINVALUES 0x08u

#define KP_KEY_WELL_KNOWN 0x01u /* member of v1.WellKnownLabels (pkg/apis/v1/labels.go:69-78) => AllowUndefined */
#define KP_KEY_HOSTNAME 0x02u   /* corev1.LabelHostname: one implicit domain per node / NodeClaim */

#define KP_RES_CPU 0x01u
#define KP_RES_MEMORY 0x02u
#define KP_RES_HUGEPAGES 0x04u /* name has prefix "hugepages-": subtracted from allocatable memory (types.go:206-215) */
#define KP_RES_NODES 0x08u     /* resources.Node, only meaningful in NodePool limits (scheduler.go:607) */

#define KP_MAX_RESOURCES 8

/* taint effects / toleration operators (k8s.io/api core/v1) */
#define KP_EFFECT_NONE 0
#define KP_EFFECT_NO_SCHEDULE 1
#define KP_EFFECT_PREFER_NO_SCHEDULE 2
#define KP_EFFECT_NO_EXECUTE 3
#define KP_TOL_EQUAL 0
#define KP_TOL_EXISTS 1
#define KP_TOL_LT 2
#define KP_TOL_GT 3

/* topology constraint kinds (topologygroup.go:36-40) */
#define KP_TOPO_SPREAD 0
#define KP_TOPO_AFFINITY 1
#define KP_TOPO_ANTI_AFFINITY 2

/* label-selector operators (metav1.LabelSelectorOperator) */
#define KP_SEL_IN 0
#define KP_SEL_NOT_IN 1
#define KP_SEL_EXISTS 2
#define KP_SEL_DOES_NOT_EXIST 3

#define KP_NODE_SCHEDULABLE 0x01u /* member of stateNodes handed to NewScheduler */
#define KP_NODE_INITIALIZED 0x02u /* StateNode.Initialized() (scheduler.go:742-750, helpers.go:121-140) */
#define KP_NODE_MANAGED 0x04u

typedef struct kp_problem {
  /* ---- node-label universe ---- */
  int32_t n_keys;
  const uint8_t* key_flags;     /* [n_keys] KP_KEY_* */
  const int32_t* key_value_off; /* [n_keys+1] value ids are local to their key: 0 .. nvalues-1 */
  const int64_t* value_int;     /* [n_values] strconv.Atoi(value) (requirement.go:326-342) */
  const uint8_t* value_is_int;  /* [n_values] 0 if Atoi fails */

  /* ---- requirement sets ---- */
  int32_t n_reqsets;
  const int32_t* reqset_off; /* [n_reqsets+1] -> entry range */
  int32_t n_reqs;
  const int32_t* req_key;        /* [n_reqs] */
  const uint8_t* req_flags;      /* [n_reqs] KP_REQ_* */
  const int64_t* req_gte;        /* [n_reqs] */
  const int64_t* req_lte;        /* [n_reqs] */
  const int32_t* req_min_values; /* [n_reqs] */
  const int32_t* req_val_off;    /* [n_reqs+1] */
  const int32_t* req_vals;       /* value ids (local to req_key) */

  /* ---- resources (dense vectors of n_resources int64, caller-chosen exact integer unit per resource) ---- */
  int32_t n_resources;
  const uint8_t* res_flags; /* [n_resources] KP_RES_* */

  /* ---- taints / tolerations: strings interned in one table, id 0 == "" ---- */
  int32_t n_tt_strings;
  const int64_t* tt_int; /* [n_tt_strings] numeric value for Gt/Lt tolerations */
  const uint8_t* tt_is_int;
  int32_t n_taints;
  const int32_t* taint_key;
  const int32_t* taint_value;
  const uint8_t* taint_effect;
  int32_t n_taintsets;
  const int32_t* taintset_off; /* [n_taintsets+1] */
  const int32_t* taintset_ids;
  int32_t n_tolerations;
  const int32_t* tol_key; /* 0 == empty key */
  const uint8_t* tol_op;  /* KP_TOL_* */
  const int32_t* tol_value;
  const uint8_t* tol_effect; /* KP_EFFECT_NONE matches all effects */
  int32_t n_tolsets;
  const int32_t* tolset_off;
  const int32_t* tolset_ids;

  /* ---- instance types (cloudprovider.InstanceType, types.go:122-138) ---- */
  int32_t n_its;
  const int32_t* it_reqset;       /* [n_its] InstanceType.Requirements */
  const int64_t* it_capacity;     /* [n_its * n_resources] */
  const uint32_t* it_cap_present; /* [n_its] bit r set iff Capacity has resource r */
  const int64_t* it_overhead;     /* [n_its * n_resources] Overhead.Total() (types.go:366-368) */
  const int32_t* it_off_off;      /* [n_its+1] offerings CSR */
  const int32_t* off_reqset;      /* [n_offerings] Offering.Requirements */
  const double* off_price;        /* [n_offerings] */
  const uint8_t* off_available;   /* [n_offerings] */
  const uint8_t* off_reserved;    /* [n_offerings], may be NULL.  1 == Offering.CapacityType() is "reserved" AND the
                                     ReservedCapacity feature gate is on, i.e. the reference runs the offering through
                                     its ReservationManager (reservationmanager.go:28-110, nodeclaim.go:240-307); such
                                     an offering needs off_reservation_id / off_reservation_capacity below. */

  /* ---- NodeClaimTemplates, one per NodePool, already in OrderByWeight order (utils/nodepool/nodepool.go:161) ---- */
  int32_t n_templates;
  const int32_t* tmpl_reqset;         /* NodePool requirements + template labels + karpenter.sh/nodepool label */
  const int32_t* tmpl_taintset;       /* Spec.Taints */
  const int32_t* tmpl_it_off;         /* [n_templates+1] instanceTypes[np.Name] before the NewScheduler prefilter */
  const int32_t* tmpl_its;            /* global instance type indices, provider order */
  const int64_t* tmpl_daemon;         /* [n_templates * n_resources] daemonOverhead (scheduler.go:782-792) */
  const int64_t* tmpl_limits;         /* [n_templates * n_resources] NodePool.Spec.Limits */
  const uint32_t* tmpl_limit_present; /* [n_templates] bit r set iff a limit is defined for r */

  /* ---- pod label sets / selectors / namespaces (for TopologyGroup.selects, topologygroup.go:431-433) ---- */
  int32_t n_labelsets;
  const int32_t* labelset_off; /* [n_labelsets+1] */
  const int32_t* label_key;    /* pod-label string ids (own id space) */
  const int32_t* label_val;
  int32_t n_selectors;
  const int32_t* selector_off; /* [n_selectors+1] -> expression range; matchLabels are In-expressions */
  const int32_t* selx_key;
  const uint8_t* selx_op; /* KP_SEL_* */
  const int32_t* selx_val_off;
  const int32_t* selx_vals;
  int32_t n_nssets;
  const int32_t* nsset_off;
  const int32_t* nsset_ids;

  /* ---- pod classes: pods that are identical for scheduling purposes share one row ---- */
  int32_t n_classes;
  const int64_t* class_requests;      /* [n_classes * n_resources] RequestsForPods incl. pods:1 (resources.go:30-39) */
  const int32_t* class_reqset;        /* PodData.Requirements (scheduler.go:471-491) */
  const int32_t* class_strict_reqset; /* PodData.StrictRequirements */
  const int32_t* class_tolset;
  const int32_t* class_namespace;
  const int32_t* class_labelset;
  const int32_t* class_filter_off; /* [n_classes+1] TopologyNodeFilter.Requirements alternatives (topologynodefilter.go:38-64) */
  const int32_t* class_filter_reqsets;
  const int32_t* class_tsc_off; /* [n_classes+1] topology constraints owned by the class */
  const uint8_t* tsc_type;      /* KP_TOPO_* */
  const int32_t* tsc_key;
  const int32_t* tsc_selector; /* -1 == nil selector (selects nothing) */
  const int32_t* tsc_nsset;
  const int32_t* tsc_max_skew;
  const int32_t* tsc_min_domains;    /* -1 == nil */
  const uint8_t* tsc_taint_policy;   /* 1 == Honor */
  const uint8_t* tsc_affinity_policy;/* 1 == Honor */
  const uint8_t* tsc_preferred;      /* may be NULL. 1 == a preferred (soft) pod affinity / anti-affinity term or a
                                        ScheduleAnyway spread: enforced like a required one until relaxed away
                                        (topology.go:428-499), but a preferred anti-affinity term registers no inverse
                                        group (topology.go:297-322) */
  /* Preferences.Relax (preferences.go:38-146, scheduler.go:438-469): class of the pod after ONE relaxation step, -1 when
   * nothing is left to relax.  A pod that fails with class X is retried at once as class_relax_next[X], and so on; the
   * queue keeps the original class.  May be NULL (no soft constraints anywhere). */
  const int32_t* class_relax_next;   /* [n_classes] */

  /* ---- pods to schedule ---- */
  int64_t n_pods;
  const int32_t* pod_class;
  const int64_t* pod_creation; /* CreationTimestamp, seconds */
  const uint64_t* pod_uid_hi;  /* UID as a 128-bit number, ordered like the canonical lower-case UUID string */
  const uint64_t* pod_uid_lo;

  /* ---- cluster nodes (state.StateNode) in sortExistingNodes order (scheduler.go:738-751) ---- */
  int32_t n_nodes;
  const uint8_t* node_flags;      /* KP_NODE_* */
  const int32_t* node_reqset;     /* labels as In{value}; hostname excluded (see node_hostname) */
  const int32_t* node_hostname;   /* value id in the hostname key */
  const int32_t* node_taintset;   /* StateNode.Taints() */
  const int64_t* node_available;  /* [n_nodes * n_resources] remainingResources (existingnode.go:40-66) */
  const uint32_t* node_avail_present;
  const int64_t* node_capacity;   /* [n_nodes * n_resources] for NodePool limits (scheduler.go:728-735) */
  const int32_t* node_template;   /* NodePool index or -1 */
  /* pods already bound to cluster nodes, counted by countDomains (topology.go:328-426) */
  int64_t n_running;
  const int32_t* run_class;
  const int32_t* run_node;

  /* ---- minValues (InstanceTypes.SatisfiesMinValues, pkg/cloudprovider/types.go:301-337) ----
   * For every key some requirement carries minValues on: the values instanceType.Requirements.Get(key).Values() of each
   * instance type, as ids that only need to be distinct per key (the 64-value masks cannot serve: value compaction folds
   * unmentioned values, and "how many different instance types / families are left" is exactly about those).
   * All NULL / 0 when no requirement has minValues. */
  int32_t n_minvalue_keys;           /* M */
  const int32_t* minvalue_key;       /* [M] key index */
  const int32_t* minvalue_it_off;    /* [M * n_its + 1] CSR over (m, instance type) */
  const int32_t* minvalue_it_vals;   /* value ids */

  /* ---- options (scheduler.go:87-114) ---- */
  /* MinValuesPolicy (scheduler.go:110-114): 0 = Strict: a NodeClaim whose remaining instance types offer fewer distinct
   * values than minValues is refused (nodeclaim.go:464-475).  1 = BestEffort: minValues never refuses; the relaxed value
   * the reference writes back (nodeclaim.go:186-191) is min(minValues, distinct values of the final claim_its), which the
   * decoder derives from the result. */
  int32_t min_values_best_effort;
  int32_t claim_order_mode; /* 0 = Go sort.Slice (pdqsort_func) tie order, 1 = stable */

  /* ---- reserved capacity (ReservationManager, reservationmanager.go:28-110; offeringsToReserve nodeclaim.go:240-287) ----
   * Offering.ReservationID() interned to 0 .. n_reservations-1 (-1 for offerings that are not reserved) and
   * Offering.ReservationCapacity.  The manager starts every id at the smallest capacity any of its offerings reports
   * (reservationmanager.go:38-47).  A NodeClaim reserves every id it could still launch into and releases what later
   * pods rule out.  reserved_offering_strict = 1 is ReservedOfferingModeStrict (scheduler.go:96-98, what the provisioner
   * and the disruption simulations run with, provisioner.go:347): compatible reserved offerings that cannot be reserved
   * fail the NodeClaim with a ReservedOfferingError, which stops the NodePool fallback (scheduler.go:632-646) and the
   * preference relaxation (scheduler.go:451).  All NULL / 0 when no offering is reserved. */
  const int32_t* off_reservation_id;       /* [n_offerings] */
  const int32_t* off_reservation_capacity; /* [n_offerings] */
  int32_t n_reservations;                  /* <= 64 */
  int32_t reserved_offering_strict;
  /* FinalizeScheduling (nodeclaim.go:291-307) pins a NodeClaim that holds reservations to capacity-type In [reserved] and
   * reservation-id In [held ids]; the returned claim requirements (and the ones consolidation prices, consolidation.go:186)
   * are the finalized ones.  Key of karpenter.sh/capacity-type and value id of "reserved" in it; key of the
   * reservation-id label and, per reservation id, its value id in that key. */
  int32_t reservation_capacity_type_key, reservation_reserved_value, reservation_id_key;
  const int32_t* reservation_value;        /* [n_reservations] */

  /* ---- host ports (pkg/scheduling/hostportusage.go:35-108) ----
   * Every distinct <hostIP, hostPort, protocol> of the Solve (pods, daemonset pods, pods bound to the nodes) interned to a bit
   * (<= 64).  hostport_conflicts[i]: the entries HostPort.Matches entry i (same protocol and port, equal IPs or one of them
   * unspecified -- :50-62; i itself included).  A pod cannot join a node / NodeClaim whose used ports Match one of its own
   * (Conflicts :75-88); joining adds its ports.  All NULL / 0: no pod of the Solve uses host ports. */
  int32_t n_hostports;
  const uint64_t* hostport_conflicts; /* [n_hostports] */
  const uint64_t* class_hostports;    /* [n_classes] GetHostPorts(pod) (:93-118) */
  const uint64_t* node_hostports;     /* [n_nodes] StateNode.HostPortUsage(): ports of the pods bound to the node */
  const uint64_t* tmpl_hostports;     /* [n_templates] daemonHostPortUsage[template] (scheduler.go:794-811) */
  /* ---- Results.TruncateInstanceTypes (scheduler.go:361-379, types.go:339-351; provisioner.go:380 calls it with
   * MaxInstanceTypes = 600 right after Solve): > 0: every new NodeClaim keeps its max_instance_types cheapest types
   * (OrderByPrice over its requirements, types.go:238-257) in claim_its; a truncated list that breaks the NodePool's minValues
   * under the Strict policy marks the claim dropped (kp_result.claim_dropped) and its pods KP_PODERR_MINVALUES_TRUNCATED.
   * 0: claim_its is the full list and the caller truncates. */
  int32_t max_instance_types;
  /* ---- several volume-topology alternatives for one pod (PodData.VolumeRequirements, nodeclaim.go:136-153,
   * existingnode.go:98-113) ----
   * The encoder registers one class per alternative -- the same pod, alternative i added to class_reqset (never to
   * class_strict_reqset: the topology sees the pod's own requirements) -- and chains them: class_vol_next[x] is the class to try
   * on a candidate that rejected x, -1 at the end.  pod_class names the head of a chain.  NULL: no pod has more than one.
   * kp_consolidate serves chains on any pod of the cluster's pod table, extra pods included, as kp_solve does. */
  const int32_t* class_vol_next; /* [n_classes] or NULL */
} kp_problem;

/* pod_target encoding */
#define KP_TARGET_UNSCHEDULED (-1)
#define KP_TARGET_CLAIM(k) (-2 - (k))

/* pod_error codes */
#define KP_PODERR_NONE 0
#define KP_PODERR_NO_TEMPLATES 1       /* scheduler.go:510-512 */
#define KP_PODERR_INCOMPATIBLE 2       /* every template rejected the pod (multierr of scheduler.go:683) */
#define KP_PODERR_RESERVED 3           /* ReservedOfferingError (nodeclaim.go:64-79): compatible reserved capacity exists but
                                          is taken; the pod was neither relaxed nor sent to a lower-weight NodePool */

#define KP_PODERR_MINVALUES_TRUNCATED 4 /* the pod's NodeClaim was dropped by TruncateInstanceTypes (scheduler.go:368-373); pod_target
                                          still names the claim */

#define KP_SLOT_PRESENT 0x10u /* or-ed with KP_REQ_* in claim_req_flags */

typedef struct kp_result {
  int64_t n_pods;
  int32_t* pod_target;    /* [n_pods] >=0 node index | KP_TARGET_CLAIM(k) | KP_TARGET_UNSCHEDULED */
  uint8_t* pod_error;     /* [n_pods] KP_PODERR_* */
  int32_t n_claims;       /* NewNodeClaims, index k = creation order */
  int32_t* claim_template;/* [n_claims] */
  int32_t* claim_npods;
  int32_t* claim_rank;    /* [n_claims] position of claim k in the returned NewNodeClaims slice (scheduler.go:504) */
  int64_t* claim_requests;/* [n_claims * n_resources] Spec.Resources.Requests */
  int32_t it_words;
  uint64_t* claim_its;    /* [n_claims * it_words] InstanceTypeOptions as a bitmap over global instance type ids */
  int32_t n_keys;
  int32_t mask_words;     /* sum over keys of ceil(nvalues/64) */
  uint8_t* claim_req_flags; /* [n_claims * n_keys] */
  int64_t* claim_req_gte;   /* [n_claims * n_keys] */
  int64_t* claim_req_lte;
  uint64_t* claim_req_mask; /* [n_claims * mask_words] */
  /* topology-domain counters after the solve (what a multi-GPU run all-reduces) */
  int32_t n_groups;
  int32_t n_domain_slots;
  int32_t* group_domain_off; /* [n_groups+1] */
  int32_t* domain_counts;    /* [n_domain_slots] non-hostname groups only */
  /* evaluation counters: define the algorithmic bytes of SURVEY.md section 8(d) */
  int64_t n_existing_evals, n_inflight_evals, n_template_evals, n_commits;
  double solve_ms; /* device time of the solve kernels (CUDA events) */
  void* _impl;
  /* NodeClaim.reservedOfferings as a bit set over reservation ids (claim_req_* already carry FinalizeScheduling's pins) */
  uint64_t* claim_reservations; /* [n_claims] */
  uint8_t* claim_dropped;       /* [n_claims] 1: TruncateInstanceTypes dropped the claim (max_instance_types > 0 only) */
} kp_result;

/* ---- consolidation ---- */
#define KP_DECISION_NOOP 0
#define KP_DECISION_DELETE 1
#define KP_DECISION_REPLACE 2
#define KP_DECISION_UNKNOWN 255 /* not evaluated: the deadline passed first (kp_consolidate returned KP_DEADLINE) */

/* kinds of the extra pods every simulation schedules next to the candidates' (helpers.go:65-91) */
#define KP_EXTRA_PENDING 1       /* provisionable pending pod: its errors are ignored (scheduler.go:330-334) */
#define KP_EXTRA_DELETING_NODE 2 /* reschedulable pod of a node marked for deletion: must schedule, but landing on an
                                    uninitialized node is no error (helpers.go:121-140) */

typedef struct kp_consol_input {
  /* cluster pods that would be evicted, grouped by the node they run on */
  const int32_t* node_pod_off; /* [n_nodes+1] into kp_problem pod arrays (pods of node i are rows off[i]..off[i+1]) */
  const int32_t* node_it;      /* [n_nodes] instance type of the node, -1 unknown (consolidation.go:323-326) */
  const uint8_t* node_is_spot; /* [n_nodes] Candidate.capacityType == spot */
  int32_t n_subsets;
  const int32_t* subset_off;   /* [n_subsets+1] */
  const int32_t* subset_nodes; /* node indices; each subset is one computeConsolidation(candidates...) call */
  int32_t spot_to_spot_enabled; /* FeatureGates.SpotToSpotConsolidation (consolidation.go:239) */
  int32_t capacity_type_key;    /* key id of karpenter.sh/capacity-type, -1 if not interned */
  int32_t ct_reserved, ct_spot, ct_on_demand; /* value ids in that key, -1 if not interned (types.go:45-47) */
  /* MultiNodeConsolidation.firstNConsolidationOption (multinodeconsolidation.go:154-163): a Replace of two or more nodes
   * goes through filterOutSameInstanceType (:189-226) -- if the replacement options contain a type that is being
   * removed, only options cheaper than the cheapest such node stay; nothing left == not a valid command, reported as
   * KP_DECISION_NOOP.  0 = plain computeConsolidation (single-node consolidation, or the caller filters itself). */
  int32_t filter_same_instance_type;
  /* SimulateScheduling schedules, together with the candidates' pods, the cluster's pending pods and the reschedulable
   * pods of nodes that are already being deleted (helpers.go:65-91); they take capacity and can open NodeClaims.  They
   * are the LAST n_extra_pods rows of the cluster's pod table (rows node_pod_off[n_nodes] .. n_pods-1), with
   * extra_pod_kind[i] = KP_EXTRA_*.  0 / NULL: none. */
  int32_t n_extra_pods;
  const uint8_t* extra_pod_kind;
  /* 1: also return, per REPLACE subset, the price order of the replacement's instance types (repl_order_*) */
  int32_t export_price_order;
} kp_consol_input;

typedef struct kp_consol_result {
  int32_t n_subsets;
  uint8_t* decision;          /* [n_subsets] KP_DECISION_* */
  int32_t it_words;
  uint64_t* replacement_its;  /* [n_subsets * it_words] instance types left after the price filter */
  int32_t* n_new_claims;      /* [n_subsets] */
  int32_t* n_unscheduled;     /* [n_subsets] */
  double solve_ms;
  void* _impl;
  /* The replacement NodeClaim of every REPLACE subset as Command.Replacements needs it (consolidation.go:206-229,
   * replacementsFromNodeClaims): its NodePool, Spec.Resources.Requests and requirements AFTER the capacity-type pins
   * (OD -> [OD, spot] becomes spot-only, :211-214; spot-to-spot pins spot, :249), in the layout of
   * kp_result.claim_req_* (hostname dropped).  Rows of other subsets are zero. */
  int32_t n_keys, mask_words, n_resources;
  int32_t* repl_template;     /* [n_subsets], -1 unless REPLACE */
  int64_t* repl_requests;     /* [n_subsets * n_resources] */
  uint8_t* repl_req_flags;    /* [n_subsets * n_keys] */
  int64_t* repl_req_gte;
  int64_t* repl_req_lte;
  uint64_t* repl_req_mask;    /* [n_subsets * mask_words] */
  /* export_price_order: instance types of replacement_its in OrderByPrice order (types.go:238-257), CSR over subsets */
  int32_t* repl_order_off;    /* [n_subsets + 1] or NULL */
  int32_t* repl_order;
} kp_consol_result;

typedef struct kp_handle kp_handle;

int kp_version(void);
/* device < 0: cudaGetDevice() current */
int kp_create(int device, kp_handle** out);
void kp_destroy(kp_handle* h);
const char* kp_last_error(kp_handle* h);

/* Solve: host pointers in, host result out (H2D / D2H inside). deadline_ms <= 0: none. */
int kp_solve(kp_handle* h, const kp_problem* p, int64_t deadline_ms, kp_result* out);
void kp_result_free(kp_result* r);

/* Two-step variant used by bench.py to time the device-resident solve separately from the transfers:
 * kp_upload copies + encodes the problem into HBM, kp_solve_resident runs only the kernels. */
int kp_upload(kp_handle* h, const kp_problem* p);
int kp_solve_resident(kp_handle* h, int64_t deadline_ms, kp_result* out);

/* Many Scheduler instances at once -- one CTA (one SM) per instance, a single launch.  What it stands for in the
 * reference: the Scheduler instances that run side by side there -- one NewScheduler + Solve per NodePool shard of a
 * provisioning pass (SURVEY.md section 8(e)), one per SimulateScheduling of a disruption pass (helpers.go:51-142, one
 * call per candidate set: multinodeconsolidation.go:118-171, singlenodeconsolidation.go:56-176), provisioner and
 * disruption controller each inside their own Scheduler (provisioner.go:354-375).  Instances share nothing: outs[b] is
 * exactly what kp_solve(problems[b]) returns (outs[b].solve_ms = device time of the whole batch).  Returns KP_DEADLINE
 * if any instance hit the deadline (every outs[b] is valid, partial for the ones that did). */
int kp_solve_batch(kp_handle* h, const kp_problem* const* problems, int32_t n, int64_t deadline_ms, kp_result* outs);
int kp_upload_batch(kp_handle* h, const kp_problem* const* problems, int32_t n);
int kp_solve_batch_resident(kp_handle* h, int64_t deadline_ms, kp_result* outs);

/* ---- multi-GPU: NodePool-sharded provisioning (SURVEY.md section 8(e)) ---------------------------------------------
 * One process per GPU, one handle per process; rank r owns the pods, templates and NodeClaims of its NodePools and runs
 * ordinary solves (kp_solve_resident / kp_solve_batch_resident).  The one exchange of the job is the global
 * topology-domain counter table -- what the reference keeps in Topology.domainGroups / TopologyGroup.domains
 * (topology.go:53-58, topologygroup.go:56-73) for the next scheduling round -- and it lives in the library:
 *   kp_comm_unique_id          ncclGetUniqueId; the caller hands rank 0's id to every rank (any transport)
 *   kp_comm_init               ncclCommInitRank on the handle's device
 *   kp_comm_counter_slots      int32 slots an uploaded instance contributes (non-hostname groups x values of their key,
 *                              the order of kp_result.domain_counts); instance < 0: the kp_upload instance
 *   kp_comm_set_counter_layout size of the global table and where each instance of this handle starts in it.  From
 *                              then on every resident solve ends, on the library's stream and inside solve_ms, with
 *                              scatter (device) + ONE ncclAllReduce(sum, int32) over NVLink.  Without kp_comm_init
 *                              (single GPU) the table is just the scatter.
 *   kp_comm_global_counts      device -> host copy of the reduced table
 * NCCL is bound at run time (dlopen("libnccl.so.2")): the library has no link-time dependency on it. */
#define KP_COMM_ID_BYTES 128
int kp_comm_unique_id(uint8_t* id128);
int kp_comm_init(kp_handle* h, const uint8_t* id128, int32_t rank, int32_t world);
int64_t kp_comm_counter_slots(kp_handle* h, int32_t instance);
int kp_comm_set_counter_layout(kp_handle* h, int64_t total_slots, const int64_t* slot_offset, int32_t n_instances);
int kp_comm_global_counts(kp_handle* h, int32_t* out, int64_t n);
double kp_comm_last_allreduce_ms(kp_handle* h); /* scatter + all-reduce share of the last solve_ms */
void kp_comm_destroy(kp_handle* h);

int kp_consolidate(kp_handle* h, const kp_problem* cluster, const kp_consol_input* in, int64_t deadline_ms,
                   kp_consol_result* out);
void kp_consol_result_free(kp_consol_result* r);

/* Feasibility matrix only (kernel K1): bit (class, template, it) == instance type `it` survives
 * filterInstanceTypesByRequirements (nodeclaim.go:412-480) for a fresh NodeClaim of `template` holding one pod of
 * `class`, ignoring topology.  out: [n_classes * n_templates * it_words] */
int kp_feasibility(kp_handle* h, const kp_problem* p, uint64_t* out_bits, int32_t* out_it_words);

/* Go's sort.Slice order (pdqsort_func, unstable) of a key array under less = "<": perm_out[i] = index of the element left at
 * position i.  Host code, no device: the disruption front-end sorts candidates by DisruptionCost with it
 * (consolidation.go:126-131, singlenodeconsolidation.go:143-146), so that cost ties fall the way the reference's do. */
int kp_go_sort_f64(const double* keys, int32_t n, int32_t* perm_out);
int kp_go_sort_i64(const int64_t* keys, int32_t n, int32_t* perm_out);

/* Test hook: the DEVICE's requirement algebra (karpenter_b200/csrc/kp_slot.hpp, what the kernels run) on caller-provided
 * requirement pairs over one 64-value key, one thread per case -- so the reference's own known-answer tables
 * (pkg/scheduling/requirement_test.go:103-1084, requirements_test.go:57-543) can be run against it directly.
 * flags: KP_REQ_COMPLEMENT | KP_REQ_HAS_GTE | KP_REQ_HAS_LTE | KP_SLOT_PRESENT (0: the key is undefined on that side). */
typedef struct kp_slot_case {
  uint64_t mask_a, mask_b;
  int64_t gte_a, lte_a, gte_b, lte_b;
  uint32_t flags_a, flags_b;
  int32_t value;           /* for Has(a, value) */
  int32_t well_known;      /* the key is in WellKnownLabels */
  int32_t allow_undefined; /* Compatible(a <- b, AllowUndefinedWellKnownLabels) */
  int32_t _pad;
} kp_slot_case;
typedef struct kp_slot_out {
  uint64_t mask;           /* Intersection(a, b) */
  int64_t gte, lte;
  uint32_t flags;
  int32_t op;              /* Operator() of the intersection: 0 In, 1 NotIn, 2 Exists, 3 DoesNotExist */
  int32_t has_intersection, has_value, compatible;
  int32_t _pad;
} kp_slot_out;
int kp_debug_slot_algebra(kp_handle* h, const int64_t* value_int /* [64] */, uint64_t value_is_int, uint64_t universe,
                          const kp_slot_case* cases, int32_t n, kp_slot_out* out);

typedef struct kp_stats {
  double upload_ms, prep_ms, solve_ms, download_ms;
  int64_t bytes_h2d, bytes_d2h;
  int64_t kernel_launches;
  int64_t cohort_pods; /* pods of the last solve that were committed by cohort steps (runs of identical pods, DESIGN.md section 4) */
} kp_stats;
int kp_get_stats(kp_handle* h, kp_stats* out);

#ifdef __cplusplus
}
#endif
#endif /* KARPSOLVE_H */
