/*
 * kueue_b200.h — C-ABI of libkueue_b200: the H100-native batched evaluator for
 * Kueue's scheduling cycle (nominate -> flavor-assign -> order -> admit/preempt).
 *
 * The reference has NO FFI for this path (it is 100% Go, SURVEY.md §2); these
 * entry points are what a cgo binding placed inside
 *     pkg/scheduler/scheduler.go:218  (*Scheduler).schedule
 * would call between `s.cache.Snapshot(ctx)` (scheduler.go:245) and the replay of
 * side effects (admit :398, IssuePreemptions :347, requeueAndUpdate :410,417).
 * Each struct field cites the reference type it flattens.  See INTEGRATION.md
 * for the Go-side stub.
 *
 * Conventions
 *   - every kb_* function returns int32: 0 = ok, <0 = kb_status error.
 *     kb_last_error(h) returns a static/handle-owned C string.
 *   - all input pointers are HOST pointers (ideally from kb_alloc_pinned);
 *     they are read-only and never retained after the call returns
 *     (cgo pointer rule).  Outputs are written only into caller buffers.
 *   - int64 quantities use the reference's units (cpu in milli, others
 *     absolute: pkg/resources/requests.go:104-109).
 *   - KB_NO_LIMIT encodes a nil BorrowingLimit / LendingLimit
 *     (pkg/cache/scheduler/resource.go:46-50).
 *   - node index space: ClusterQueues are nodes [0, n_cq); Cohorts are nodes
 *     [n_cq, n_cq+n_cohort).  parent[] holds a node index or -1.
 *   - flavor-resource cell index:  fr = flavor * n_resource + resource.
 */
#ifndef KUEUE_B200_H
#define KUEUE_B200_H

#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define KB_NO_LIMIT INT64_MAX
#define KB_MAX_RESOURCES 16   /* n_resource <= 16  */
#define KB_MAX_FLAVORS   64   /* n_flavor   <= 64 (eligibility bitmask is u64) */
#define KB_MAX_DEPTH     16   /* parent hops from a ClusterQueue to its root <= 16: paths of <= 17 nodes */
#define KB_MAX_WL_PODSETS 8   /* podsets per workload <= 8 (Workload spec.podSets MaxItems=8,
                                 apis/kueue/v1beta2/workload_types.go) */
#define KB_N_KERNELS     20

typedef enum kb_status {
  KB_OK = 0,
  KB_ERR_INVALID = -1,      /* malformed snapshot (bounds, cycles, sizes)   */
  KB_ERR_CUDA = -2,         /* CUDA runtime failure: caller runs the Go path */
  KB_ERR_CAPACITY = -3,     /* an output buffer (targets) was too small      */
  KB_ERR_UNSUPPORTED = -4,  /* feature bit set that this build cannot honour  */
  KB_ERR_NO_DEVICE = -5
} kb_status;

/* FlavorAssignmentMode — pkg/scheduler/flavorassigner/flavorassigner.go:337-348 */
enum { KB_MODE_NOFIT = 0, KB_MODE_PREEMPT = 1, KB_MODE_FIT = 2 };

/* PreemptionPolicy — apis/kueue/v1beta2/clusterqueue_types.go:455-520 */
enum { KB_POLICY_NEVER = 0, KB_POLICY_LOWER_PRIORITY = 1,
       KB_POLICY_LOWER_OR_NEWER_EQUAL_PRIORITY = 2, KB_POLICY_ANY = 3 };
/* FlavorFungibilityPolicy — clusterqueue_types.go:394-420 */
enum { KB_FUNG_MAY_STOP_SEARCH = 0, KB_FUNG_TRY_NEXT_FLAVOR = 1 };
/* FlavorFungibilityPreference — clusterqueue_types.go:385-388 (0 = unset) */
enum { KB_PREF_UNSET = 0, KB_PREF_BORROWING_OVER_PREEMPTION = 1,
       KB_PREF_PREEMPTION_OVER_BORROWING = 2 };
/* QueueingStrategy — clusterqueue_types.go:87-96 */
enum { KB_QUEUE_BEST_EFFORT_FIFO = 0, KB_QUEUE_STRICT_FIFO = 1 };

/* Preemption target reasons — apis/kueue/v1beta2/workload_types.go:918-932 */
enum { KB_REASON_IN_CLUSTER_QUEUE = 1, KB_REASON_IN_COHORT_RECLAMATION = 2,
       KB_REASON_IN_COHORT_FAIR_SHARING = 3,
       KB_REASON_IN_COHORT_RECLAIM_WHILE_BORROWING = 4 };

/* Outcome of one entry in one cycle.  It refines the reference's
 * entryStatus (scheduler.go:431-442) with the branch of the admit loop
 * (scheduler.go:269-401) that produced it. */
enum {
  KB_DEC_NOFIT = 0,               /* mode NoFit: :292-301; status ""            */
  KB_DEC_PREEMPT_NO_TARGETS = 1,  /* mode Preempt, no targets: :303-318         */
  KB_DEC_SKIPPED_OVERLAP = 2,     /* setSkipped, overlapping targets: :321-325  */
  KB_DEC_SKIPPED_NO_FIT = 3,      /* setSkipped, no longer fits: :328-334       */
  KB_DEC_PREEMPTING = 4,          /* IssuePreemptions: :344-359                 */
  KB_DEC_ASSUMED = 5              /* admit(): :397-400; status "assumed"        */
};

/* Feature gates / config read on the path (SURVEY.md §5).  Bits of
 * kb_snapshot.flags.  Defaults of the reference = KB_FLAGS_DEFAULT. */
enum {
  KB_F_FAIR_SHARING = 1u << 0,                 /* fairsharing.Enabled(s.fairSharing) scheduler.go:259 */
  KB_F_PARTIAL_ADMISSION = 1u << 1,            /* features.PartialAdmission scheduler.go:604          */
  KB_F_FLAVOR_FUNGIBILITY = 1u << 2,           /* flavorassigner.go:863,883                            */
  KB_F_PRIORITY_SORTING_WITHIN_COHORT = 1u << 3, /* scheduler.go:799                                   */
  KB_F_FS_PRIORITIZE_NON_BORROWING = 1u << 4,  /* fair_sharing_iterator.go:171                         */
  KB_F_FS_PREEMPT_WITHIN_NOMINAL = 1u << 5,    /* preemption.go:350                                    */
  KB_F_FS_STRATEGY_S2A = 1u << 6,              /* LessThanOrEqualToFinalShare configured (strategy.go) */
  KB_F_FS_STRATEGY_S2B = 1u << 7,              /* LessThanInitialShare configured                      */
  KB_F_FS_STRATEGY_S2B_FIRST = 1u << 8,        /* strategies = [S2-b, ...] instead of [S2-a, S2-b]     */
  KB_F_TS_PREEMPTION_BUFFER = 1u << 9,         /* features.SchedulerTimestampPreemptionBuffer (alpha, default off):
                                                  LowerOrNewerEqualPriority needs the candidate > 5 min newer
                                                  (preemption_policy.go:28,44-46)                       */
  KB_F_USAGE_RESIDENT = 1u << 16               /* upload hint, not a scheduler setting: keep this call's cq_usage table on
                                                  the device so that following calls may pass only the rows that changed
                                                  (kb_snapshot.usage_delta_*)                            */
};
#define KB_FLAGS_DEFAULT (KB_F_PARTIAL_ADMISSION | KB_F_FLAVOR_FUNGIBILITY | \
  KB_F_PRIORITY_SORTING_WITHIN_COHORT | KB_F_FS_PRIORITIZE_NON_BORROWING |   \
  KB_F_FS_PREEMPT_WITHIN_NOMINAL | KB_F_FS_STRATEGY_S2A | KB_F_FS_STRATEGY_S2B)

/* ------------------------------------------------------------------------
 * Input: one flattened pkg/cache/scheduler.Snapshot + the heads of
 * pkg/cache/queue.Manager, all SoA.
 * ---------------------------------------------------------------------- */
typedef struct kb_snapshot {
  /* ---- dimensions ---- */
  int32_t n_cq;        /* Q: ClusterQueueSnapshot count (snapshot.go:151-215)       */
  int32_t n_cohort;    /* C: CohortSnapshot count                                    */
  int32_t n_flavor;    /* F: distinct ResourceFlavors                                 */
  int32_t n_resource;  /* R: distinct resource names, index order == name order
                          (DRS tie-break "rName < dominantResource", fair_sharing.go:149) */
  int32_t n_rg;        /* total ResourceGroups over all CQs                           */
  int32_t n_wl;        /* W: pending workload.Info records                            */
  int32_t n_podset;    /* total PodSetResources over all pending workloads            */
  int32_t n_adm;       /* A: admitted workloads (ClusterQueueSnapshot.Workloads)      */
  int32_t n_adm_use;   /* total (fr, qty) usage cells over admitted workloads         */
  int32_t n_heads;     /* entries of this cycle (queues.Heads, scheduler.go:230)      */
  int32_t pods_resource; /* index of corev1.ResourcePods or -1 (flavorassigner.go:585) */
  uint32_t flags;      /* KB_F_* */
  int64_t now_ns;      /* clock.Now() for candidates lacking QuotaReserved
                          (preemption/common/ordering.go:93-100)                      */

  /* ---- node tables [n_cq + n_cohort] (hierarchy + resourceNode) ---- */
  const int32_t *parent;       /* hierarchy.ClusterQueue.cohort / Cohort.parent; -1 = none */
  const double  *fair_weight;  /* FairWeight (clusterqueue_snapshot.go:44, cohort_snapshot) */
  /* [node][F*R] — resourceNode.Quotas (resource_node.go:30-43) */
  const int64_t *nominal;      /* ResourceQuota.Nominal                                  */
  const int64_t *borrow_limit; /* *BorrowingLimit or KB_NO_LIMIT                          */
  const int64_t *lend_limit;   /* *LendingLimit  or KB_NO_LIMIT                           */
  /* [n_cq][F*R] — ClusterQueueSnapshot.ResourceNode.Usage.  Cohort usage and
   * every SubtreeQuota are rebuilt on the device (resource_node.go:183-217).  */
  const int64_t *cq_usage;

  /* ---- ClusterQueue attribute tables [n_cq] ---- */
  const uint8_t *cq_within_cq;        /* Preemption.WithinClusterQueue   KB_POLICY_* */
  const uint8_t *cq_reclaim_within;   /* Preemption.ReclaimWithinCohort  KB_POLICY_* */
  const uint8_t *cq_borrow_within;    /* BorrowWithinCohort.Policy: NEVER | LOWER_PRIORITY */
  const uint8_t *cq_has_bwc_threshold;/* BorrowWithinCohort.MaxPriorityThreshold != nil */
  const int32_t *cq_bwc_threshold;    /* *MaxPriorityThreshold                          */
  const uint8_t *cq_when_can_borrow;  /* FlavorFungibility.WhenCanBorrow  KB_FUNG_*   */
  const uint8_t *cq_when_can_preempt; /* FlavorFungibility.WhenCanPreempt KB_FUNG_*   */
  const uint8_t *cq_preference;       /* FlavorFungibility.Preference     KB_PREF_*   */
  const uint8_t *cq_strategy;         /* QueueingStrategy                 KB_QUEUE_*  */
  const int64_t *cq_generation;       /* AllocatableResourceGeneration (clusterqueue_snapshot.go:51-53) */
  /* ResourceGroups (pkg/cache/scheduler/resource.go:31-38), CSR per CQ */
  const int32_t *cq_rg_start;         /* [n_cq+1] into rg_*                            */
  const uint32_t *rg_res_mask;        /* [n_rg] CoveredResources as bit r             */
  const int32_t *rg_flavor_start;     /* [n_rg+1] into rg_flavors                     */
  const int32_t *rg_flavors;          /* ordered ResourceGroup.Flavors (global flavor idx) */

  /* ---- pending workloads [n_wl] (pkg/workload.Info, workload.go:193-218) ---- */
  const int32_t *wl_cq;        /* Info.ClusterQueue                                     */
  const int32_t *wl_priority;  /* priority.Priority(Obj) (pkg/util/priority/priority.go:32-37) */
  const int64_t *wl_ts;        /* Ordering.GetQueueOrderTimestamp, ns (workload.go:1174-1193) */
  const int64_t *wl_uid;       /* total order consistent with Obj.UID string compare    */
  const int64_t *wl_last_gen;  /* LastAssignment.ClusterQueueGeneration; -1 = LastAssignment nil */
  const int32_t *wl_ps_start;  /* [n_wl+1] CSR into podset tables                       */
  /* ---- podsets [n_podset] (workload.PodSetResources, workload.go:220-236) ---- */
  const int64_t *ps_req;       /* [n_podset][R] Requests (total for Count pods)         */
  const uint32_t *ps_req_mask; /* bit r: resource r is a key of Requests                */
  const int32_t *ps_count;     /* Count                                                  */
  const int32_t *ps_min_count; /* *MinCount or -1 (PodSet.MinCount, partial admission)   */
  const uint64_t *ps_flavor_ok;/* bit f: flavor f passes checkFlavorForPodSets
                                  (taints/affinity, flavorassigner.go:899-944), host-evaluated */
  const int8_t  *ps_last_tried;/* [n_podset][R] LastState.LastTriedFlavorIdx or -1       */

  /* ---- admitted workloads [n_adm] (preemption candidates) ---- */
  const int32_t *adm_cq;
  const int32_t *adm_priority;
  const int64_t *adm_ts;       /* GetQueueOrderTimestamp of the admitted workload, ns    */
  const int64_t *adm_qr_ts;    /* QuotaReserved LastTransitionTime ns, or INT64_MIN = unset
                                  (ordering.go:93-100 -> now)                             */
  const int64_t *adm_uid;
  const uint8_t *adm_evicted;  /* workload.IsEvicted(Obj)                                */
  const int32_t *adm_use_start;/* [n_adm+1] CSR: Info.FlavorResourceUsage (workload.go:363-376) */
  const int32_t *adm_use_fr;   /* flavor*R + resource                                    */
  const int64_t *adm_use_qty;

  /* ---- entries of this cycle ---- */
  const int32_t *heads;        /* [n_heads] indices into the pending tables.
                                  Reference mode: one per CQ (manager.go:770-794);
                                  batched mode: any subset, e.g. all of them.            */

  /* ---- optional per-workload tables: NULL = absent ---- */
  const uint8_t *wl_has_quota_reservation; /* [n_wl] workload.HasQuotaReservation(Obj): entries that already hold a quota
                                  reservation (second pass) come first in the classical order (scheduler.go:781-789) */
  const int64_t *wl_sched_hash; /* [n_wl] 64-bit digest of Info.SchedulingHash, 0 = SchedulingHashUnknown
                                  (workload.go:311-343).  Read by kb_run_drain only: a NoFit head of a BestEffortFIFO
                                  queue moves every queued workload of the same class to the inadmissible set
                                  (handleInadmissibleHash, cluster_queue.go:408-425). */
  const int32_t *ps_group;     /* [n_podset] PodSetGroupName of the podset's TopologyRequest as a small id, -1 = none.
                                  Consecutive podsets of one workload with the same id get their flavors together: the
                                  requests are summed and one search serves the group (flavorassigner.go:613-675;
                                  LeaderWorkerSet leader + workers).  The podsets of a group must be adjacent. */

  /* ---- upload hint ---- */
  int64_t static_generation;   /* 0 = none.  When non-zero and equal to the value of the previous call on
                                  this handle (with unchanged n_cq/n_cohort/n_flavor/n_resource/n_rg), the
                                  STATIC tables — parent, fair_weight, nominal, borrow_limit, lend_limit, all
                                  cq_* policy tables and the resource-group tables — are not read again: the
                                  device copies and the cohort topology derived from them are reused.  The Go
                                  shim bumps it whenever a ClusterQueue / Cohort spec changes (the event that
                                  increments AllocatableResourceGeneration, clusterqueue_snapshot.go:51-53). */

  /* ---- incremental usage (optional; SURVEY.md f2).  The scheduler cache knows which ClusterQueues' usage changed
     since the previous cycle (admissions it issued: cache.go:619-711 AddOrUpdateWorkload / DeleteWorkload; finished
     workloads).  When usage_delta_cq != NULL the library takes the usage table it kept from the previous call on this
     handle (that call, or an earlier one in an unbroken sequence of delta calls, carried KB_F_USAGE_RESIDENT and the
     full cq_usage), replaces the listed rows and evaluates the cycle on the result; cq_usage is not read and may be
     NULL.  Requires the static tables of that call (same non-zero static_generation and dimensions); otherwise
     KB_ERR_INVALID.  Not available for kb_run_drain. ---- */
  int32_t n_usage_delta;            /* rows in the two tables below                                   */
  const int32_t *usage_delta_cq;    /* [n_usage_delta] ClusterQueue index, each at most once; NULL = cq_usage is the full table */
  const int64_t *usage_delta_rows;  /* [n_usage_delta][F*R] the rows' new values (same layout as a cq_usage row) */

  /* ---- AdmissionFairSharing (optional; read by kb_run_drain).  wl_lq == NULL: AFS is off and every other table of
     this block is ignored.  With afs.Enabled(cfg) (the AdmissionFairSharing gate on and the Configuration's
     admissionFairSharing set), a ClusterQueue whose spec.admissionScope.admissionMode is UsageBasedAdmissionFairSharing
     orders its queue by LocalQueue usage first (queueOrderingFunc, pkg/cache/queue/cluster_queue.go:636-685):
       usage(lq) = sum_r afs_res_weight[r] * AsApproximateFloat64(consumed_r (+) penalty_r), then / lq_weight[lq]
     (Info.CalcLocalQueueFSUsage, pkg/workload/workload.go:391-427), where (+) is Quantity.Add (int64Amount.Add,
     apimachinery amount.go:162-199: a zero operand keeps the other's scale, otherwise the sum takes the smaller scale)
     and AsApproximateFloat64 is value * Pow10(scale) (quantity.go:468-483; Pow10(-k) = 1 / 10^k).  Canonical choices:
     Go sums over a map in random order, the library sums in resource-index order; after penalties the reference's Pop
     (rebuildAll + heap.Fix per item in map order, cluster_queue.go:494-531) may return a workload that is not the
     minimum, the library takes the true minimum of (usage, -priority, timestamp, UID) over the LocalQueue heads.  A
     sticky workload is refused here (kb_snapshot.cq_sticky).  Every admitted workload of such a ClusterQueue adds its entry penalty to its
     LocalQueue (scheduler.go:727-742,946-960; pkg/util/admissionfairsharing/admission_fair_sharing.go):
       penalty_r += int64(float64(MilliValue(SumTotalRequests_r)) * afs_alpha)   (milli-units, truncated toward zero)
     over the workload's full TotalRequests (ps_req where ps_req_mask has bit r, before partial admission).
     Errors: KB_ERR_INVALID for an index out of range, lq_cq[wl_lq[w]] != wl_cq[w] or LocalQueues not numbered
     ClusterQueue-major; KB_ERR_UNSUPPORTED for a scale outside [-22, 22] or a sum that overflows int64 (the reference
     would leave the int64Amount form for inf.Dec).
     Preemption guard: with AFS, CandidatesOrdering (preemption/common/ordering.go:41-100) compares LocalQueue usage only
     between candidates of one ClusterQueue, which is not a transitive order across ClusterQueues, so the order
     slices.SortFunc produces depends on the sort algorithm.  kb_run_cycle, kb_upload and kb_run_drain therefore return
     KB_ERR_UNSUPPORTED when wl_lq != NULL, some cq_afs is set and some ClusterQueue has a preemption policy (a target
     search is possible); the caller then runs the Go cycle.  Without a possible target search kb_run_cycle accepts the
     tables and ignores them: the heads of a single cycle come from the caller's queue. ---- */
  int32_t n_lq;                     /* LocalQueues                                                                  */
  const int32_t *wl_lq;             /* [n_wl] LocalQueue of each pending workload (Spec.QueueName); NULL = AFS off  */
  const int32_t *lq_cq;             /* [n_lq] ClusterQueue of each LocalQueue; non-decreasing (ClusterQueue-major)  */
  const uint8_t *cq_afs;            /* [n_cq] afs.ResourceWeights(cq.Spec.AdmissionScope, cfg) enabled (admission_fair_sharing.go) */
  const double  *lq_weight;         /* [n_lq] Spec.FairSharing.Weight.AsApproximateFloat64(), 1.0 when nil          */
  const int64_t *lq_consumed;       /* [n_lq][R] AfsConsumedResources entry as int64Amount values (0 = absent)      */
  const int32_t *lq_consumed_scale; /* [n_lq][R] their scales (resource.Scale: value * 10^scale)                    */
  const int64_t *lq_penalty;        /* [n_lq][R] AfsEntryPenalties.Peek at the start, milli-units; NULL = none      */
  const double  *afs_res_weight;    /* [R] AdmissionFairSharing.ResourceWeights, 1 for a resource not listed        */
  const int64_t *afs_milli_mul;     /* [R] MilliValue factor of the library's unit: 1 for cpu (milli), else 1000   */
  double afs_alpha;                 /* 1 - 0.5^(UsageSamplingInterval / UsageHalfLifeTime), 0 when the half-life is 0
                                       (calculateAlphaRate); computed by the caller so the Go shim passes math.Pow's bits */

  /* ---- eviction replay (optional; read by kb_run_drain only, kb_run_cycle ignores it) ----
     adm_wl[a] = index into the pending tables of admitted workload a's own record: its spec as it would be requeued
     (full counts and per-podset requests; its adm_use_* cells may reflect a partial admission).  Those records hold
     quota, so they start out of every queue.  NULL = evictions are not replayed and the drain is unchanged.
     With adm_wl, every target of a Preempting entry of cycle c leaves the admitted tables before cycle c+1 (its cells
     leave its ClusterQueue's usage, its row is removed) and its record returns to its queue with LastAssignment nil;
     then every workload set aside by the ClusterQueues of the victims' root cohort trees returns to its queue
     (QueueAssociatedInadmissibleWorkloadsAfter, manager.go:670-697; inadmissible_workloads.go:128-223).  See
     kb_run_drain.  Errors: KB_ERR_INVALID for an index out of range, an index named twice or
     wl_cq[adm_wl[a]] != adm_cq[a]; KB_ERR_UNSUPPORTED without KB_F_PRIORITY_SORTING_WITHIN_COHORT (a preempted
     workload's queue-order timestamp would become its eviction time, workload.go:1174-1193). */
  const int32_t *adm_wl;            /* [n_adm] */

  /* ---- arrivals and completions: event mode (optional; read by kb_run_drain only, kb_run_cycle ignores them) ----
     The reference's scheduler performance runner (test/performance/scheduler) creates workloads at fixed intervals
     (runner/generator/generator.go) and finishes each one runtimeMs after its admission (runner/controller/
     controller.go:100-160; an eviction restarts that clock, setAdmittedTime :62-72).  A finish is
     workload_controller.go:936-952: the workload leaves the cache and QueueAssociatedInadmissibleWorkloadsAfter
     requeues its root cohort tree (the same step as an eviction).  A creation is AddOrUpdateWorkload -> PushOrUpdate
     (manager.go:524-560), which requeues nothing else.  "Event mode" = at least one of the three tables, or wl_evict_ns, is non-NULL;
     without them kb_run_drain is unchanged.  INT64_MAX as a time means never.  Errors (KB_ERR_INVALID):
     adm_finish_ns[a] <= now_ns, adm_wl naming a record with wl_create_ns > now_ns. */
  int64_t drain_cycle_ns;           /* simulated time one cycle takes; <= 0 means 1 (cycle c at now_ns + c)         */
  const int64_t *wl_create_ns;      /* [n_wl] creation time; <= now_ns: present at the start; NULL = all present    */
  const int64_t *wl_run_ns;         /* [n_wl] run time once admitted; < 0: never finishes; NULL = none finishes     */
  const int64_t *adm_finish_ns;     /* [n_adm] finish time of each row admitted before the drain; NULL = never      */

  /* ---- decay of AdmissionFairSharing consumed usage (optional; event mode of kb_run_drain with wl_lq only) ----
     lq_last_update_ns == NULL: off, and every launch, index and result of the drain stays as without this block.  With
     it, the consumed usage of every LocalQueue of an AFS ClusterQueue decays over simulated time as the LocalQueue
     reconciler decays it (localqueue_controller.go:210-229,363-398; CalculateDecayedConsumed,
     admission_fair_sharing.go:39-66):
       Decay(consumed, adm, elapsed) = MulByFloat(consumed, 1 - a) (+) MulByFloat(adm, a),  a = 1 - 0.5^(elapsed / half-life)
     where MulByFloat(q, f) = int64(float64(MilliValue(q)) * f) milli-units (resource.go:72-99), every resource is
     written back as (milli, -3), MilliValue rounds a finer scale away from zero (negativeScaleInt64) and fails with
     KB_ERR_UNSUPPORTED when a coarser one overflows, and adm[r] is the LocalQueue's admitted usage: the cells with
     fr % R == r of its live admitted rows (library units; its MilliValue is adm[r] * afs_milli_mul[r]).  Durations
     go through Duration.Seconds() before the division.
       1. samples: the next one of a LocalQueue is due at LastUpdate + afs_sampling_ns.  At the start every sample due
          at or before now_ns is taken; at every boundary t -> t' (cycle or jump) every sample due in (t, t'], in time
          order, before the boundary's completions, with a = afs_alpha (one interval elapsed).  With afs_half_life_ns = 0
          a sample resets consumed to empty.  A sample sets LastUpdate to its due time;
       2. an admission at t_c of a workload of LocalQueue l (workload_controller.go:965-971,1030-1056): its cells join
          adm[l], consumed = Decay(consumed, adm, t_c - LastUpdate) (+) entry penalty, LastUpdate = t_c.  The penalty
          goes into consumed, not into the pending penalties (lq_penalty stays as the snapshot gave it);
       3. a completion takes its row's cells out of adm[adm_lq[row]]; consumed changes at the next sample;
       4. the LocalQueue usage of the queue order is recomputed whenever consumed changes.
     Canonical choices: samples do not wake the clock (a quiet cycle still waits for the next arrival or completion,
     and the drain still ends without one); the early resample while penalties are pending (HasPendingFor,
     localqueue_controller.go:219) is not modelled; 0.5^x is the library's afs_half_pow (kb_drain.cuh; Go's math.Pow
     bits depend on the platform), restated in kueue_b200/drain.py.  A LocalQueue without a cache entry is initialised
     by the caller as initializeAfsIfNeeded does (localqueue_controller.go:327-353): consumed = its admitted usage,
     LastUpdate = now_ns.  A drain that runs no cycle (max_cycles = 0, no pending workload) takes no sample.
     Errors (KB_ERR_INVALID): the tables without wl_lq or outside event mode, afs_half_life_ns < 0,
     afs_sampling_ns <= 0, afs_alpha outside [0, 1) or non-zero with half-life 0, lq_last_update_ns[l] > now_ns,
     adm_lq NULL while n_adm > 0, adm_lq[a] outside [-1, n_lq) or lq_cq[adm_lq[a]] != adm_cq[a]. */
  int64_t afs_half_life_ns;         /* UsageHalfLifeTime (>= 0, pkg/config/validation.go:360-366)                   */
  int64_t afs_sampling_ns;          /* UsageSamplingInterval (> 0)                                                 */
  const int64_t *lq_last_update_ns; /* [n_lq] AfsConsumedResources LastUpdate, each <= now_ns; NULL = no decay      */
  const int32_t *adm_lq;            /* [n_adm] LocalQueue of each admitted row, -1 for none                         */

  /* ---- eviction latency (optional; read by kb_run_drain only, kb_run_cycle ignores them) ----
     In the reference an eviction releases nothing at once: IssuePreemptions only sets the Evicted condition
     (pkg/scheduler/preemption/preemption.go:175-215); the quota is released when the job is stopped and its pods are
     gone (pkg/controller/jobframework/reconciler.go:576-590, UnsetQuotaReservationWithCondition), then the cache drops
     the workload and its root cohort tree is requeued (workload_controller.go:973-1004).  wl_evict_ns == NULL: every
     eviction completes before the next cycle, as without this block.  A non-NULL wl_evict_ns turns on event mode and
     delays every release by the evicted workload's latency (see kb_run_drain).  adm_evict_end_ns gives the end time of
     the evictions under way before the drain (rows with adm_evicted set; read only there, INT64_MAX = never); NULL =
     such rows are issued like any other row when a preemptor targets them.  Errors (KB_ERR_INVALID): either table
     without adm_wl, adm_evict_end_ns without wl_evict_ns, wl_evict_ns[w] < 0, adm_evict_end_ns[a] <= now_ns on a row
     with adm_evicted set. */
  const int64_t *wl_evict_ns;       /* [n_wl] time from the workload's eviction until its quota is released (>= 0)  */
  const int64_t *adm_evict_end_ns;  /* [n_adm] end of the eviction under way of a row with adm_evicted; NULL = none */

  /* ---- sticky workload (optional; read by kb_run_drain only, kb_run_cycle ignores it: the caller picks the heads of a
     single cycle) ----
     In the reference a BestEffortFIFO ClusterQueue keeps a preemptor that waits for its evictions at its head
     (stickyWorkload, pkg/cache/queue/cluster_queue.go:64-93; kueue#6929, kueue#7101): RequeueIfNotPresent (:609-619)
     sets it to a workload requeued with RequeueReasonPendingPreemption, queueOrderingFunc (:656-665) orders it before
     every other workload (after the AFS LocalQueue usage, before priority), and only delete (:330-340) clears it.
     cq_sticky[q] is the pending index of ClusterQueue q's sticky workload at the start, -1 = none (the shim reads it
     from the queue manager, INTEGRATION.md).  NULL = the rule is off and the drain is as without this block; non-NULL
     turns it on in plain and event drains, and kb_drain_out.cq_sticky receives the slots after the drain.  See
     kb_run_drain.  Errors: KB_ERR_INVALID for an index outside [-1, n_wl), wl_cq[cq_sticky[q]] != q, an index named by
     adm_wl (a record that holds quota was deleted from its queue) or a record with wl_create_ns > now_ns;
     KB_ERR_UNSUPPORTED for a sticky workload on a ClusterQueue with cq_afs set (in the reference that state needs a
     preemption policy, which the AFS preemption guard refuses). */
  const int32_t *cq_sticky;         /* [n_cq] */

  /* ---- admission checks (optional; read by kb_run_drain only, kb_run_cycle ignores them) ----
     In the reference a workload whose ClusterQueue has admission checks (ProvisioningRequest: the autoscaler has to
     find nodes) reserves quota first and becomes Admitted once every check is Ready (SyncAdmittedCondition,
     admissionchecks.go:36-70); the run clock starts at Admitted (the performance runner, controller.go:62-72,131).  A
     failing attempt n goes to Retry while n <= BackoffLimitCount and to Rejected otherwise (provisioning controller.go:
     536-580).  Retry evicts (reason AdmissionCheck), releases the quota and requeues the workload once RequeueAt = verdict
     + WaitTime(n) has passed (workload_controller.go:330-375,650-678); while it waits its queue-order timestamp is the
     eviction time (GetQueueOrderTimestamp, workload.go:1180-1182).  Rejected deactivates the workload.  wl_check_ns ==
     NULL: off, and every launch, copy and result of the drain stays as without this block.  A non-NULL wl_check_ns turns
     on event mode.  With the tables wl_ts is the creation timestamp.  See kb_run_drain.  Errors: KB_ERR_INVALID for any
     table of this block without adm_wl or without wl_check_ns (wl_requeue_at_ns is also accepted with
     wl_pods_ready_ns), wl_check_ns[w] < 0, wl_check_fail[w] < 0,
     wl_check_retries[w] < 0, adm_check_end_ns[a] <= now_ns on a row (INT64_MIN excepted), wl_requeue_at_ns on a record
     named by adm_wl or created after now_ns, a row with a check under way that also has an eviction under way (adm_evicted
     with adm_evict_end_ns), check_backoff_base_s <= 0, check_backoff_max_s < 0, check_backoff_limit < 0;
     KB_ERR_UNSUPPORTED when the longest WaitTime of attempts 1..limit (see kb_run_drain) is 10,000 s or more (the
     reference's jitter makes it random there) and for the tables together with lq_last_update_ns (a workload with
     checks never makes the Pending -> Admitted transition that updates consumed usage, workload_controller.go:965-972). */
  const int64_t *wl_check_ns;       /* [n_wl] time from a quota reservation to that attempt's verdict; 0 = Ready at once */
  const int32_t *wl_check_fail;     /* [n_wl] how many next attempts fail before one is Ready; INT32_MAX = all; NULL = 0  */
  const int32_t *wl_check_retries;  /* [n_wl] Status.AdmissionChecks[*].RetryCount at the start; NULL = 0              */
  const int64_t *wl_check_evict_ns; /* [n_wl] Evicted LastTransitionTime of a record last evicted by an admission check;
                                       INT64_MIN = not; read for records adm_wl does not name; NULL = none             */
  const int64_t *wl_requeue_at_ns;  /* [n_wl] Status.RequeueState.RequeueAt of a record in check backoff; INT64_MIN = none */
  const int64_t *adm_check_end_ns;  /* [n_adm] verdict time of the attempt under way; INT64_MIN = the row is Admitted   */
  int32_t check_backoff_base_s;     /* RetryStrategy.BackoffBaseSeconds (> 0)                                            */
  int32_t check_backoff_max_s;      /* RetryStrategy.BackoffMaxSeconds (0 = no cap)                                      */
  int32_t check_backoff_limit;      /* RetryStrategy.BackoffLimitCount (>= 0)                                            */

  /* ---- WaitForPodsReady (optional; read by kb_run_drain only, kb_run_cycle ignores them) ----
     In the reference a workload whose pods are not all Ready within waitForPodsReady.timeout of its Admitted condition
     is evicted (reason PodsReadyTimeout), so it stops holding quota it cannot use; it is requeued after an exponential
     backoff (requeuingStrategy) and deactivated once backoffLimitCount is exceeded (workload_controller.go:805-855,
     workload.go:707-722; defaults apis/config/v1beta2/defaults.go:95-100, validation pkg/config/validation.go:196-230).
     wl_pods_ready_ns == NULL: off, and every launch, copy and result of the drain stays as without this block.  A
     non-NULL wl_pods_ready_ns turns on event mode and needs adm_wl.  The block composes with admission checks (the
     attempt starts at the Ready verdict), eviction latency, the sticky table and AFS with or without decay.  See
     kb_run_drain.  blockAdmission: true is not modelled (a caller keeps its own path for it).  Errors: KB_ERR_INVALID
     for any table of this block without adm_wl or without wl_pods_ready_ns, a negative delay, fail or count,
     pods_ready_timeout_ns <= 0, a backoff base or max < 0, a limit < -1, pods_ready_requeue_creation outside {0, 1},
     adm_admitted_ns[a] > now_ns (INT64_MIN excepted) or set on a row whose checks run (adm_check_end_ns) or whose
     eviction is under way (adm_evicted with adm_evict_end_ns), wl_pods_ready_evict_ns on a record named by adm_wl or
     on one that also has wl_check_evict_ns (a workload has one Evicted condition). */
  const int64_t *wl_pods_ready_ns;       /* [n_wl] Admitted -> PodsReady delay of an attempt that becomes ready          */
  const int32_t *wl_pods_ready_fail;     /* [n_wl] next attempts that never become ready; INT32_MAX = all; NULL = 0     */
  const int32_t *wl_pods_ready_count;    /* [n_wl] Status.RequeueState.Count at the start; NULL = 0                      */
  const int64_t *wl_pods_ready_evict_ns; /* [n_wl] Evicted LastTransitionTime of a record last evicted by a timeout, read
                                            under the Eviction timestamp only; INT64_MIN = not; NULL = none              */
  const int64_t *adm_admitted_ns;        /* [n_adm] Admitted time of a row whose pods are not ready yet; INT64_MIN = ready */
  int64_t pods_ready_timeout_ns;         /* waitForPodsReady.timeout (> 0)                                                */
  int32_t pods_ready_backoff_base_s;     /* requeuingStrategy.backoffBaseSeconds (>= 0)                                  */
  int32_t pods_ready_backoff_max_s;      /* requeuingStrategy.backoffMaxSeconds (>= 0; 0 = no cap)                       */
  int32_t pods_ready_backoff_limit;      /* requeuingStrategy.backoffLimitCount; -1 = nil (requeue forever)              */
  int32_t pods_ready_requeue_creation;   /* requeuingStrategy.timestamp: 0 = Eviction (default), 1 = Creation            */

  /* ---- MaximumExecutionTimeSeconds (optional; read by kb_run_drain only, kb_run_cycle ignores them) ----
     In the reference a workload that has spent spec.maximumExecutionTimeSeconds in the Admitted state, summed over its
     admissions in status.accumulatedPastExecutionTimeSeconds, is deactivated with reason MaximumExecutionTimeExceeded
     and never requeued (workload_types.go:71-77,658-662; reconcileMaxExecutionTime workload_controller.go:619-646;
     SyncAdmittedCondition admissionchecks.go:36-86).  wl_max_exec_s == NULL: off, and every launch, copy and result of
     the drain stays as without this block.  A non-NULL wl_max_exec_s turns on event mode and needs adm_wl.  The block
     composes with admission checks (the clock starts at the Ready verdict), WaitForPodsReady, eviction latency, the
     sticky table and AFS.  See kb_run_drain.  Errors: KB_ERR_INVALID for any table of this block without
     wl_max_exec_s or without adm_wl, wl_max_exec_s[w] < 0, wl_exec_acc_s[w] < -1, adm_exec_since_ns NULL while
     n_adm > 0, adm_exec_since_ns[a] > now_ns, INT64_MIN on a row whose checks do not run or another value on one whose
     checks run (adm_check_end_ns), a value other than adm_admitted_ns[a] where that is set; KB_ERR_UNSUPPORTED when an
     attempt's seconds or the accumulated sum leaves int32 (the reference's int32 conversion is then undefined). */
  const int32_t *wl_max_exec_s;     /* [n_wl] spec.maximumExecutionTimeSeconds; 0 = nil (no limit)                      */
  const int32_t *wl_exec_acc_s;     /* [n_wl] status.accumulatedPastExecutionTimeSeconds at the start; -1 = nil; NULL =
                                       every value nil                                                                  */
  const int64_t *adm_exec_since_ns; /* [n_adm] Admitted LastTransitionTime of each row; INT64_MIN = its checks run     */

  /* ---- ClusterQueue and Cohort quota changes (optional; read by kb_run_drain only, kb_run_cycle ignores them) ----
     Planned edits of the quota rows of one node (a ClusterQueue or a Cohort), applied on the drain's clock.  In the
     reference a spec update goes through the cache (updateClusterQueue clusterqueue.go:130-145 /
     updateQuotasAndResourceGroups :199-209, updateCohort cohort.go:44-52 -> updateCohortTreeResources
     resource_node.go:168-198, which bumps AllocatableResourceGeneration of every ClusterQueue of the root tree,
     :160-165) and through the queue manager (UpdateClusterQueue with specUpdated, clusterqueue_controller.go:384,
     AddOrUpdateCohort manager.go:251-262 -> notifyRetryInadmissibleWithoutLock inadmissible_workloads.go:206-223).
     n_quota_change == 0 or qc_ns == NULL: off, and every launch, copy and result of the drain stays as without this
     block.  Otherwise the block turns on event mode (adm_wl is not needed).  Resource groups, flavor order, cohort
     membership and every policy table stay static.  See kb_run_drain.  Errors (KB_ERR_INVALID): a NULL table with
     n_quota_change > 0, n_quota_change < 0, qc_ns decreasing or <= now_ns (an edit already made belongs in the
     snapshot's own rows), qc_node outside [0, n_cq + n_cohort), a negative nominal, KB_NO_LIMIT in a nominal row, a
     negative limit other than KB_NO_LIMIT, and for a ClusterQueue a change to a cell its resource groups do not cover. */
  int32_t n_quota_change;           /* edits below                                                                    */
  const int64_t *qc_ns;             /* [n_quota_change] time of the edit, non-decreasing, each > now_ns               */
  const int32_t *qc_node;           /* [n_quota_change] node in [0, n_cq + n_cohort)                                  */
  const int64_t *qc_nominal;        /* [n_quota_change][F*R] the node's new nominal row                               */
  const int64_t *qc_borrow_limit;   /* [n_quota_change][F*R] its new borrowing-limit row (KB_NO_LIMIT = nil)          */
  const int64_t *qc_lend_limit;     /* [n_quota_change][F*R] its new lending-limit row (KB_NO_LIMIT = nil)            */

  /* ---- workload deactivation and reactivation (optional; read by kb_run_drain only, kb_run_cycle ignores them) ----
     Planned edits of spec.active (kueuectl stop workload / resume workload), applied on the drain's clock.
     n_active_change == 0 or ac_ns == NULL: no edits.  Edits turn event mode on; the edits and wl_inactive need adm_wl.
     See kb_run_drain.  Errors (KB_ERR_INVALID): a NULL table with n_active_change > 0, n_active_change < 0, ac_ns
     decreasing or <= now_ns, ac_wl outside [0, n_wl), ac_active other than 0 or 1, an edit at or before its record's
     wl_create_ns, wl_inactive above 4, and an inactive start record that adm_wl names or that is created after now_ns. */
  int32_t n_active_change;          /* edits below                                                                    */
  const int64_t *ac_ns;             /* [n_active_change] time of the edit, non-decreasing, each > now_ns              */
  const int32_t *ac_wl;             /* [n_active_change] pending record                                               */
  const uint8_t *ac_active;         /* [n_active_change] 0 = set spec.active false (stop), 1 = set it true (resume)   */
  const uint8_t *wl_inactive;       /* [n_wl] start state: 0 = active, 1-4 = inactive with the reason of the
                                       deactivation in force (kb_drain_out.wl_deactivation_reason codes); NULL = all 0 */
} kb_snapshot;

/* ------------------------------------------------------------------------
 * Output of one cycle, caller-allocated, indexed by ENTRY (position in
 * heads[]) unless stated otherwise.
 * ---------------------------------------------------------------------- */
typedef struct kb_cycle_out {
  uint8_t *decision;     /* [n_heads] KB_DEC_*                                          */
  uint8_t *mode;         /* [n_heads] Assignment.RepresentativeMode()                   */
  int32_t *borrow;       /* [n_heads] Assignment.Borrowing (flavorassigner.go:128)      */
  int32_t *commit_rank;  /* [n_heads] position in the iterator order among the entries of
                            the same ROOT cohort (scheduler.go:778-817 / tournament)     */
  /* per podset, indexed like the INPUT podset tables: row = wl_ps_start[wl] + podset
   * for wl = heads[entry].  Rows of workloads that are not heads are left untouched. */
  int8_t  *ps_flavor;    /* [n_podset][R] assigned global flavor idx or -1
                            (PodSetAssignment.Flavors, flavorassigner.go:262-273)        */
  int8_t  *ps_res_mode;  /* [n_podset][R] FlavorAssignment.Mode or -1                   */
  int8_t  *ps_tried_idx; /* [n_podset][R] FlavorAssignment.TriedFlavorIdx (-1 none)     */
  int32_t *ps_count;     /* [n_podset] admitted Count (partial admission)               */
  /* preemption targets, CSR by entry (preemption.go:111-115) */
  int32_t *tgt_start;    /* [n_heads+1]                                                 */
  int32_t *tgt_adm;      /* [tgt_capacity] index into admitted tables                   */
  uint8_t *tgt_reason;   /* [tgt_capacity] KB_REASON_*                                  */
  int32_t tgt_capacity;
  int32_t n_targets;     /* out: total targets written                                  */
  /* final node usage after the cycle [n_cq+n_cohort][F*R] (may be NULL) */
  int64_t *node_usage;
} kb_cycle_out;

/* Per-(node, fr) quota state, for K1 parity (TestAvailable / TestDominantResourceShare). */
typedef struct kb_tree_out {
  int64_t *subtree_quota;        /* [N][FR] resourceNode.SubtreeQuota                    */
  int64_t *usage;                /* [N][FR] resourceNode.Usage (cohorts accumulated)     */
  int64_t *available;            /* [n_cq][FR] ClusterQueueSnapshot.Available            */
  int64_t *potential_available;  /* [n_cq][FR] ClusterQueueSnapshot.PotentialAvailable   */
  int64_t *drs_rounded;          /* [N] DRS.roundedWeightedShare value                   */
  int32_t *drs_resource;         /* [N] dominant resource idx or -1                      */
  uint8_t *drs_borrowing;        /* [N]                                                  */
} kb_tree_out;

typedef struct kb_stats {
  double last_cycle_gpu_ms;      /* device time of the last kb_* compute call            */
  double last_h2d_ms, last_d2h_ms;
  int64_t h2d_bytes, d2h_bytes;  /* of the last call                                     */
  int32_t kernel_launches;       /* kernels of this library launched by the last call    */
  int32_t sm_count;
  /* per-kernel device time of the last kb_cycle_resident when kb_set_profile(h, 1):
   * CUDA events recorded on the launching stream around each kernel.  After kb_run_drain: summed over its cycles,
   * KB_K_DRAIN = the queue layer after every cycle (decisions applied, admissions, penalties, next heads). */
  float   kernel_ms[KB_N_KERNELS];
  /* target-search counters of the last cycle: [0] searches run, [1] candidate records classified (32 B each),
   * [2] candidates visited by the greedy loops, [3] workloads removed (incl. fill-back), [4] the part of [1] classified by
   * multi-column searches (GetTargets of k_nominate_walk),
   * [5..7] SM clock cycles summed over warps: column load / classification / greedy (diagnostics) */
  int64_t search_stat[8];
  /* after a cycle run by the fused flat-cohort kernel (k_cycle_flat), over the first 1024 entries of the first root:
   * [0] entries nominated by the group walk (one podset that cannot be reduced), [1] all entries */
  int64_t flat_group_walk[2];
} kb_stats;

/* indices into kb_stats.kernel_ms */
enum { KB_K_TREE = 0, KB_K_LONE = 1, KB_K_NOMINATE = 2, KB_K_SCAN = 3, KB_K_SCATTER = 4,
       KB_K_ADMIT = 5, KB_K_RANK = 6, KB_K_PREEMPT = 7 /* fair-sharing target search (+ k_over) */,
       KB_K_RANKADM = 8 /* ranking of the admitted workloads */, KB_K_SEARCH_TABLES = 9 /* k_columns + candidate buckets */,
       KB_K_SEARCH_CELLS = 10, KB_K_WALK = 11, KB_K_FAIR_PREP = 12, KB_K_DRAIN = 13 /* queue layer of kb_run_drain */,
       KB_K_TAS = 14 /* kb_tas_find, all kernels */, KB_K_CYCLE_ROOT = 15 /* fused per-root cycle */,
       KB_K_TAS_LEAF = 16, KB_K_TAS_REDUCE = 17, KB_K_TAS_SELECT = 18 };

typedef struct kb_handle kb_handle;

typedef struct kb_config {
  int32_t device;        /* CUDA device ordinal */
  int32_t reserved;
} kb_config;

/* lifecycle */
int32_t kb_create(const kb_config *cfg, kb_handle **out);
void    kb_destroy(kb_handle *h);
const char *kb_last_error(const kb_handle *h);
int32_t kb_alloc_pinned(void **ptr, uint64_t bytes);
int32_t kb_free_pinned(void *ptr);
/* Output buffers of kb_run_cycle / kb_download in ONE page-locked block laid out like the library's device-side
 * result tables: the eight per-entry / per-podset tables then come back with a single DMA (separately allocated
 * buffers work too, one copy per table).  n_node_cells = (n_cq + n_cohort) * F * R to receive node_usage, 0 to leave
 * it NULL.  Fills every pointer of *out and tgt_capacity; release with kb_free_pinned(out->decision).
 * Replaces the per-cycle result maps of the reference's loop (entry.assignment / preemptionTargets, scheduler.go:255-401). */
int32_t kb_alloc_cycle_out(int32_t n_heads, int32_t n_podset, int32_t n_resource, int32_t tgt_capacity, int64_t n_node_cells, kb_cycle_out *out);
int32_t kb_version(void);

/* K1: rebuild the resource-node tree on the device and return the derived
 * quantities (resource_node.go:91-133,183-217; fair_sharing.go:126-174). */
int32_t kb_tree_eval(kb_handle *h, const kb_snapshot *s, kb_tree_out *out);

/* One scheduling cycle over s->heads: nominate (scheduler.go:464-501) ->
 * iterator (:752-821, fair_sharing_iterator.go) -> admit loop (:269-401).
 * Host buffers in, host buffers out (copies inside). */
int32_t kb_run_cycle(kb_handle *h, const kb_snapshot *s, kb_cycle_out *out);

/* Split form used by the resident-input benchmark and by drain mode:
 * upload once, run many.  kb_cycle_resident runs the same kernels as
 * kb_run_cycle on the uploaded snapshot and leaves results on the device;
 * kb_download copies them out. */
int32_t kb_upload(kb_handle *h, const kb_snapshot *s);
int32_t kb_cycle_resident(kb_handle *h);
int32_t kb_download(kb_handle *h, kb_cycle_out *out);

/* Drain mode (SURVEY.md §8d): iterate scheduling cycles over a snapshot whose pending tables hold WHOLE QUEUES
 * (s->heads / s->n_heads are ignored) until a cycle admits nothing or max_cycles is reached.  The queue layer of
 * pkg/cache/queue runs on the device: per-ClusterQueue order by queueOrderingFunc (cluster_queue.go:636-685), one
 * head per ClusterQueue per cycle (manager.go:770-794), and after every cycle what schedule() + requeueAndUpdate do
 * (scheduler.go:405-418,823-850):
 *   assumed                 -> leaves the queue; Assignment.Usage joins the ClusterQueue usage, the workload joins
 *                              the admitted tables (QuotaReserved time = now_ns + cycle);
 *   every other entry       -> keeps LastAssignment (tried flavor indexes + ClusterQueue generation), nil after
 *                              issuing preemptions (scheduler.go:345);
 *   StrictFIFO              -> stays the head (cluster_queue.go:622-624);
 *   BestEffortFIFO          -> skipped / preempting entries stay; NoFit and Preempt-without-targets entries stay only
 *                              while LastAssignment.PendingFlavors() (workload.go:163-176), else the next workload
 *                              becomes the head; a NoFit head with a known wl_sched_hash also sets aside every queued
 *                              workload of its class (handleInadmissibleHash, cluster_queue.go:408-425).
 * Without kb_snapshot.adm_wl evictions are not replayed: the targets of a Preempting entry stay admitted, and the drain
 * ends with the first cycle that admits nothing.  With adm_wl the drain takes the limit in which every eviction issued
 * in cycle c completes before cycle c+1 (in the reference it completes asynchronously), in this order:
 *   1. the decisions are applied as above;
 *   2. every target of every Preempting entry (adm_evicted or not) leaves the admitted tables: its cells leave its own
 *      ClusterQueue's usage (cache.DeleteWorkload), its row is removed (the other rows keep their order), and its
 *      record adm_wl[row] returns to its queue at once (preemption sets no RequeueState, workload_controller.go:827-832)
 *      with LastAssignment nil (wl_last_gen = -1, ps_last_tried = -1, HasQuotaReservation false);
 *   3. for every root cohort with a victim in its tree (the ClusterQueue itself when it has no cohort) every workload
 *      its ClusterQueues set aside returns to its queue and keeps its LastAssignment (requeueWorkloadsCohort /
 *      queueInadmissibleWorkloads, inadmissible_workloads.go:128-223; the scheduling-hash sets are cleared);
 *   4. the head of every queue in cycle c+1 is its first queued workload in queueOrderingFunc order; a requeued victim
 *      takes the place its priority, creation timestamp and UID give it (workload.go:1174-1193).
 * The drain then ends after the first cycle that neither admits nor evicts.  Evictions under way before the drain
 * (adm_evicted rows that are never targeted) are not completed, except with kb_snapshot.adm_evict_end_ns (eviction
 * latency, below).
 * Cycle c runs with now_ns + c.  Bit-exact with iterating kb_run_cycle under the same rules (kueue_b200/drain.py).
 * With the AdmissionFairSharing tables (kb_snapshot.wl_lq != NULL), the queue of a ClusterQueue with cq_afs set is one
 * segment per LocalQueue, each in the order above; its head is the workload with the smallest (LocalQueue usage by
 * cmp.Compare — NaN first —, -priority, timestamp, UID) among the segments' heads, and every admission adds its entry
 * penalty to its LocalQueue before the next cycle.  StrictFIFO keeps the head (the next cycle picks the minimum again),
 * BestEffortFIFO advances the head's own segment, the scheduling-hash move covers every segment of the ClusterQueue.
 * Consumed usage does not decay inside a drain, except in event mode with kb_snapshot.lq_last_update_ns (see there).
 *
 * Event mode (kb_snapshot.wl_create_ns / wl_run_ns / adm_finish_ns / wl_evict_ns, any non-NULL): a simulated clock t starts at
 * now_ns; cycle c runs at t_c (its now_ns and the QuotaReserved time of its admissions).  Two more queue states:
 * ABSENT (created after t, in no queue) and FINISHED (never requeued).  A pending event is the finish time of a live
 * admitted row or the creation time of an ABSENT workload.  The loop:
 *   1. no queue has a head: t jumps to E, the earliest pending event, and steps 5-7 apply the events at E (no cycle is
 *      counted); without E the drain ends;
 *   2. cycle c runs at t_c and its decisions are applied as above; 3. evictions are replayed as above (adm_wl);
 *   4. a cycle that admitted or evicted: t_{c+1} = t_c + drain_cycle_ns; a quiet cycle (the stop rule of the plain
 *      drain) waits instead: t_{c+1} = max(t_c + drain_cycle_ns, E), and without E the drain ends;
 *   5. every live row with finish <= t_{c+1} finishes (a row admitted at t finishes at t + wl_run_ns, saturating; one
 *      admitted in cycle c that finishes by t_{c+1} never enters the tables): its cells leave its ClusterQueue's usage,
 *      its row is removed, its record (adm_wl for the rows of the snapshot) becomes FINISHED, its root tree is marked;
 *   6. every ABSENT workload with create <= t_{c+1} joins its queue, except that in a BestEffortFIFO ClusterQueue a
 *      workload whose known wl_sched_hash is in the ClusterQueue's NoFit set goes straight to the inadmissible set
 *      (PushOrUpdate, cluster_queue.go:288-293).  The NoFit set holds the hashes of the NoFit heads since the
 *      ClusterQueue's last inadmissible requeue (handleInadmissibleHash :414; cleared by queueInadmissibleWorkloads,
 *      inadmissible_workloads.go:174);
 *   7. the inadmissible requeue of step 3 runs over every root tree marked in steps 3 or 5;  8. heads of cycle c+1.
 * Steps 5-7 only set state bytes and lower cursors: their order does not change the result.  A quiet cycle waiting for
 * the next event is the canonical choice; with every run time < 0 and every creation <= now_ns the drain equals the
 * plain drain.  An evicted workload loses its finish time; a readmission restarts the full run time.  The clock is
 * global (a quiet cycle depends on every root), so event drains are not sharded.  max_cycles counts cycles; the drain
 * stops before running cycle max_cycles.  Events applied before cycle 0 count in n_finished / n_arrived only; the
 * events applied between the start of cycle c and the start of cycle c+1 count in cycle_finished / cycle_arrived[c].
 *
 * Eviction latency (kb_snapshot.wl_evict_ns != NULL, with adm_wl; event mode): an eviction is issued at once and
 * completes later, on the clock, as in the reference (preemption.go:175-215 issues, reconciler.go:576-590 releases the
 * quota once the pods are gone, workload_controller.go:973-1004 requeues).  Step 3 becomes the issue and the release
 * joins step 5:
 *   3. issue at t_c: every target row of every Preempting entry that is not already evicting gets adm_evicted = 1 and
 *      the end time t_c + wl_evict_ns[adm_wl[row]] (saturating at INT64_MAX), which replaces its finish time (an
 *      evicted workload never finishes; the runner's controller.go:119-127).  It counts in cycle_evicted, n_evicted,
 *      wl_evictions and the active-cycle rule of step 4.  The row keeps its cells in the usage and stays in the
 *      admitted tables, a preemption candidate ordered first because it is evicted (preemption/common/ordering.go:
 *      41-47); its record still holds quota.  A target already evicting gets nothing ("Preemption ongoing",
 *      preemption.go:183-186): its preemptor stays PendingPreemption (scheduler.go:345-358), and a cycle whose
 *      Preempting entries only re-target evicting rows is quiet and waits for E;
 *   5. every evicting row with end <= t_{c+1} completes: its cells leave the usage, its row is removed, its record
 *      returns to its queue with LastAssignment nil and HasQuotaReservation false, and its root tree is marked for the
 *      requeue of step 7.  It counts in n_evict_done / cycle_evict_done.  E includes these end times.
 * Rows with adm_evicted set before the drain complete at adm_evict_end_ns and count as ongoing when targeted; without
 * that table they are issued at t_c like any other row.  With every wl_evict_ns <= max(drain_cycle_ns, 1) and no
 * adm_evict_end_ns the drain equals the drain without latency (heads, decisions, evictions, usage, per-workload
 * results): every issued eviction completes at the next boundary, and steps 5-7 do not depend on their order.
 *
 * Sticky workload (kb_snapshot.cq_sticky != NULL; plain and event drains): one slot per ClusterQueue, seeded from the
 * table, as the reference keeps a preemptor that waits for its evictions at the head of its queue
 * (cluster_queue.go:64-93,330-340,609-624,656-665):
 *   - heads (step 4 / 8): a ClusterQueue whose sticky workload is queued takes it as its head; otherwise the head is its
 *     first queued workload.  A set-aside sticky workload has no effect and is first again once requeued;
 *   - after the decisions (step 1): an assumed head that is its ClusterQueue's sticky workload clears the slot (admission
 *     deletes the workload from its queue, workload_controller.go:965-966); a Preempting head of a BestEffortFIFO
 *     ClusterQueue becomes the sticky workload (scheduler.go:344-358: targets already evicting count,
 *     preemption.go:183-194), replacing the previous one; every other decision leaves the slot alone, a sticky head
 *     that goes NoFit and is set aside included;
 *   - arrivals, completions, releases and the inadmissible requeue only change state bytes.  The head may lie past the
 *     first queued workload: it is set aside from its own position, and the scheduling-hash move excludes it by identity.
 * With every slot -1 at the start the drain equals the drain without the table when (a) there is no adm_wl and no event
 * table (nothing ahead of a Preempting head ever becomes queued again), (b) every ClusterQueue is StrictFIFO, or (c) no
 * ClusterQueue has a preemption policy.
 * Not modelled: preemption expectations between issue and observation (the drain observes an eviction at once).
 *
 * Admission checks (kb_snapshot.wl_check_ns != NULL, with adm_wl; event mode).  Two more queue states: BACKOFF and
 * DEACTIVATED.  Each record has a queue-order timestamp: wl_check_evict_ns when set (records adm_wl does not name),
 * else wl_ts.  Additions to the loop above:
 *   1. an admission at t_c of a workload with wl_check_ns > 0 reserves quota and starts attempt k = RetryCount + 1; its
 *      verdict comes at t_c + wl_check_ns (saturating).  With 0 the row is Ready at t_c, as without the tables;
 *   2. verdicts are events (E includes them), applied in step 5 before the completions.  Ready (no failure left):
 *      wl_ready_ns = verdict, finish = verdict + wl_run_ns (saturating), the row may finish in the same boundary.
 *      Retry (a failing attempt, k <= check_backoff_limit): the row's cells leave the usage, the row is removed, its
 *      root tree is marked; the record goes to BACKOFF with RequeueAt = verdict + WaitTime(k), RetryCount = k, queue
 *      timestamp = verdict and LastAssignment nil.  Rejected (k > limit): released the same way, the record is
 *      DEACTIVATED and never queued again.  A failing attempt uses up one unit of wl_check_fail;
 *   3. a BACKOFF record whose RequeueAt <= t_{c+1} arrives through step 6 (NoFit rule included); E includes RequeueAt;
 *   4. an admission resets the queue timestamp to wl_ts; the new row's adm_ts is wl_ts;
 *   5. a preempted row whose checks run holds no pods: with wl_evict_ns it is released at the next boundary; the
 *      attempt under way is dropped, not counted and uses up no failure (a canonical choice);
 *   6. the cycle sees the queue timestamp (entry order, preemption policy), and the queues are re-sorted by it whenever a
 *      record enters its queue with a timestamp other than the key of its position (n_resorts);
 *   7. with every wl_check_ns = 0, every wl_check_fail = 0 and no start-state tables the drain equals the drain without
 *      the tables.
 * WaitTime(k) is wait.NewBackoff(base, max, 2, 0.0001).WaitTime(k) truncated to whole seconds (kb_drain.cuh
 * kb_check_wait_ns; exact below 10,000 s): min(check_backoff_base_s * 2^(k-1), check_backoff_max_s or infinity), except
 * that with base > max > 0 the first Step returns the base uncapped (attempt 1 waits base, later ones max).  Verdicts
 * applied between the start of cycle c and of c+1 count in cycle_check_retry / cycle_check_rejected[c].
 *
 * WaitForPodsReady (kb_snapshot.wl_pods_ready_ns != NULL, with adm_wl; event mode).  It uses the BACKOFF and
 * DEACTIVATED states, RequeueAt, the queue-order timestamp and the re-sort of the admission checks above.  An attempt is
 * one admission of a workload.  Additions to the loop:
 *   1. the attempt starts at Admitted: the reservation at t_c when the workload has no check delay, else the Ready
 *      verdict time;
 *   2. it fails if the record has failures left in wl_pods_ready_fail (it uses up one; INT32_MAX = every attempt fails)
 *      or wl_pods_ready_ns > pods_ready_timeout_ns; otherwise it is ready.  A delay equal to the timeout is ready (a
 *      canonical tie-break).  A ready attempt reaches PodsReady at Admitted + wl_pods_ready_ns (wl_pods_ready_at_ns) and
 *      finishes at PodsReady + wl_run_ns (saturating): no event is added.  With every delay 0 this is the finish without
 *      the block;
 *   3. a failing attempt has an event at T = Admitted + pods_ready_timeout_ns (saturating; E includes it), applied in
 *      step 5 after that boundary's check verdicts (a Ready verdict and its timeout can fall in one boundary) and before
 *      its completions (workload_controller.go:805-835,1106-1130).  With pods_ready_backoff_limit >= 0 and Count + 1 >
 *      limit it is a deactivation (triggerDeactivation :840-855): Count = 0, the record will be DEACTIVATED and
 *      wl_deactivated = 1.  Otherwise (UpdateRequeueState workload.go:707-722) Count += 1 (saturating at INT32_MAX),
 *      RequeueAt = T + WaitTime(Count) (saturating), and under the Eviction timestamp the queue timestamp becomes T
 *      (GetQueueOrderTimestamp workload.go:1174-1182; under Creation it is unchanged);
 *   4. the timed-out row is evicted at T.  With wl_evict_ns it gets adm_evicted and the end time T + wl_evict_ns: it keeps
 *      its cells, stays a preemption candidate, and a preemptor that targets it is ongoing (as for an evicting row).
 *      Without, it is released at the boundary that applies T.  At release its cells leave the usage, the row is
 *      removed, its root tree is marked, and the record goes to DEACTIVATED or to BACKOFF with LastAssignment nil; a
 *      BACKOFF record is queued by rule 3 of the admission checks (at RequeueAt, in that same boundary when RequeueAt
 *      <= t_{c+1}, NoFit rule included);
 *   5. a row preempted while its attempt waits for PodsReady (before PodsReady, or before T) loses the attempt: it is not
 *      counted, uses up no failure (workload_controller.go:808-811), and wl_pods_ready_at_ns keeps its previous value.
 *      The row is released like any preempted row, with its pods' latency;
 *   6. an admission resets the queue timestamp to wl_ts; Count survives a ready attempt;
 *   7. start state: wl_pods_ready_count (Count), adm_admitted_ns (rows whose pods are not ready: their attempt runs from
 *      there by rules 2-3, in place of adm_finish_ns), wl_requeue_at_ns (records in backoff) and wl_pods_ready_evict_ns
 *      (the queue timestamp under Eviction of a record adm_wl does not name);
 *   8. with every wl_pods_ready_ns = 0, every wl_pods_ready_fail = 0 and no start-state tables the drain equals the drain
 *      without the block.
 * WaitTime(k) is the jitter-free Backoff.WaitTime of wait.NewBackoff(base_s, max_s, 2, 0.0001) in nanoseconds (kb_drain.cuh
 * kb_pods_ready_wait_ns):
 * min(base * 2^(k-1), max, or MaxInt64 / 2 with max 0), the base uncapped for k = 1, and 0 with base 0.  The reference
 * adds a random jitter below wait * 1e-4 and stores RequeueAt at second precision; the drain takes the jitter-free value.
 * Timeouts applied between the start of cycle c and of c+1 count in cycle_pods_ready_timeout / _deactivated[c].
 * Not modelled: waitForPodsReady.blockAdmission (the reference stops the admit loop mid-cycle until every admitted
 * workload is ready, scheduler.go:361-373, which a cycle evaluated at one instant cannot express) and recoveryTimeout
 * (the drain models no pod failure after PodsReady).
 *
 * MaximumExecutionTimeSeconds (kb_snapshot.wl_max_exec_s != NULL, with adm_wl; event mode).  Every record has a limit
 * max (wl_max_exec_s, 0 = nil) and an accumulated time acc (wl_exec_acc_s, -1 = nil, read as 0 below).  Additions:
 *   1. every row has an Admitted time A: the reservation t_c when the workload has no check delay, else its Ready
 *      verdict time; a row whose checks run has none (SyncAdmittedCondition admissionchecks.go:36-70: Admitted is
 *      QuotaReserved with every check Ready).  A row of a record with a limit has the deadline D = A + (max - acc) * 1e9
 *      (saturating) and the effective deadline max(D, A, now_ns): a negative max - acc, or a snapshot row already past
 *      its limit, expires at the first boundary that can apply it (reconcileMaxExecutionTime workload_controller.go:
 *      619-646 computes remaining = (max - acc) s - (now - A) and acts on remaining <= 0);
 *   2. the expiry is an event: the finish column holds the earlier of the row's own next event (its finish, or the
 *      PodsReady timeout T of a failing attempt) and the effective deadline, and a row whose deadline came first is
 *      marked (kb_drain.cuh KB_PH_EXPIRE).  Ties go to the own event: a finish at the deadline finishes, a PodsReady
 *      timeout at the deadline is a timeout (rule 4 then deactivates the workload at its release).  Expiries are applied
 *      in step 5 after the check verdicts and the PodsReady timeouts, before the completions;
 *   3. at its expiry the workload is deactivated (reason MaximumExecutionTimeExceeded, SetDeactivationTarget
 *      :619-646; the inactive branch :316-321,386-420 evicts it and clears RequeueState: Count 0, no RequeueAt) and acc
 *      becomes nil.  A WaitForPodsReady attempt still waiting is dropped (not counted, no failure used,
 *      wl_pods_ready_at_ns keeps its previous value).  The row is evicted at the effective deadline: with wl_evict_ns it
 *      holds its cells as an evicting row until deadline + latency (a preemptor that targets it is ongoing); without, it
 *      is released at the boundary that applies the deadline.  At release the record is DEACTIVATED;
 *   4. every release of a row that has an Admitted time (a completed preemption, a PodsReady-timeout release, an expiry
 *      release) adds d = int32(Duration(t - A).Seconds()) to acc, or sets acc = d when nil (the Admitted true -> false
 *      transition happens when the quota reservation is removed, UnsetQuotaReservationWithCondition workload.go:684-704,
 *      so termination latency counts).  t is the end of the eviction: T or the effective deadline without latency, t_c
 *      for a preemption without latency.  Completions and rows whose checks run add nothing.  Truncation is per
 *      attempt: Seconds() is float64(sec) + float64(nsec) / 1e9, which from about 2^24 s can round up to sec + 1
 *      (kb_drain.cuh kb_exec_seconds).  If a row's deadline D is at or before its release t and the workload was not
 *      deactivated already (RequeuingLimitExceeded sets DeactivationTarget first, :840-851, and reconcileMaxExecutionTime
 *      then leaves it), rule 3 applies at that release in place of the requeue or the backoff: a deadline that passes
 *      while an eviction is under way (both reconcilers run while the reservation is held, :509-536).  It leaves acc =
 *      d of that last attempt (the nil reset, then the addition) and counts at the boundary of the release;
 *   5. condition times keep nanoseconds (the API server stores seconds).  With every limit nil and no start state the
 *      drain equals the drain without the block in heads, decisions, evictions, usage and per-workload results; only
 *      wl_exec_acc_s_out is new.
 * Deactivations (at an expiry or a release) between the start of cycle c and of c+1 count in
 * cycle_max_exec_deactivated[c].  Not modelled: MultiKueue's handling of the field.  Reactivation: see below.
 *
 * Quota changes (kb_snapshot.n_quota_change > 0 with every qc_* table; event mode).  Edit i replaces the three quota
 * rows of node qc_node[i] at qc_ns[i].  Additions to the loop:
 *   1. every edit time is a pending event: E includes the next edit not applied yet; a quiet cycle waits for it, with no
 *      head the clock jumps to it; after the last edit the stop rule is as before;
 *   2. at a boundary t -> t' every edit with qc_ns in (t, t'] is applied in table order, in step 5 before the check
 *      verdicts: its rows replace the node's (of two edits of one node in one boundary the later wins);
 *   3. an edit whose three rows equal the node's rows at that point changes nothing (specUpdated is false: no bump, no
 *      requeue); it still counts in n_quota_changes;
 *   4. every other edit adds 1 to AllocatableResourceGeneration of every ClusterQueue of the node's root tree (of the
 *      ClusterQueue alone when it has no cohort), which outdates every remembered LastAssignment there
 *      (lastAssignmentOutdated flavorassigner.go:533: the next attempt searches flavors from the first), and marks the
 *      root tree for the inadmissible requeue of step 7 (its NoFit sets are cleared, as in any requeue);
 *   5. nothing is evicted: admitted rows keep their cells, usage above the new quota stays (as in the reference);
 *   6. the LastAssignment of an entry that stays pending records the current generation;
 *   7. the block composes with eviction latency, the sticky table, admission checks, WaitForPodsReady,
 *      MaximumExecutionTimeSeconds and AFS with or without decay: none of their rules reads quotas.
 * Edits applied between the start of cycle c and of c+1 count in cycle_quota_changes[c]; cq_generation receives the
 * generations after the drain, for the caller to write back.  Resident tables: the drain edits the handle's device
 * copies of nominal / borrow_limit / lend_limit / cq_generation and the tables derived from them, so a kb_run_drain with
 * the block on resets the handle's static generation: the next kb_run_cycle / kb_upload on the handle uploads its
 * static tables again whatever its static_generation.
 *
 * Deactivation and reactivation (kb_snapshot.n_active_change > 0 with every ac_* table: event mode; and / or
 * kb_snapshot.wl_inactive; both need adm_wl).  Edit i sets spec.active of record ac_wl[i] to ac_active[i] at ac_ns[i].
 * In the reference an Update event that leaves a workload inactive takes the `status == Finished || !active` branch
 * (workload_controller.go:937-952): queues.DeleteWorkload and, inside QueueAssociatedInadmissibleWorkloadsAfter,
 * cache.DeleteWorkload at once, whatever the status: a deactivated workload leaves the usage and the preemption
 * candidates when spec.active turns false, not when its pods are gone.  Additions to the loop:
 *   1. every edit time is a pending event: E includes the next edit not applied yet, a quiet cycle waits for it, with no
 *      head the clock jumps to it.  At a boundary t -> t' the edits with ac_ns in (t, t'] are applied in table order.
 *      A record's edits are ordered in time against its own events (arrival, finish, check verdict, PodsReady timeout,
 *      expiry, eviction end, RequeueAt); an own event at the time of an edit goes first;
 *   2. stop, record active and holding no row (QUEUED, SET_ASIDE, BACKOFF): it leaves its queue and is DEACTIVATED
 *      with reason 4 (Deactivated by a user); RequeueState is cleared (Count 0, no RequeueAt; the inactive branch
 *      :386-420); a sticky workload clears its ClusterQueue's slot (delete, cluster_queue.go:330-340); its root tree is
 *      marked for the inadmissible requeue (QueueAssociatedInadmissibleWorkloadsAfter, manager.go:676-697);
 *   3. stop at d, record active and holding a row in any phase (running, checks under way, waiting for PodsReady,
 *      evicting): the row's cells leave the usage at d and the row is removed; the root tree is marked; RequeueState is
 *      cleared and a PodsReady attempt still waiting is dropped, as at an expiry; a check attempt under way is dropped
 *      (not counted, no failure used); the record is DEACTIVATED with reason 4 and LastAssignment nil.  A row with an
 *      Admitted time adds int32(Seconds) of t - Admitted to acc (rule 4 of MaximumExecutionTimeSeconds), with t the
 *      QuotaReserved unset, which comes after the pods terminate (jobframework/reconciler.go:576-590): the end of an
 *      eviction already under way, else d + wl_evict_ns (d without the table).  acc is not reset (only
 *      MaximumExecutionTimeExceeded resets it, :635);
 *   4. stop, record already inactive (whatever its state) or FINISHED: nothing changes; the edit still counts as applied;
 *   5. resume, record DEACTIVATED (any reason): reason 0, and it joins its queue as an arrival does (PushOrUpdate, the
 *      NoFit rule of a BestEffortFIFO ClusterQueue included; with AFS in its LocalQueue's segment), with LastAssignment
 *      nil (queues.DeleteWorkload dropped its queue entry) and Count 0.  wl_check_retries is unchanged, as at every
 *      eviction the drain replays (resetChecksOnEviction admissionchecks.go:88-109 keeps the RetryCount of a Pending
 *      check).  A resume on any other record changes nothing: an active one, or one still holding a row while the
 *      eviction of its deactivation (MaximumExecutionTimeExceeded, RequeuingLimitExceeded) is under way;
 *   6. the queue-order timestamp does not change: a deactivation sets Evicted(reason Deactivated) only on a workload
 *      that is not evicted, and GetQueueOrderTimestamp (workload.go:1174-1193) reads creation time for that reason; an
 *      evicted record keeps its Evicted condition and its timestamp.  A record that rejoins its queue with a timestamp
 *      other than its sort key re-sorts the queues as a requeue after a backoff does;
 *   7. start state: a record with wl_inactive 1-4 starts DEACTIVATED with that reason, in no queue, without RequeueAt;
 *   8. the block composes with eviction latency, the sticky table, admission checks, WaitForPodsReady,
 *      MaximumExecutionTimeSeconds, quota changes and AFS with or without decay; with no edit and every wl_inactive 0
 *      the drain equals the drain without the block in every output.
 * n_stopped / n_resumed count the edits that changed the state (rules 2, 3, 5); those applied between the start of
 * cycle c and of c+1 count in cycle_stopped[c] / cycle_resumed[c].  wl_deactivated / wl_deactivation_reason describe
 * the state at the end: 1 and the reason while the record is inactive, 0 after a reactivation. */
typedef struct kb_drain_out {
  int32_t max_cycles;        /* in */
  int32_t n_cycles;          /* out: cycles run */
  int64_t n_decisions;       /* out: entries evaluated over all cycles */
  int64_t n_admitted;        /* out */
  int32_t *cycle_heads;      /* [max_cycles] entries per cycle (may be NULL) */
  int32_t *cycle_admitted;   /* [max_cycles] admissions per cycle (may be NULL) */
  /* per pending workload [n_wl] (each may be NULL) */
  int32_t *wl_admit_cycle;   /* cycle of its last admission if it holds quota at the end, else -1 */
  uint8_t *wl_last_decision; /* KB_DEC_* of its last evaluation, 0xff = never a head */
  int32_t *wl_evals;         /* cycles that evaluated it */
  /* assignment of the last evaluation, indexed like the input podset tables (may be NULL) */
  int8_t  *ps_flavor;        /* [n_podset][R] */
  int32_t *ps_count;         /* [n_podset] */
  int64_t *cq_usage;         /* [n_cq][F*R] ClusterQueue usage after the drain (may be NULL) */
  /* optional trace for parity checks: entries of every cycle in order, concatenated */
  int32_t *trace_wl;         /* [trace_capacity] pending workload index */
  uint8_t *trace_decision;   /* [trace_capacity] KB_DEC_* */
  int64_t trace_capacity;
  double gpu_ms;             /* out: device time of all cycles (kernels of the cycles + queue layer) */
  /* eviction replay (kb_snapshot.adm_wl != NULL; zero otherwise) */
  int64_t n_evicted;         /* out: evictions over all cycles */
  int32_t *cycle_evicted;    /* [max_cycles] evictions per cycle (may be NULL) */
  int32_t *wl_evictions;     /* [n_wl] times each pending record was evicted (may be NULL) */
  /* event mode (zero / unset otherwise; every pointer may be NULL) */
  int64_t n_finished;        /* out: completions applied */
  int64_t n_arrived;         /* out: arrivals applied */
  int64_t end_ns;            /* out: the clock when the drain stopped (last cycle start or last event applied) */
  int64_t *cycle_start_ns;   /* [max_cycles] t_c */
  int32_t *cycle_finished;   /* [max_cycles] completions applied from the start of cycle c to the start of c+1 */
  int32_t *cycle_arrived;    /* [max_cycles] arrivals, likewise */
  int64_t *wl_admit_ns;      /* [n_wl] time of the workload's last admission, INT64_MIN if never admitted */
  int64_t *wl_finish_ns;     /* [n_wl] finish time, INT64_MAX if it has not finished */
  /* decay of consumed usage (kb_snapshot.lq_last_update_ns != NULL; untouched otherwise; each pointer may be NULL):
     the AfsConsumedResources entries after the drain, for AfsConsumedResources.Set */
  int64_t *lq_consumed;       /* [n_lq][R] int64Amount values (0 = absent) */
  int32_t *lq_consumed_scale; /* [n_lq][R] their scales */
  int64_t *lq_last_update_ns; /* [n_lq] LastUpdate */
  int64_t n_afs_samples;      /* out: decay samples due over the drain (those a fixed point skips included); 0 without decay */
  /* eviction latency (kb_snapshot.wl_evict_ns != NULL; zero / untouched otherwise; the pointer may be NULL) */
  int64_t n_evict_done;       /* out: evictions completed (quota released), those before cycle 0 included */
  int32_t *cycle_evict_done;  /* [max_cycles] evictions completed from the start of cycle c to the start of c+1 */
  /* sticky workload (kb_snapshot.cq_sticky != NULL; untouched otherwise; the pointer may be NULL): the slots after the
     drain, for the caller to write back */
  int32_t *cq_sticky;         /* [n_cq] pending index of each ClusterQueue's sticky workload, -1 = none */
  /* admission checks (kb_snapshot.wl_check_ns != NULL; zero / untouched otherwise; each pointer may be NULL) */
  int64_t n_check_ready, n_check_retry, n_check_rejected;  /* out: verdicts over the drain, those before cycle 0 included */
  int32_t *cycle_check_retry;    /* [max_cycles] Retry verdicts applied from the start of cycle c to the start of c+1 */
  int32_t *cycle_check_rejected; /* [max_cycles] Rejected verdicts, likewise */
  int64_t *wl_ready_ns;          /* [n_wl] time of the last Admitted in the drain, INT64_MIN if none */
  int32_t *wl_check_retries_out; /* [n_wl] final RetryCount */
  uint8_t *wl_deactivated;       /* [n_wl] 1 if the workload was deactivated (Rejected, RequeuingLimitExceeded with
                                    kb_snapshot.wl_pods_ready_ns or MaximumExecutionTimeExceeded with
                                    kb_snapshot.wl_max_exec_s, which also write it and the two fields below) */
  int64_t n_resorts;             /* out: queue re-sorts (a record entered its queue with a new queue-order timestamp) */
  double resort_ms;              /* out: device time of those re-sorts (part of gpu_ms) */
  /* WaitForPodsReady (kb_snapshot.wl_pods_ready_ns != NULL; zero / untouched otherwise; each pointer may be NULL).
     n_evicted, wl_evictions and n_evict_done keep counting preemptions only. */
  int64_t n_pods_ready_timeout;          /* out: timeouts that requeue (deactivations excluded), those before cycle 0 included */
  int64_t n_pods_ready_deactivated;      /* out: timeouts past the requeue limit */
  int32_t *cycle_pods_ready_timeout;     /* [max_cycles] timeouts applied from the start of cycle c to the start of c+1 */
  int32_t *cycle_pods_ready_deactivated; /* [max_cycles] deactivations, likewise */
  int64_t *wl_pods_ready_at_ns;          /* [n_wl] PodsReady time of the last attempt that reached it, or will (a row still
                                            waiting at the end of the drain); INT64_MIN if none */
  int32_t *wl_pods_ready_count_out;      /* [n_wl] final RequeueState.Count */
  /* MaximumExecutionTimeSeconds (kb_snapshot.wl_max_exec_s != NULL; zero / untouched otherwise; each pointer may be
     NULL).  wl_deactivation_reason is written whenever wl_deactivated is. */
  int64_t n_max_exec_deactivated;        /* out: deactivations for MaximumExecutionTimeExceeded, those before cycle 0 included */
  int32_t *cycle_max_exec_deactivated;   /* [max_cycles] deactivations from the start of cycle c to the start of c+1 */
  int32_t *wl_exec_acc_s_out;            /* [n_wl] final accumulatedPastExecutionTimeSeconds, -1 = nil */
  uint8_t *wl_deactivation_reason;       /* [n_wl] 0 none, 1 Rejected, 2 RequeuingLimitExceeded, 3 MaximumExecutionTimeExceeded,
                                            4 Deactivated by a user (kb_snapshot.ac_*, wl_inactive) */
  /* quota changes (kb_snapshot.n_quota_change > 0; zero / untouched otherwise; each pointer may be NULL) */
  int64_t n_quota_changes;               /* out: edits applied, no-op edits included */
  int32_t *cycle_quota_changes;          /* [max_cycles] edits applied from the start of cycle c to the start of c+1 */
  int64_t *cq_generation;                /* [n_cq] AllocatableResourceGeneration after the drain */
  /* deactivation and reactivation (kb_snapshot.n_active_change > 0 or wl_inactive; zero / untouched otherwise; each
     pointer may be NULL).  wl_deactivated and wl_deactivation_reason (4 = Deactivated by a user) are written with it. */
  int64_t n_stopped;                     /* out: stop edits that deactivated a record, those before cycle 0 included */
  int64_t n_resumed;                     /* out: resume edits that reactivated a record, likewise */
  int32_t *cycle_stopped;                /* [max_cycles] stops from the start of cycle c to the start of c+1 */
  int32_t *cycle_resumed;                /* [max_cycles] resumes, likewise */
} kb_drain_out;
int32_t kb_run_drain(kb_handle *h, const kb_snapshot *s, kb_drain_out *out);

/* ------------------------------------------------------------------------
 * Topology-aware scheduling (SURVEY.md §8 a19): TASFlavorSnapshot.FindTopologyAssignmentsForFlavor
 * (pkg/cache/scheduler/tas_flavor_snapshot.go:485-560) for the podsets that reach
 * findTopologyAssignment (:765-970) with BestFit / LeastFreeCapacity placement: no leader/worker podset groups,
 * no balanced placement (TASBalancedPlacement, off by default), no multi-layer slices, no node replacement,
 * no elastic slices — the shim keeps those on the Go path.
 *
 * One TAS ResourceFlavor = one topology: a forest of domains, `n_levels` levels, every level-(l) domain has one
 * level-(l-1) parent; the leaves are the lowest level.  Domains are numbered level-major (level 0 first); inside a
 * level in ASCENDING lexicographic order of their levelValues (the reference's final tie-break, sortedDomains
 * :1495-1515, and the order of the returned assignment, buildAssignment :1455-1466).
 * ---------------------------------------------------------------------- */
typedef struct kb_tas_topology {
  int32_t n_levels;             /* len(levelKeys)                                                      */
  int32_t n_domains;            /* all domains of all levels                                           */
  int32_t n_resource;           /* resources tracked per leaf, INCLUDING corev1.ResourcePods           */
  int32_t pods_resource;        /* index of corev1.ResourcePods among them                            */
  const int32_t *level_start;   /* [n_levels+1] first domain of every level                            */
  const int32_t *parent;        /* [n_domains] parent domain (previous level) or -1 at level 0         */
  /* leaves = domains [level_start[n_levels-1], n_domains), tables indexed by leaf = domain - first leaf */
  const int64_t *free_capacity; /* [n_leaves][n_resource] leafDomain.freeCapacity (allocatable - non-TAS usage) */
  const uint32_t *cap_mask;     /* [n_leaves] bit r: resource r is a key of freeCapacity (CountIn returns 0 for a
                                   requested resource the node does not expose, requests.go:187-190)  */
  const int64_t *tas_usage;     /* [n_leaves][n_resource] leafDomain.tasUsage (incl. pods)              */
  const uint32_t *usage_mask;   /* [n_leaves] keys of tasUsage                                         */
} kb_tas_topology;

enum { KB_TAS_REQUIRED = 1u << 0,       /* TopologyRequest.Required != nil (isRequired :1107)             */
       KB_TAS_UNCONSTRAINED = 1u << 1,  /* isUnconstrained :1111 (explicit, implied, or slice-only request) */
       KB_TAS_SIMULATE_EMPTY = 1u << 2, /* WithSimulateEmpty: ignore tasUsage (:1583-1585)                 */
       KB_TAS_PROFILE_MIXED = 1u << 3   /* features.TASProfileMixed (default on): LeastFreeCapacity for
                                           unconstrained requests (useLeastFreeCapacityAlgorithm :1291)  */ };
enum { KB_TAS_OK = 0, KB_TAS_NO_FIT = 1, KB_TAS_BAD_REQUEST = 2 };

/* A batch of podset requests against one topology.  Requests with the same chain id are the podsets of one
 * workload: they are placed in input order and every placed podset's usage (SinglePodRequests x count per leaf,
 * addAssumedUsage :619-627) is assumed by the following ones; a failure stops the chain (:551-553).  Different
 * chains are independent (each sees the snapshot's tasUsage only). */
typedef struct kb_tas_requests {
  int32_t n_req;
  const int32_t *chain;          /* [n_req] non-decreasing chain id                                      */
  const int64_t *pod_request;    /* [n_req][n_resource] TASPodSetRequests.SinglePodRequests (WITHOUT pods)  */
  const uint32_t *request_mask;  /* [n_req] keys of SinglePodRequests                                     */
  const int32_t *count;          /* [n_req] TASPodSetRequests.Count                                       */
  const int32_t *slice_size;     /* [n_req] getSliceSizeWithSinglePodAsDefault (:1129-1147), >= 1          */
  const int32_t *level;          /* [n_req] resolved index of the requested topology level (:813-820)     */
  const int32_t *slice_level;    /* [n_req] resolved index of the slice level (>= level, :822-829)        */
  const uint32_t *flags;         /* [n_req] KB_TAS_*                                                      */
  const uint32_t *leaf_ok;       /* [n_req][ceil(n_leaves/32)] or NULL: bit = the leaf passes taints/tolerations,
                                    nodeSelector and required node affinity (fillInCounts :1541-1571, host-evaluated) */
} kb_tas_requests;

typedef struct kb_tas_out {
  int32_t *status;               /* [n_req] KB_TAS_* (requests after a failed one in the same chain: KB_TAS_NO_FIT with no attempt = -1) */
  int32_t *asg_start;            /* [n_req+1] CSR into the assignment arrays                              */
  int32_t *asg_leaf;             /* [capacity] leaf index (ascending = lexicographic levelValues order)    */
  int32_t *asg_count;            /* [capacity] pods on that leaf (TopologyDomainAssignment.Count)          */
  int32_t capacity;
  int32_t n_assigned;            /* out */
} kb_tas_out;

int32_t kb_tas_find(kb_handle *h, const kb_tas_topology *t, const kb_tas_requests *r, kb_tas_out *out);

int32_t kb_get_stats(const kb_handle *h, kb_stats *out);
int32_t kb_set_profile(kb_handle *h, int32_t on);  /* per-kernel event timing on/off */

#ifdef __cplusplus
}
#endif
#endif /* KUEUE_B200_H */
