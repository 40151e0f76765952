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
#define KB_MAX_DEPTH     16   /* CQ -> root path length <= 16 */
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
   * CUDA events recorded on the launching stream around each kernel. */
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
 * Evictions are asynchronous in the reference and are not replayed: the targets of a Preempting entry stay admitted.
 * Cycle c runs with now_ns + c.  Bit-exact with iterating kb_run_cycle under the same rules (kueue_b200/drain.py). */
typedef struct kb_drain_out {
  int32_t max_cycles;        /* in */
  int32_t n_cycles;          /* out: cycles run */
  int64_t n_decisions;       /* out: entries evaluated over all cycles */
  int64_t n_admitted;        /* out */
  int32_t *cycle_heads;      /* [max_cycles] entries per cycle (may be NULL) */
  int32_t *cycle_admitted;   /* [max_cycles] admissions per cycle (may be NULL) */
  /* per pending workload [n_wl] (each may be NULL) */
  int32_t *wl_admit_cycle;   /* cycle that admitted it, -1 = still pending */
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
