// kb_device.cuh — device-side view of one flattened snapshot and the quota-tree
// arithmetic shared by the kernels.  sm_90a (H100).
//
// Reference semantics restated per function (paths relative to the kueue repository):
// resourceNode arithmetic = pkg/cache/scheduler/resource_node.go, borrow height =
// pkg/scheduler/preemption/classical/hierarchical_preemption.go:202-227.
#pragma once

#include <cstdint>
#include <cuda_runtime.h>

#include "../../include/kueue_b200.h"

typedef long long i64;
typedef unsigned long long u64;

#define KB_LEVELS (KB_MAX_DEPTH + 2)
#define KB_MAX_CELLS 128  // distinct flavor-resource cells in one workload's usage

// Status word bits written by kernels (checked by the host after a cycle).
enum { KBS_UNSUPPORTED_PREEMPTION = 1u << 0, KBS_TARGET_OVERFLOW = 1u << 1, KBS_PATH_TOO_DEEP = 1u << 2, KBS_INTERNAL_LOOP = 1u << 3,
       KBS_AFS_OVERFLOW = 1u << 4 /* kb_run_drain: an AdmissionFairSharing quantity left int64 */ };

// Static + per-cycle state of one (node, flavor-resource) cell, transposed per root (kb_search.cuh): everything the
// column arithmetic of a target search reads besides the usage itself.  32 B, loaded as two 16 B words.
struct __align__(16) ColStat {
  i64 sub, lq, bl;     // SubtreeQuota, localQuota, BorrowingLimit
  int32_t parent;      // local handle of the parent inside the root's tree, -1 = root
  int16_t depth, height;
};
// One candidate record of a (root, flavor-resource) bucket, in CandidatesOrdering rank order.
struct __align__(16) FrRec {
  int32_t adm, hcq, prio;  // admitted workload, local handle of its ClusterQueue, priority
  uint32_t info;           // bit 0 evicted | depth of the ClusterQueue << 1 | above-nominal mask of its ancestors << 8
  i64 qty;                 // quantity in this flavor-resource
  int32_t tin, cq;         // Euler-tour entry time of the ClusterQueue inside its tree; global ClusterQueue id
};
// Memoised result of one SimulatePreemption call: (cell, quantity) -> (preemption mode, borrow height)
struct SimMemo { i64 val; int pm, borrow; };

struct DevSnap {
  // dimensions
  int Q, C, N, F, R, FR, W, P, A, AU, H, NRG, pods_res;
  uint32_t flags;
  i64 now_ns;
  // ---- inputs (device copies of kb_snapshot tables) ----
  const int32_t *parent;
  const double *fair_weight;
  const i64 *nominal, *blimit, *llimit, *cq_usage;
  const uint8_t *cq_within_cq, *cq_reclaim_within, *cq_borrow_within, *cq_has_bwc_threshold;
  const int32_t *cq_bwc_threshold;
  const uint8_t *cq_when_can_borrow, *cq_when_can_preempt, *cq_preference, *cq_strategy;
  const i64 *cq_generation;
  const int32_t *cq_rg_start;
  const uint32_t *rg_res_mask;
  const int32_t *rg_flavor_start, *rg_flavors;
  const int32_t *wl_cq, *wl_priority;
  const i64 *wl_ts, *wl_uid, *wl_last_gen;
  const int32_t *wl_ps_start;
  const i64 *ps_req;
  const uint32_t *ps_req_mask;
  const int32_t *ps_count, *ps_min_count;
  const u64 *ps_flavor_ok;
  const int8_t *ps_last_tried;
  const int32_t *adm_cq, *adm_priority;
  const i64 *adm_ts, *adm_qr_ts, *adm_uid;
  const uint8_t *adm_evicted;
  const int32_t *adm_use_start, *adm_use_fr;
  const i64 *adm_use_qty;
  const int32_t *heads;
  // Node-table index space.  Normally the node tables (nominal .. potential, parent, height, fs_*) are indexed by
  // the global node id.  The fused per-root kernel (k_cycle_root) passes a copy of this struct whose node tables
  // live in shared memory and are indexed by the LOCAL handle inside the root's tree: tab_local = 1, and every
  // function that takes a global node id maps it with nix().  gparent is always the global parent table.
  int tab_local;
  const int32_t *gparent;
  const i64 *lq;              // localQuota per cell when precomputed (tab_local), else nullptr
  const int32_t *cq_entry;    // [Q] entry (position in heads) of the ClusterQueue's single head, or -1 (k_cycle_root)
  const uint8_t *wl_has_qr;    // optional (nullptr = absent): workload.HasQuotaReservation
  const i64 *wl_sched_hash;    // optional: scheduling equivalence class, 0 = unknown (drain only)
  const int32_t *ps_group;     // optional: PodSetGroup id per podset, -1 = none (members adjacent)
  // ---- relocated per-root view (k_cycle_flat, tab_local == 2): every id (workload, entry, podset row, ClusterQueue,
  // resource group) is LOCAL to one root cohort and all tables above point into shared memory.  These map back.
  const int32_t *ent_gid;      // [entries of the root] global entry index (iterator tie-break), nullptr otherwise
  const int32_t *node_gid;     // [nodes of the root] global node id, nullptr otherwise
  int local_flat;              // tree_flat of the root the local view belongs to
  // static per-tree tables in local numbering (one contiguous block per tree, built by the host at static upload)
  const unsigned char *tree_blob; const int32_t *tree_blob_off;  // [nTrees+1] byte offsets
  const int4 *cq_rec;          // [tree_start[nTrees]] head record per tree node (kb_flat.cuh: cq_rec_write), valid when stamped rec_stamp
  unsigned rec_stamp;
  // quota tables in tree-local row order (row = tree_start[t] + local handle): one root's rows are contiguous, so
  // k_cycle_flat stages each table with ONE bulk copy (cp.async.bulk).  Static ones are built when the static tables
  // are uploaded (k_tl_static / k_tl_root: SubtreeQuota and localQuota, final for every row of a flat tree), the usage
  // by k_flat_prep / k_cq_rec every cycle (zero rows for cohorts).
  const i64 *tl_subtree, *tl_blimit, *tl_lquota; i64 *tl_usage;
  // ---- derived, static per topology (host-built at upload) ----
  const int32_t *root_slot;   // [N] dense index of the node's root among all roots
  const int32_t *depth;       // [N] distance to the root
  const int32_t *height;      // [N] getNodeHeight (cohorts), 0 for CQs
  const int32_t *tree_start;  // [nTrees+1] into tree_nodes (cohort-rooted trees)
  const int32_t *tree_nodes;  // per tree: nodes ordered by depth ascending (root first)
  const int32_t *tree_level;  // [nTrees][KB_LEVELS] start (relative) of each depth level
  const int32_t *local_idx;   // [N] position of the node inside its tree (0 for lone CQs)
  const int32_t *lone_cqs;    // CQs without a cohort
  const int32_t *cq_path;     // [Q][path_stride] node ids from the ClusterQueue up to its root (-1 padded)
  const int32_t *cq_plen;     // [Q] path length
  int path_stride;
  const int32_t *child_start; // [N+1] children CSR: child cohorts ascending, then child CQs ascending
  const int32_t *child_list;
  int32_t *cq_adm_start;      // [Q+1] admitted workloads grouped by CQ (device-built, kb_rank.cuh)
  int32_t *cq_adm;            // [A] in adm_rank order inside every ClusterQueue
  int nTrees, nLone, nRoots;
  int lone_fast;  // cohort-less CQs take the warp-per-root admit kernel (no preemption targets possible, FR <= 64)
  // ---- derived per cycle ----
  i64 *subtree;    // [N][FR] resourceNode.SubtreeQuota
  i64 *usage;      // [N][FR] resourceNode.Usage (mutated by the admit kernel)
  i64 *avail;      // [N][FR] available() at cycle start (may be negative)
  i64 *potential;  // [N][FR] potentialAvailable()
  // entry grouping by root
  int32_t *root_count;   // [nRoots]
  int32_t *root_offset;  // [nRoots+1]
  int32_t *root_cursor;  // [nRoots]
  int32_t *root_entries; // [H]
  int32_t *sorted;       // [H] entries of every root in iterator order (k_rank)
  int32_t *pos_slot;     // [H] root slot of every position of root_entries (k_scatter)
  u64 *ekey;             // [H][4] iterator order key of every entry
  u64 *skey;             // [H][4] the same keys in root-segment order
  i64 *fs_over;          // [Q][R]  sum_f max(0, usage - SubtreeQuota)
  i64 *fs_lend;          // [N][R]  sum_f potentialAvailable
  const uint8_t *tree_flat; // [nTrees] every ClusterQueue of the tree hangs directly off the root cohort
  // ---- outputs (device) ----
  uint8_t *decision, *mode;
  int32_t *borrow, *rank;
  int8_t *ps_flavor, *ps_res_mode, *ps_tried;
  int32_t *ps_count_out;
  uint32_t *status;  // [1] KBS_* bits
  // ---- preemption ----
  int32_t *root_adm_start;       // [nRoots+1] admitted workloads per root (prefix sums)
  int32_t *adm_rank;             // [A] position of the workload among its root's admitted workloads ordered by
                                 //     (evicted desc, priority asc, more recently reserved first, uid) — kb_rank.cuh
  int32_t *root_adm_count, *cq_adm_count;  // [nRoots+1] / [Q+1] histograms of the ranking pass
  const int32_t *root_cq_start;  // [nRoots+1] ClusterQueues per root (segments of over_list)
  int32_t *over_list;            // [Q] per root: ClusterQueues above nominal in some flavor-resource at cycle start (k_over)
  int32_t *over_count;           // [nRoots]
  int32_t *ps_list, *ps_n, *ps_cursor;  // entries deferred to the target search
  int32_t *tgt_off, *tgt_cnt;    // [H] targets of an entry inside the pool
  int32_t *tgt_pool_adm; uint8_t *tgt_pool_reason; int32_t *tgt_pool_used; int tgt_pool_cap;
  uint8_t *preempted;            // [A] PreemptedWorkloads membership (admit loop)
  i64 *usage_shadow;             // [N][FR] usage without the workloads preempted so far (admit loop, see Tab)
  // per-CTA scratch of k_nominate_search
  int32_t *sc_cand, *sc_tgt, *sc_cq_lca, *sc_aux1, *sc_aux2; uint8_t *sc_variant, *sc_tgt_reason; int8_t *sc_cq_class, *sc_on_path;
  i64 *sc_usage;
  uint8_t *sc_dirty; double *sc_drs_ratio; int8_t *sc_drs_meta;  // [G][node cap] DRS cache of the fair search
  int sc_adm_cap, sc_node_cap;
  // per-LANE scratch of the speculative single-cell searches (k_nominate_search phase A)
  int32_t *sl_cand, *sl_tgt, *sl_cq_lca, *sl_aux1; uint8_t *sl_variant, *sl_tgt_reason; int8_t *sl_cq_class, *sl_on_path;
  i64 *sl_col;            // [G*32][node cap] one usage column per lane
  unsigned char *sl_ctx;  // [G*32] PreCtx
  int sl_adm_cap;
  // ---- warp-cooperative classical search (kb_search.cuh) ----
  const int32_t *sn_node;     // [N] slot-node numbering -> global node id (cohort-less ClusterQueues first, then the trees)
  const int32_t *slot_base;   // [nRoots+1] first slot-node of every root
  const int32_t *nd_tin, *nd_tout;  // [N] Euler-tour interval of every slot-node inside its tree
  int32_t *adm_sorted;        // [A] admitted workloads of every root in adm_rank order (segments root_adm_start)
  i64 *colU; ColStat *colS; uint32_t *ovm;  // [N*FR] transposed per root: index = slot_base*FR + fr*nn + h
  int32_t *frl_count, *frl_start;  // [nRoots*FR (+1)] buckets of the fr-lists
  FrRec *frl;                 // [AU]
  FrRec *rrec;                // [A] the roots' ranked lists as packed records (qty field = used flavor-resource bit set)
  SimMemo *memo; int memo_items;  // [memo_items][FR] results of the speculative single-cell searches (item = position in ps_list)
  int32_t *cell_cursor;       // work counter of k_search_cells
  int32_t *cell_count, *cell_start, *cell_fill;  // [nRoots*FR (+1)] oracle cells per (root, flavor-resource) bucket
  int32_t *cell_list, *cell_bucket;              // [memo_items*FR] memo index / bucket of every oracle cell, grouped by bucket
  u64 *sstat;                 // [8] search counters (kb_stats.search_stat)
  i64 *ws_col; size_t ws_col_stride;  // per-warp global column storage when shared memory is too small (stride in i64)
  uint8_t *ws_codes; int32_t *ws_tgt; uint8_t *ws_tgt_reason;  // per-warp [list_cap of the kernel]
  i64 *ws_tgtq; int ws_tgtq_cap;  // per-warp [ws_tgtq_cap] target quantities of single-column searches
  // ---- fair-sharing scratch ----
  i64 *q_scratch;        // [H][FR] dense Assignment.Usage.Quota per entry (absent = -1)
  unsigned char *fs_state; // [H] x (48 + 16*KB_MAX_DEPTH) B: per-entry tournament state when it does not fit shared memory
  int32_t *fs_cq_entry;  // [N] entry of a CQ still waiting in this cycle, or -1
  int32_t *fs_winner;    // [N] tournament winner of a cohort, or -1
};

__device__ __forceinline__ i64 imax(i64 a, i64 b) { return a > b ? a : b; }
__device__ __forceinline__ i64 imin(i64 a, i64 b) { return a < b ? a : b; }

// localQuota resource_node.go:66-71
__device__ __forceinline__ i64 local_quota(i64 subtree, i64 lend_limit) {
  return lend_limit != KB_NO_LIMIT ? imax(0, subtree - lend_limit) : 0;
}

// FindHeightOfLowestSubtreeThatFits hierarchical_preemption.go:214-227, on the
// cycle-start usage.  Returns the borrow height; *may_reclaim = second result.
__device__ __forceinline__ int nix(const DevSnap &D, int node) { return D.tab_local == 1 ? D.local_idx[node] : node; }
__device__ __forceinline__ i64 lq_of(const DevSnap &D, size_t c) { return D.lq ? D.lq[c] : local_quota(D.subtree[c], D.llimit[c]); }
__device__ inline int find_height(const DevSnap &D, const i64 *usage, int cq, int fr, i64 val, bool *may_reclaim) {
  int FR = D.FR;
  int hq = nix(D, cq);
  int p = D.parent[hq];
  size_t c = (size_t)hq * FR + fr;
  i64 ucq = usage[c];
  if (!(ucq + val > D.nominal[c]) || p < 0) { *may_reclaim = p >= 0; return 0; }
  i64 remaining = val - imax(0, lq_of(D, c) - ucq);
  int t = p, last = p;
  while (t >= 0) {
    size_t i = (size_t)t * FR + fr;
    i64 u = usage[i], sub = D.subtree[i];
    if (!(u + remaining > sub)) { *may_reclaim = D.parent[t] >= 0; return D.height[t]; }
    remaining -= imax(0, lq_of(D, i) - u);
    last = t;
    t = D.parent[t];
  }
  *may_reclaim = false;
  return D.height[last];
}

// DominantResourceShare value (fair_sharing.go:43-100)
struct DevDRS {
  double weight, ratio;
  int res;
  bool borrowing;
};
__device__ __forceinline__ bool drs_zero_weight_borrows(const DevDRS &d) { return d.weight == 0 && d.ratio != 0; }
__device__ __forceinline__ double drs_precise(const DevDRS &d) {  // :75-83
  if (d.ratio == 0) return 0.0;
  if (d.weight == 0) return __longlong_as_double(0x7ff0000000000000LL);
  return d.ratio / d.weight;
}
__device__ __forceinline__ int cmp_d(double a, double b) { return a < b ? -1 : (a > b ? 1 : 0); }
__device__ inline int drs_compare(const DevDRS &a, const DevDRS &b) {  // CompareDRS :89-100
  bool za = drs_zero_weight_borrows(a), zb = drs_zero_weight_borrows(b);
  if (za && zb) return cmp_d(a.ratio, b.ratio);
  if (za) return 1;
  if (zb) return -1;
  return cmp_d(drs_precise(a), drs_precise(b));
}
