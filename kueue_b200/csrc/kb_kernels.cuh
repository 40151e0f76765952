// kb_kernels.cuh — sm_90a (H100) kernels of the scheduling cycle.
//
//   K1  k_tree / k_lone   resource-node tree: SubtreeQuota, cohort Usage (bottom-up,
//                         resource_node.go:183-217), available / potentialAvailable
//                         (top-down, :104-133) for every (node, flavor-resource) cell.
//   K1d k_drs             dominantResourceShare per node (fair_sharing.go:126-174).
//   K2  k_nominate        flavorassigner.Assign for every entry of the cycle
//                         (flavorassigner.go:540-1047), one thread per workload,
//                         coalesced reads of the podset request rows.
//   K3  k_scan / k_scatter group entries by root cohort.
//   K5  k_admit           per-root ordered admit loop (scheduler.go:269-401,778-817):
//                         block-local bitonic sort of the root's entries, then one warp
//                         commits them in order with one lane per flavor-resource cell.
//
// All of it is integer compare/add work bounded by HBM/L2 bandwidth and latency:
// no tensor cores.
#pragma once

#include "kb_device.cuh"
#include "kb_preempt.cuh"
#include "kb_search.cuh"
#include "kb_rank.cuh"
#include "kb_drain.cuh"
#include "kb_tas.cuh"

#define KB_RANK_CAP 2048  // roots up to this many entries are ordered by the all-pairs k_rank kernel

// ---------------------------------------------------------------------------
// K1: tree pass, one CTA per cohort-rooted tree.
// ---------------------------------------------------------------------------
__global__ void __launch_bounds__(1024) k_tree(DevSnap D) {
  int t = blockIdx.x;
  int FR = D.FR;
  const int32_t *nodes = D.tree_nodes + D.tree_start[t];
  int nn = D.tree_start[t + 1] - D.tree_start[t];
  const int32_t *lvl = D.tree_level + (size_t)t * KB_LEVELS;
  int nlev = 0;
  while (nlev + 1 < KB_LEVELS && lvl[nlev + 1] > lvl[nlev]) nlev++;  // levels [0, nlev)
  // init: SubtreeQuota = Nominal; Usage = CQ usage | 0 (updateCohortResourceNode :184-190)
  for (int i = threadIdx.x; i < nn * FR; i += blockDim.x) {
    int n = nodes[i / FR], fr = i % FR;
    size_t c = (size_t)n * FR + fr;
    D.subtree[c] = D.nominal[c];
    D.usage[c] = n < D.Q ? D.cq_usage[c] : 0;
  }
  __syncthreads();
  // bottom-up accumulateFromChild :210-217
  for (int L = nlev - 1; L >= 1; L--) {
    int a = lvl[L], b = lvl[L + 1];
    for (int i = threadIdx.x; i < (b - a) * FR; i += blockDim.x) {
      int n = nodes[a + i / FR], fr = i % FR;
      size_t c = (size_t)n * FR + fr;
      size_t pc = (size_t)D.parent[n] * FR + fr;
      i64 sub = D.subtree[c];
      i64 lq = local_quota(sub, D.llimit[c]);
      atomicAdd((u64 *)&D.subtree[pc], (u64)(sub - lq));
      i64 spill = imax(0, D.usage[c] - lq);
      if (spill) atomicAdd((u64 *)&D.usage[pc], (u64)spill);
    }
    __syncthreads();
  }
  // top-down available / potentialAvailable :104-133
  for (int L = 0; L < nlev; L++) {
    int a = lvl[L], b = lvl[L + 1];
    for (int i = threadIdx.x; i < (b - a) * FR; i += blockDim.x) {
      int n = nodes[a + i / FR], fr = i % FR;
      size_t c = (size_t)n * FR + fr;
      i64 sub = D.subtree[c], u = D.usage[c];
      if (L == 0) {
        D.avail[c] = sub - u;
        D.potential[c] = sub;
      } else {
        size_t pc = (size_t)D.parent[n] * FR + fr;
        i64 lq = local_quota(sub, D.llimit[c]);
        i64 bl = D.blimit[c];
        i64 pa = D.avail[pc];
        i64 pot = lq + D.potential[pc];
        if (bl != KB_NO_LIMIT) {
          i64 stored = sub - lq, used = imax(0, u - lq);
          pa = imin(stored - used + bl, pa);
          pot = imin(sub + bl, pot);
        }
        D.avail[c] = imax(0, lq - u) + pa;
        D.potential[c] = pot;
      }
    }
    __syncthreads();
  }
}

// ClusterQueues without a cohort: the node is its own root.
__global__ void k_lone(DevSnap D) {
  int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= D.nLone * D.FR) return;
  int n = D.lone_cqs[i / D.FR], fr = i % D.FR;
  size_t c = (size_t)n * D.FR + fr;
  i64 nom = D.nominal[c], u = D.cq_usage[c];
  D.subtree[c] = nom;
  D.usage[c] = u;
  D.avail[c] = nom - u;
  D.potential[c] = nom;
}

// ---------------------------------------------------------------------------
// K1d: DominantResourceShare of every node (fair_sharing.go:126-156, wlReq = nil).
// ---------------------------------------------------------------------------
// DRS of node n when its usage row is `u[fr] + extra[fr]` (extra may be null).
template <typename UsageFn>
__device__ inline DevDRS drs_node(const DevSnap &D, int n, UsageFn usage_of) {
  DevDRS d{D.fair_weight[n], 0.0, -1, false};
  int p = D.parent[n];
  if (p < 0) return d;
  int R = D.R, F = D.F, FR = D.FR;
  for (int r = 0; r < R; r++) {
    i64 b = 0, lend = 0;
    for (int f = 0; f < F; f++) {
      int fr = f * R + r;
      i64 over = usage_of(fr) - D.subtree[(size_t)n * FR + fr];
      if (over > 0) b += over;
      lend += D.potential[(size_t)p * FR + fr];  // calculateLendable :160-174
    }
    if (b > 0) {
      d.borrowing = true;
      if (lend > 0) {
        double ratio = (double)b * 1000.0 / (double)lend;
        if (ratio > d.ratio) { d.ratio = ratio; d.res = r; }  // ascending r => smaller name wins ties
      }
    }
  }
  return d;
}
__global__ void k_drs(DevSnap D, i64 *drs_rounded, int32_t *drs_res, uint8_t *drs_borrowing) {
  int n = blockIdx.x * blockDim.x + threadIdx.x;
  if (n >= D.N) return;
  const i64 *u = D.usage + (size_t)n * D.FR;
  DevDRS d = drs_node(D, n, [&](int fr) { return u[fr]; });
  i64 v;
  if (drs_zero_weight_borrows(d)) v = INT64_MAX;  // roundedWeightedShare :110-118
  else v = (i64)ceil(drs_precise(d));
  drs_rounded[n] = v;
  drs_res[n] = d.res;
  drs_borrowing[n] = d.borrowing;
}

// ---------------------------------------------------------------------------
// K2: nominate.  preemptionMode values flavorassigner.go:399-407
// ---------------------------------------------------------------------------
enum { PM_NOFIT = 0, PM_NOCAND = 1, PM_PREEMPT = 2, PM_RECLAIM = 3, PM_FIT = 4 };

__device__ __forceinline__ bool gm_preferred(int apm, int ab, int bpm, int bb, int pref) {  // isPreferred :410-441
  if (apm == PM_NOFIT) return false;
  if (bpm == PM_NOFIT) return true;
  if (pref == KB_PREF_PREEMPTION_OVER_BORROWING) {
    if (ab != bb) return ab < bb;
    return apm > bpm;
  }
  if (apm != bpm) return apm > bpm;
  return ab < bb;
}
__device__ __forceinline__ int fa_mode(int pm) {  // flavorAssignmentMode :470-485
  return pm == PM_NOFIT ? KB_MODE_NOFIT : (pm == PM_FIT ? KB_MODE_FIT : KB_MODE_PREEMPT);
}
// One step of findFlavorForPodSets' ordered flavor walk: does the next flavor, with representative mode rpm and borrow
// height rb over its resources, replace the best one so far, and does the walk stop there (*done)?  With fungibility
// the walk stops at the first flavor whenCanBorrow / whenCanPreempt accept and otherwise keeps the preferred one
// (isPreferred); without it the flavor with the better mode wins and a Fit stops the walk.
__device__ __forceinline__ bool flavor_take(bool fung, int wcb, int wcp, int pref, int rpm, int rb, int best_pm, int best_rb, bool *done) {
  if (fung) {
    const bool try_next = rpm == PM_NOFIT || rpm == PM_NOCAND || ((rpm == PM_PREEMPT || rpm == PM_RECLAIM) && wcp == KB_FUNG_TRY_NEXT_FLAVOR) ||
                          (rb != 0 && wcb == KB_FUNG_TRY_NEXT_FLAVOR);
    if (!try_next) { *done = true; return true; }
    return gm_preferred(rpm, rb, best_pm, best_rb, pref);
  }
  if (rpm > best_pm) { *done = rpm == PM_FIT; return true; }
  return false;
}
__device__ __forceinline__ int rg_by_resource(const DevSnap &D, int cq, int r) {  // RGByResource clusterqueue_snapshot.go:67-74
  for (int g = D.cq_rg_start[cq]; g < D.cq_rg_start[cq + 1]; g++)
    if (D.rg_res_mask[g] & (1u << r)) return g;
  return -1;
}
// Effective request of podset `row` for resource r with `count` pods admitted
// (ScaledTo workload.go:258-275; pods resource flavorassigner.go:585-587).
__device__ __forceinline__ i64 ps_request(const DevSnap &D, int row, int r, int count, bool covers_pods) {
  if (covers_pods && r == D.pods_res) return count;
  i64 q = D.ps_req[(size_t)row * D.R + r];
  int full = D.ps_count[row];
  if (full != 0 && full != count) q = q / full * count;
  return q;
}

// Can a preemption candidate exist at all for workloads of this CQ?  (own CQ: policy
// WithinClusterQueue != Never and the CQ has admitted workloads; cohort: ReclaimWithinCohort
// != Never and another CQ of the root has admitted workloads.)  When not, getTargets returns
// nil and SimulatePreemption returns NoCandidates without any search.
__device__ __forceinline__ bool candidates_possible(const DevSnap &D, int cq) {
  if (D.tab_local == 2) return false;  // the relocated view only exists for cycles in which no ClusterQueue can have candidates
  int own_n = D.cq_adm_start[cq + 1] - D.cq_adm_start[cq];
  if (D.cq_within_cq[cq] != KB_POLICY_NEVER && own_n > 0) return true;
  if (D.gparent[cq] >= 0 && D.cq_reclaim_within[cq] != KB_POLICY_NEVER) {
    int slot = D.root_slot[cq];
    if (D.root_adm_start[slot + 1] - D.root_adm_start[slot] - own_n > 0) return true;
  }
  return false;
}

// Oracle policy of the thread-per-entry nominate pass: everything that needs a target
// search is deferred to k_nominate_search (the entry is re-evaluated there).
struct NomThread {
  bool need_search = false;
  __device__ __forceinline__ int simulate(const DevSnap &D, int wl, int cq, int fr, i64 val, int *borrow_after) {
    if (candidates_possible(D, cq)) need_search = true;
    bool may_reclaim;
    *borrow_after = find_height(D, D.usage, cq, fr, val, &may_reclaim);
    return PM_NOCAND;  // preemption_oracle.go:52-56 when there are no candidates: height on the untouched snapshot
  }
  __device__ __forceinline__ int get_targets(const DevSnap &D, int wl) {
    if (candidates_possible(D, D.wl_cq[wl])) need_search = true;
    return 0;
  }
};

// fitsResourceQuota :1017-1047
template <typename Oracle>
__device__ inline int fits_resource_quota(const DevSnap &D, Oracle &orc, int wl, int cq, int fr, i64 assumed, i64 request, int *borrow) {
  size_t c = (size_t)nix(D, cq) * D.FR + fr;
  i64 avail = imax(0, D.avail[c]);
  i64 val = assumed + request;
  if (val > D.potential[c]) { *borrow = 0; return PM_NOFIT; }
  bool may_reclaim;
  int b = find_height(D, D.usage, cq, fr, val, &may_reclaim);
  if (val <= avail) { *borrow = b; return PM_FIT; }
  bool can_pwb = D.cq_borrow_within[cq] != KB_POLICY_NEVER ||
                 ((D.flags & KB_F_FAIR_SHARING) && D.cq_reclaim_within[cq] != KB_POLICY_NEVER);  // :1049-1052
  if (val <= D.nominal[c] || may_reclaim || can_pwb) return orc.simulate(D, wl, cq, fr, val, borrow);
  *borrow = b;
  return PM_NOFIT;
}

// One workload: Assign + assignFlavors (:540-715) writing PodSetAssignment rows.
// counts == nullptr => full counts.  Returns the representative mode; *borrowing_out =
// Assignment.Borrowing.
template <typename Oracle>
__device__ inline int assign_workload(const DevSnap &D, Oracle &orc, int wl, const int32_t *counts, int *borrowing_out) {
  const int R = D.R;
  int cq = D.wl_cq[wl];
  int ps0 = D.wl_ps_start[wl], ps1 = D.wl_ps_start[wl + 1];
  i64 lg = D.wl_last_gen[wl];
  bool use_last = lg >= 0 && !(D.cq_generation[cq] > lg);  // lastAssignmentOutdated :532-534
  bool fung = D.flags & KB_F_FLAVOR_FUNGIBILITY;
  bool covers_pods = D.pods_res >= 0 && rg_by_resource(D, cq, D.pods_res) >= 0;
  int pref = D.cq_preference[cq];
  int wcb = D.cq_when_can_borrow[cq], wcp = D.cq_when_can_preempt[cq];
  int borrowing = 0, rep = KB_MODE_FIT;
  if (ps1 == ps0) rep = KB_MODE_NOFIT;  // RepresentativeMode :148-151
  bool stop = false;
  // A unit is one podset, or the run of consecutive podsets that share a PodSetGroupName (groupedRequests :613-623):
  // the group's requests are summed, one flavor search serves all of them, each member keeps the flavors of the
  // resources it requests.
  int row_end;
  for (int row = ps0; row < ps1; row = row_end) {
    row_end = row + 1;
    if (D.ps_group && D.ps_group[row] >= 0) while (row_end < ps1 && D.ps_group[row_end] == D.ps_group[row]) row_end++;
    auto cnt_of = [&](int m) { int full = D.ps_count[m]; return (counts && full != 0) ? counts[m - ps0] : full; };
    uint32_t mask = 0;
    u64 ok = ~0ull;
    for (int m = row; m < row_end; m++) {
      int8_t *fl = D.ps_flavor + (size_t)m * R, *md = D.ps_res_mode + (size_t)m * R, *tr = D.ps_tried + (size_t)m * R;
      for (int r = 0; r < R; r++) { fl[r] = -1; md[r] = -1; tr[r] = -1; }
      D.ps_count_out[m] = stop ? D.ps_count[m] : cnt_of(m);
      mask |= D.ps_req_mask[m];
      ok &= D.ps_flavor_ok[m];  // checkFlavorForPodSets walks every podset of the group :915-941
    }
    if (stop) continue;
    if (covers_pods) mask |= 1u << D.pods_res;
    auto unit_request = [&](int r) {  // requests.Add(podset.podSet.Requests) :627-631
      i64 q = 0;
      for (int m = row; m < row_end; m++) q += ps_request(D, m, r, cnt_of(m), covers_pods);
      return q;
    };
    bool has_reasons = false, failed = false;
    int ps_borrow = 0;
    uint32_t assigned = 0;
    for (int r0 = 0; r0 < R; r0++) {  // :639-661
      if (!(mask & (1u << r0))) continue;
      if (assigned & (1u << r0)) continue;  // got the flavor of its resource group already
      int g = rg_by_resource(D, cq, r0);
      if (g < 0) {
        if (unit_request(r0) == 0) continue;  // zero request for an undefined resource
        has_reasons = true; failed = true; break;  // :770-772
      }
      // findFlavorForPodSets :762-897
      uint32_t rgm = D.rg_res_mask[g] & mask;
      int fl0 = D.rg_flavor_start[g], nfl = D.rg_flavor_start[g + 1] - fl0;
      int best_f = -1, best_pm = PM_NOFIT, best_rb = INT32_MAX, best_maxb = 0;
      uint32_t best_pmask = 0;  // resources whose FlavorAssignment.Mode is Preempt in the best flavor
      bool any_reason = false;
      int attempted = -1;
      int idx = 0;
      if (fung && use_last) idx = D.ps_last_tried[(size_t)row * R + r0] + 1;  // NextFlavorToTryForPodSetResource(psIDs[0], ...)
      for (; idx < nfl; idx++) {
        attempted = idx;
        int f = D.rg_flavors[fl0 + idx];
        if (!((ok >> f) & 1)) { any_reason = true; continue; }  // checkFlavorForPodSets :798-806
        int rpm = PM_FIT, rb = 0, maxb = 0;
        uint32_t pmask = 0;
        for (int r = 0; r < R; r++) {
          if (!(rgm & (1u << r))) continue;
          // quota assumed by the previous podsets of this workload on (f, r): assignmentUsage[fr] :839
          i64 assumed = 0;
          for (int prow = ps0; prow < row; prow++)
            if (D.ps_flavor[(size_t)prow * R + r] == f) assumed += ps_request(D, prow, r, D.ps_count_out[prow], covers_pods);
          int b;
          int pm = fits_resource_quota(D, orc, wl, cq, f * R + r, assumed, unit_request(r), &b);
          if (pm != PM_FIT) any_reason = true;
          if (gm_preferred(rpm, rb, pm, b, pref)) { rpm = pm; rb = b; }  // :846-848 keep the worst
          if (rpm == PM_NOFIT) break;                                    // :849-852
          if (fa_mode(pm) == KB_MODE_PREEMPT) pmask |= 1u << r;
          if (b > maxb) maxb = b;
        }
        bool take = false, done = false;
        if (fung) {  // :863-872
          bool try_next = rpm == PM_NOFIT || rpm == PM_NOCAND ||
                          ((rpm == PM_PREEMPT || rpm == PM_RECLAIM) && wcp == KB_FUNG_TRY_NEXT_FLAVOR) ||
                          (rb != 0 && wcb == KB_FUNG_TRY_NEXT_FLAVOR);  // shouldTryNextFlavor :946-963
          if (!try_next) { take = true; done = true; }
          else if (gm_preferred(rpm, rb, best_pm, best_rb, pref)) take = true;
        } else if (rpm > best_pm) {  // :873-880
          take = true;
          done = rpm == PM_FIT;
        }
        if (take) { best_f = f; best_pm = rpm; best_rb = rb; best_maxb = maxb; best_pmask = pmask; }
        if (done) break;
      }
      if (best_f < 0) { has_reasons = true; failed = true; break; }  // :652-656
      int tried = fung ? (attempted == nfl - 1 ? -1 : attempted) : 0;  // :883-891
      for (int m = row; m < row_end; m++) {  // FilterKeys(groupFlavors, keys(podSet.Requests)) :666
        uint32_t mm = (D.ps_req_mask[m] | (covers_pods ? 1u << D.pods_res : 0u)) & rgm;
        for (int r = 0; r < R; r++) {
          if (!(mm & (1u << r))) continue;
          D.ps_flavor[(size_t)m * R + r] = (int8_t)best_f;
          D.ps_res_mode[(size_t)m * R + r] = (best_pmask >> r) & 1 ? KB_MODE_PREEMPT : KB_MODE_FIT;
          D.ps_tried[(size_t)m * R + r] = (int8_t)tried;
        }
      }
      assigned |= rgm;
      if (best_maxb > ps_borrow) ps_borrow = best_maxb;
      if (best_pm != PM_FIT && any_reason) has_reasons = true;  // status is nil when the best mode is fit :892-894
    }
    if (failed) {
      for (int m = row; m < row_end; m++)
        for (int r = 0; r < R; r++) { D.ps_flavor[(size_t)m * R + r] = -1; D.ps_res_mode[(size_t)m * R + r] = -1; D.ps_tried[(size_t)m * R + r] = -1; }
      rep = KB_MODE_NOFIT;
      stop = true;  // :677-679 return assignment
    } else {
      if (ps_borrow > borrowing) borrowing = ps_borrow;  // Assignment.append :721-723
      for (int m = row; m < row_end; m++) {
        int psmode = KB_MODE_FIT;  // PodSetAssignment.RepresentativeMode :277-295
        if (has_reasons) {
          const int8_t *fl = D.ps_flavor + (size_t)m * R, *md = D.ps_res_mode + (size_t)m * R;
          int nfl_assigned = 0;
          for (int r = 0; r < R; r++) if (fl[r] >= 0) { nfl_assigned++; if (md[r] < psmode) psmode = md[r]; }
          if (nfl_assigned == 0) psmode = KB_MODE_NOFIT;
        }
        if (psmode < rep) rep = psmode;
      }
    }
  }
  *borrowing_out = borrowing;
  return rep;
}

#define KB_MAX_PODSETS 16

// getInitialAssignments scheduler.go:584-625 incl. PodSetReducer.Search podset_reducer.go:56-86.
// Leaves the final PodSetAssignment rows in the output tables; returns the representative
// mode, *borrowing_out = Assignment.Borrowing, *ntargets = len(preemptionTargets).
template <typename Oracle>
__device__ inline int get_assignments(const DevSnap &D, Oracle &orc, int wl, int *borrowing_out, int *ntargets) {
  *ntargets = 0;
  int mode = assign_workload(D, orc, wl, nullptr, borrowing_out);
  if (mode == KB_MODE_FIT) return mode;
  if (mode == KB_MODE_PREEMPT) {
    int nt = orc.get_targets(D, wl);
    if (nt > 0) { *ntargets = nt; return mode; }
  }
  if (!(D.flags & KB_F_PARTIAL_ADMISSION)) return mode;
  int ps0 = D.wl_ps_start[wl], np = D.wl_ps_start[wl + 1] - ps0;
  if (np > KB_MAX_PODSETS) return mode;
  int total = 0; bool can = false;  // CanBePartiallyAdmitted workload.go:514-522; deltas podset_reducer.go:47-53
  for (int i = 0; i < np; i++) {
    int mc = D.ps_min_count[ps0 + i], full = D.ps_count[ps0 + i];
    if (mc >= 0) { total += full - mc; if (full > mc) can = true; }
  }
  if (!can || total == 0) return mode;
  int32_t counts[KB_MAX_PODSETS];
  auto fill = [&](int i) {  // fillPodSetSizesForSearchIndex :56-62
    for (int k = 0; k < np; k++) {
      int mc = D.ps_min_count[ps0 + k], full = D.ps_count[ps0 + k];
      int delta = mc >= 0 ? full - mc : 0;
      counts[k] = full - (int32_t)((i64)delta * i / total);
    }
  };
  int last_good = -1, lo = 0, hi = total + 1;
  while (lo < hi) {  // sort.Search(total+1, fits)
    int mid = lo + (hi - lo) / 2;
    fill(mid);
    int b;
    int m = assign_workload(D, orc, wl, counts, &b);
    bool good = m == KB_MODE_FIT;
    if (!good && m == KB_MODE_PREEMPT) good = orc.get_targets(D, wl) > 0;
    if (good) { last_good = mid; hi = mid; } else lo = mid + 1;
  }
  if (last_good >= 0 && lo == last_good) {
    fill(last_good);
    mode = assign_workload(D, orc, wl, counts, borrowing_out);
    if (mode == KB_MODE_PREEMPT) *ntargets = orc.get_targets(D, wl);
    return mode;
  }
  mode = assign_workload(D, orc, wl, nullptr, borrowing_out);  // :624 return fullAssignment, nil
  return mode;
}

// ---------------------------------------------------------------------------
// K2 (cooperative form): KB_NG lanes per entry.  Every lane runs the same (scalar) flavor
// assignment control flow on register state; the flavors of a resource group are evaluated
// one per lane (each lane walks the resources of "its" flavor), and a short ordered scan with
// shuffles applies the selection rules of findFlavorForPodSets (:794-897) exactly as the
// sequential loop would.  This cuts the dependent-load chain of one entry by ~KB_NG and keeps
// the lanes of a warp converged.  Lane 0 of the group is the single writer of the output rows.
// Cells that would need the preemption oracle are only *flagged* (when the scan reaches them):
// the entry is then re-evaluated by k_nominate_search, like in the thread-per-entry kernel.
// ---------------------------------------------------------------------------
#define KB_NG 8
enum { PM_NEED = 5 };

// fitsResourceQuota :1017-1047 for a quantity val <= potentialAvailable: Fit within available, else PM_NEED where
// SimulatePreemption would run (within nominal, the lowest fitting subtree is below the root, or preemption while
// borrowing is allowed: can_pwb(), asked only then), else NoFit.
template <typename PwbFn>
__device__ __forceinline__ int fits_mode(i64 val, i64 avail, i64 nominal, bool may_reclaim, PwbFn can_pwb) {
  if (val <= imax(0, avail)) return PM_FIT;
  return (val <= nominal || may_reclaim || can_pwb()) ? PM_NEED : PM_NOFIT;
}
// fitsResourceQuota without the oracle call: PM_NEED where SimulatePreemption would run.
__device__ __forceinline__ int cell_eval(const DevSnap &D, int cq, int fr, i64 assumed, i64 request, int *borrow) {
  size_t c = (size_t)nix(D, cq) * D.FR + fr;
  i64 val = assumed + request;
  if (val > D.potential[c]) { *borrow = 0; return PM_NOFIT; }
  bool may_reclaim;
  *borrow = find_height(D, D.usage, cq, fr, val, &may_reclaim);
  return fits_mode(val, D.avail[c], D.nominal[c], may_reclaim, [&] {
    return D.cq_borrow_within[cq] != KB_POLICY_NEVER || ((D.flags & KB_F_FAIR_SHARING) && D.cq_reclaim_within[cq] != KB_POLICY_NEVER);
  });
}

template <int NG = KB_NG>  // lanes per entry (a power of two <= 32): NG flavors of a resource group are evaluated per round
__device__ inline int assign_workload_coop(const DevSnap &D, bool *need_search, int wl, const int32_t *counts, int *borrowing_out,
                                           unsigned gmask, int gbase, int glane) {
  const int R = D.R;
  int cq = D.wl_cq[wl];
  int ps0 = D.wl_ps_start[wl], ps1 = D.wl_ps_start[wl + 1];
  i64 lg = D.wl_last_gen[wl];
  bool use_last = lg >= 0 && !(D.cq_generation[cq] > lg);
  bool fung = D.flags & KB_F_FLAVOR_FUNGIBILITY;
  bool covers_pods = D.pods_res >= 0 && rg_by_resource(D, cq, D.pods_res) >= 0;
  int pref = D.cq_preference[cq];
  int wcb = D.cq_when_can_borrow[cq], wcp = D.cq_when_can_preempt[cq];
  bool cand_possible = candidates_possible(D, cq);
  int borrowing = 0, rep = KB_MODE_FIT;
  if (ps1 == ps0) rep = KB_MODE_NOFIT;
  bool stop = false;
  int row_end;
  for (int row = ps0; row < ps1; row = row_end) {  // units as in assign_workload: a podset or a run of one PodSetGroup
    row_end = row + 1;
    if (D.ps_group && D.ps_group[row] >= 0) while (row_end < ps1 && D.ps_group[row_end] == D.ps_group[row]) row_end++;
    auto cnt_of = [&](int m) { int full = D.ps_count[m]; return (counts && full != 0) ? counts[m - ps0] : full; };
    uint32_t mask = 0;
    u64 ok = ~0ull;
    for (int m = row; m < row_end; m++) {
      if (glane == 0) {
        int8_t *fl = D.ps_flavor + (size_t)m * R, *md = D.ps_res_mode + (size_t)m * R, *tr = D.ps_tried + (size_t)m * R;
        for (int r = 0; r < R; r++) { fl[r] = -1; md[r] = -1; tr[r] = -1; }
        D.ps_count_out[m] = stop ? D.ps_count[m] : cnt_of(m);
      }
      mask |= D.ps_req_mask[m];
      ok &= D.ps_flavor_ok[m];
    }
    if (stop) continue;
    if (covers_pods) mask |= 1u << D.pods_res;
    auto unit_request = [&](int r) {
      i64 q = 0;
      for (int m = row; m < row_end; m++) q += ps_request(D, m, r, cnt_of(m), covers_pods);
      return q;
    };
    bool has_reasons = false, failed = false;
    int ps_borrow = 0;
    uint32_t assigned = 0, ps_pmask = 0;  // resources with a flavor / with Mode == Preempt in this unit
    for (int r0 = 0; r0 < R; r0++) {
      if (!(mask & (1u << r0))) continue;
      if (assigned & (1u << r0)) continue;
      int g = rg_by_resource(D, cq, r0);
      if (g < 0) {
        if (unit_request(r0) == 0) continue;
        has_reasons = true; failed = true; break;
      }
      uint32_t rgm = D.rg_res_mask[g] & mask;
      int fl0 = D.rg_flavor_start[g], nfl = D.rg_flavor_start[g + 1] - fl0;
      int best_f = -1, best_pm = PM_NOFIT, best_rb = INT32_MAX, best_maxb = 0;
      uint32_t best_pmask = 0;
      bool any_reason = false;
      int attempted = -1;
      int idx0 = 0;
      if (fung && use_last) idx0 = D.ps_last_tried[(size_t)row * R + r0] + 1;
      bool done = false;
      for (int base = idx0; base < nfl && !done; base += NG) {
        // ---- one flavor per lane ----
        int idx = base + glane;
        u64 res = 0;  // [0..2] rpm [3..9] rb [10..16] maxb [17] any_reason [18] need [19] eligible [32..47] pmask
        int myf = -1;
        if (idx < nfl) {
          int f = D.rg_flavors[fl0 + idx];
          myf = f;
          if ((ok >> f) & 1) {
            int rpm = PM_FIT, rb = 0, maxb = 0; uint32_t pmask = 0; bool reason = false, need = false;
            for (int r = 0; r < R; r++) {
              if (!(rgm & (1u << r))) continue;
              i64 assumed = 0;
              for (int prow = ps0; prow < row; prow++)
                if (D.ps_flavor[(size_t)prow * R + r] == f) assumed += ps_request(D, prow, r, D.ps_count_out[prow], covers_pods);
              int b;
              int pm = cell_eval(D, cq, f * R + r, assumed, unit_request(r), &b);
              if (pm == PM_NEED) { pm = PM_NOCAND; need = need || cand_possible; }  // what the deferring oracle returns (b = height on the untouched snapshot)
              if (pm != PM_FIT) reason = true;
              if (gm_preferred(rpm, rb, pm, b, pref)) { rpm = pm; rb = b; }
              if (rpm == PM_NOFIT) break;
              if (fa_mode(pm) == KB_MODE_PREEMPT) pmask |= 1u << r;
              if (b > maxb) maxb = b;
            }
            res = (u64)rpm | ((u64)(rb & 127) << 3) | ((u64)(maxb & 127) << 10) | ((u64)reason << 17) | ((u64)need << 18) | (1ull << 19) |
                  ((u64)pmask << 32);
          }
        }
        // ---- ordered scan over the KB_NG flavors of this round ----
        for (int j = 0; j < NG && base + j < nfl; j++) {
          u64 rj = __shfl_sync(gmask, res, gbase + j);
          int fj = __shfl_sync(gmask, myf, gbase + j);
          attempted = base + j;
          if (!((rj >> 19) & 1)) { any_reason = true; continue; }  // checkFlavorForPodSets failed
          int rpm = (int)(rj & 7), rb = (int)((rj >> 3) & 127), maxb = (int)((rj >> 10) & 127);
          uint32_t pmask = (uint32_t)(rj >> 32) & 0xffffu;
          if ((rj >> 17) & 1) any_reason = true;
          if ((rj >> 18) & 1) *need_search = true;  // the sequential walk would have called SimulatePreemption here
          if (flavor_take(fung, wcb, wcp, pref, rpm, rb, best_pm, best_rb, &done)) { best_f = fj; best_pm = rpm; best_rb = rb; best_maxb = maxb; best_pmask = pmask; }
          if (done) break;
        }
      }
      if (best_f < 0) { has_reasons = true; failed = true; break; }
      int tried = fung ? (attempted == nfl - 1 ? -1 : attempted) : 0;
      if (glane == 0)
        for (int m = row; m < row_end; m++) {
          uint32_t mm = (D.ps_req_mask[m] | (covers_pods ? 1u << D.pods_res : 0u)) & rgm;
          for (int r = 0; r < R; r++) {
            if (!(mm & (1u << r))) continue;
            D.ps_flavor[(size_t)m * R + r] = (int8_t)best_f;
            D.ps_res_mode[(size_t)m * R + r] = (best_pmask >> r) & 1 ? KB_MODE_PREEMPT : KB_MODE_FIT;
            D.ps_tried[(size_t)m * R + r] = (int8_t)tried;
          }
        }
      assigned |= rgm;
      ps_pmask |= best_pmask & rgm;
      if (best_maxb > ps_borrow) ps_borrow = best_maxb;
      if (best_pm != PM_FIT && any_reason) has_reasons = true;
    }
    if (failed) {
      if (glane == 0)
        for (int m = row; m < row_end; m++)
          for (int r = 0; r < R; r++) { D.ps_flavor[(size_t)m * R + r] = -1; D.ps_res_mode[(size_t)m * R + r] = -1; D.ps_tried[(size_t)m * R + r] = -1; }
      rep = KB_MODE_NOFIT;
      stop = true;
    } else {
      if (ps_borrow > borrowing) borrowing = ps_borrow;
      for (int m = row; m < row_end; m++) {
        int psmode = KB_MODE_FIT;
        if (has_reasons) {
          uint32_t mm = D.ps_req_mask[m] | (covers_pods ? 1u << D.pods_res : 0u);
          if ((assigned & mm) == 0) psmode = KB_MODE_NOFIT;
          else if (ps_pmask & mm) psmode = KB_MODE_PREEMPT;
        }
        if (psmode < rep) rep = psmode;
      }
    }
    __syncwarp(gmask);  // rows written by lane 0 are read by every lane for the next podset's assumed usage
  }
  *borrowing_out = borrowing;
  return rep;
}

// getInitialAssignments (scheduler.go:584-625) in cooperative form; targets are never produced here (deferred).
template <int NG = KB_NG>
__device__ inline int get_assignments_coop(const DevSnap &D, bool *need_search, int wl, int *borrowing_out, unsigned gmask, int gbase, int glane) {
  int mode = assign_workload_coop<NG>(D, need_search, wl, nullptr, borrowing_out, gmask, gbase, glane);
  if (mode == KB_MODE_FIT) return mode;
  if (mode == KB_MODE_PREEMPT && candidates_possible(D, D.wl_cq[wl])) *need_search = true;  // GetTargets might find targets
  if (!(D.flags & KB_F_PARTIAL_ADMISSION)) return mode;
  int ps0 = D.wl_ps_start[wl], np = D.wl_ps_start[wl + 1] - ps0;
  if (np > KB_MAX_PODSETS) return mode;
  int total = 0; bool can = false;
  for (int i = 0; i < np; i++) {
    int mc = D.ps_min_count[ps0 + i], full = D.ps_count[ps0 + i];
    if (mc >= 0) { total += full - mc; if (full > mc) can = true; }
  }
  if (!can || total == 0) return mode;
  int32_t counts[KB_MAX_PODSETS];
  auto fill = [&](int i) {
    for (int k = 0; k < np; k++) {
      int mc = D.ps_min_count[ps0 + k], full = D.ps_count[ps0 + k];
      int delta = mc >= 0 ? full - mc : 0;
      counts[k] = full - (int32_t)((i64)delta * i / total);
    }
  };
  int last_good = -1, lo = 0, hi = total + 1;
  while (lo < hi) {
    int mid = lo + (hi - lo) / 2;
    fill(mid);
    int b;
    __syncwarp(gmask);
    int m = assign_workload_coop<NG>(D, need_search, wl, counts, &b, gmask, gbase, glane);
    bool good = m == KB_MODE_FIT;  // Preempt with targets is only decidable by the search kernel (entry already flagged)
    if (good) { last_good = mid; hi = mid; } else lo = mid + 1;
  }
  __syncwarp(gmask);
  if (last_good >= 0 && lo == last_good) {
    fill(last_good);
    return assign_workload_coop<NG>(D, need_search, wl, counts, borrowing_out, gmask, gbase, glane);
  }
  return assign_workload_coop<NG>(D, need_search, wl, nullptr, borrowing_out, gmask, gbase, glane);
}

__global__ void __launch_bounds__(128) k_nominate_coop(DevSnap D) {
  int gid = (blockIdx.x * blockDim.x + threadIdx.x) / KB_NG;
  int lane = threadIdx.x & 31, glane = lane % KB_NG, gbase = lane - glane;
  unsigned gmask = (KB_NG == 32 ? 0xffffffffu : ((1u << KB_NG) - 1u)) << gbase;
  if (gid >= D.H) return;
  int e = gid;
  int wl = D.heads[e];
  bool need_search = false;
  int borrowing;
  int mode = get_assignments_coop(D, &need_search, wl, &borrowing, gmask, gbase, glane);
  if (glane != 0) return;
  D.mode[e] = (uint8_t)mode;
  D.borrow[e] = borrowing;
  D.decision[e] = KB_DEC_NOFIT;
  D.rank[e] = -1;
  D.tgt_cnt[e] = 0;
  D.tgt_off[e] = 0;
  if (need_search) D.ps_list[atomicAdd(D.ps_n, 1)] = e;
  {
    int slot = D.root_slot[D.wl_cq[wl]];
    unsigned act = __activemask();
    unsigned m = __match_any_sync(act, slot);
    if (lane == __ffs(m) - 1) atomicAdd(&D.root_count[slot], __popc(m));
  }
}

__global__ void __launch_bounds__(128) k_nominate(DevSnap D) {
  int e = blockIdx.x * blockDim.x + threadIdx.x;
  if (e >= D.H) return;
  int wl = D.heads[e];
  NomThread orc;
  int borrowing, nt;
  int mode = get_assignments(D, orc, wl, &borrowing, &nt);
  D.mode[e] = (uint8_t)mode;
  D.borrow[e] = borrowing;
  D.decision[e] = KB_DEC_NOFIT;
  D.rank[e] = -1;
  D.tgt_cnt[e] = 0;
  D.tgt_off[e] = 0;
  if (orc.need_search) {
    D.ps_list[atomicAdd(D.ps_n, 1)] = e;
  }
  {  // count entries per root: one atomic per distinct root in the warp (heads are usually grouped by CQ)
    int slot = D.root_slot[D.wl_cq[wl]];
    unsigned act = __activemask();
    unsigned m = __match_any_sync(act, slot);
    if ((threadIdx.x & 31) == __ffs(m) - 1) atomicAdd(&D.root_count[slot], __popc(m));
  }
}

// ClusterQueues (with a cohort) whose usage exceeds nominal in some flavor-resource at cycle
// start, listed per root: the only queues a target search can take cohort candidates from
// (IsWithinNominalInResources resource_node.go:248-255 is false only for them).
__global__ void k_over(DevSnap D) {
  int q = blockIdx.x * blockDim.x + threadIdx.x;
  if (q >= D.Q || D.parent[q] < 0) return;
  const int FR = D.FR;
  bool over = false;
  for (int fr = 0; fr < FR; fr++) over |= D.usage[(size_t)q * FR + fr] > D.subtree[(size_t)q * FR + fr];
  if (!over) return;
  int slot = D.root_slot[q];
  D.over_list[D.root_cq_start[slot] + atomicAdd(&D.over_count[slot], 1)] = q;
}

// ---------------------------------------------------------------------------
// K6: nominate with target search for the entries k_nominate deferred.
//
// Classical / hierarchical preemption: k_search_cells runs every SimulatePreemption call the flavor walks of
// the deferred entries can make for their first podset (one warp per (entry, flavor-resource) cell, results
// memoised by quantity), then k_nominate_walk replays getInitialAssignments per entry (one warp each, all lanes
// executing the scalar control flow redundantly and cooperating inside the searches, kb_search.cuh).
// Fair sharing: k_nominate_search_fair (the DominantResourceShare tournament reads every column of the tree).
// ---------------------------------------------------------------------------
__device__ __forceinline__ size_t align16(size_t x) { return (x + 15) & ~(size_t)15; }

// Would the flavor walk of the first podset of entry `item` call the preemption oracle on flavor-resource fr?
// (fitsResourceQuota flavorassigner.go:1017-1047 reaches SimulatePreemption.)  *req = the quantity it would pass.
__device__ inline bool oracle_cell_needed(const DevSnap &D, int item, int fr, int *wl_out, int *cq_out, i64 *req) {
  const int R = D.R;
  int wl = D.heads[D.ps_list[item]], cq = D.wl_cq[wl];
  *wl_out = wl; *cq_out = cq;
  int row = D.wl_ps_start[wl];
  if (!(D.wl_ps_start[wl + 1] > row) || !candidates_possible(D, cq)) return false;
  int f = fr / R, r = fr % R;
  bool covers_pods = D.pods_res >= 0 && rg_by_resource(D, cq, D.pods_res) >= 0;
  uint32_t mask = D.ps_req_mask[row] | (covers_pods ? 1u << D.pods_res : 0u);
  int g = ((mask >> r) & 1) && ((D.ps_flavor_ok[row] >> f) & 1) ? rg_by_resource(D, cq, r) : -1;
  bool in_rg = false;
  if (g >= 0) for (int k = D.rg_flavor_start[g]; k < D.rg_flavor_start[g + 1]; k++) in_rg |= D.rg_flavors[k] == f;
  if (!in_rg) return false;
  *req = ps_request(D, row, r, D.ps_count[row], covers_pods);
  int b0;
  return cell_eval(D, cq, fr, 0, *req, &b0) == PM_NEED;
}

// Ungrouped form (trees too large to share a column per CTA): warps pull (entry, flavor-resource) cells in order.
__global__ void __launch_bounds__(512) k_search_cells(DevSnap D, int col_smem_elems, int codes_smem, int list_cap) {
  extern __shared__ __align__(16) unsigned char smem_raw[];
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, wpb = blockDim.x >> 5;
  const size_t gw = (size_t)blockIdx.x * wpb + warp;
  const size_t ctx_b = align16(sizeof(WCtx<1>)), col_b = align16((size_t)col_smem_elems * 8), codes_b = align16((size_t)codes_smem);
  unsigned char *base = smem_raw + (size_t)warp * (ctx_b + col_b + codes_b);
  WCtx<1> *w = reinterpret_cast<WCtx<1> *>(base);
  WScratch S;
  S.col = col_smem_elems ? reinterpret_cast<i64 *>(base + ctx_b) : D.ws_col + gw * D.ws_col_stride;
  S.codes = codes_smem ? base + ctx_b + col_b : D.ws_codes + gw * list_cap;
  S.tgt = D.ws_tgt + gw * list_cap; S.tgt_reason = D.ws_tgt_reason + gw * list_cap;
  S.tgtq = D.ws_tgtq + gw * D.ws_tgtq_cap;
  const int FR = D.FR;
  const int n_items = min(*D.ps_n, D.memo_items);
  const long long total = (long long)n_items * FR;
  while (true) {
    int chunk = 0;
    if (lane == 0) chunk = atomicAdd(D.cell_cursor, 1);
    chunk = __shfl_sync(0xffffffffu, chunk, 0);
    long long idx = (long long)chunk * 32 + lane;
    if ((long long)chunk * 32 >= total) break;
    bool need = false; int item = 0, fr = 0, wl = 0, cq = 0; i64 req = 0;
    if (idx < total) { item = (int)(idx / FR); fr = (int)(idx % FR); need = oracle_cell_needed(D, item, fr, &wl, &cq, &req); }
    if (idx < total && !need) D.memo[idx].val = -1;  // memo row index = item * FR + fr: no oracle call expected here
    unsigned m = __ballot_sync(0xffffffffu, need);
    while (m) {
      int src = __ffs(m) - 1; m &= m - 1;
      int s_item = __shfl_sync(0xffffffffu, item, src), s_fr = __shfl_sync(0xffffffffu, fr, src);
      int s_wl = __shfl_sync(0xffffffffu, wl, src), s_cq = __shfl_sync(0xffffffffu, cq, src);
      i64 s_req = __shfl_sync(0xffffffffu, req, src);
      int borrow;
      int pm = ws_simulate<1>(D, w, S, s_wl, s_cq, s_fr, s_req, &borrow);
      if (lane == 0) { SimMemo mm; mm.val = s_req; mm.pm = pm; mm.borrow = borrow; D.memo[(size_t)s_item * FR + s_fr] = mm; }
      __syncwarp();
    }
  }
}

// Grouped form: the oracle cells are bucketed by (root, flavor-resource) first (k_cells_mark -> scan -> k_cells_scatter),
// so that a CTA works on ONE column at a time: the column's static cell records (32 B per node) and cycle-start usage
// are staged in shared memory once per task and every dependent step of its warps' greedy loops (removeUsage /
// available walks, above-nominal checks) is a shared-memory access.
__global__ void k_cells_mark(DevSnap D) {
  const int FR = D.FR;
  long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  const int n_items = min(*D.ps_n, D.memo_items);
  if (idx >= (long long)n_items * FR) return;
  int item = (int)(idx / FR), fr = (int)(idx % FR), wl, cq; i64 req = 0;
  bool need = oracle_cell_needed(D, item, fr, &wl, &cq, &req);
  SimMemo mm; mm.val = need ? req : -1; mm.pm = -1; mm.borrow = 0;  // pm -1: search pending
  D.memo[idx] = mm;
  if (need) atomicAdd(&D.cell_count[(size_t)D.root_slot[cq] * FR + fr], 1);
}
__global__ void k_cells_scatter(DevSnap D) {
  const int FR = D.FR;
  long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  const int n_items = min(*D.ps_n, D.memo_items);
  if (idx >= (long long)n_items * FR) return;
  if (D.memo[idx].val < 0) return;
  int item = (int)(idx / FR), fr = (int)(idx % FR);
  int cq = D.wl_cq[D.heads[D.ps_list[item]]];
  int b = D.root_slot[cq] * FR + fr;
  int pos = D.cell_start[b] + atomicAdd(&D.cell_fill[b], 1);
  D.cell_list[pos] = (int)idx; D.cell_bucket[pos] = b;
}
#define KB_CELL_TASK 512     // oracle cells per CTA task: at most / at least
#define KB_CELL_TASK_MIN 32
__global__ void __launch_bounds__(512) k_search_cells_grouped(DevSnap D, int ncap, int codes_smem, int list_cap) {
  extern __shared__ __align__(16) unsigned char smem_raw[];
  __shared__ int s_task, s_task_n, s_next;
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, wpb = blockDim.x >> 5;
  const size_t gw = (size_t)blockIdx.x * wpb + warp;
  const int FR = D.FR;
  ColStat *sh_stat = reinterpret_cast<ColStat *>(smem_raw);
  i64 *sh_base = reinterpret_cast<i64 *>(smem_raw + (size_t)ncap * sizeof(ColStat));
  const size_t shared_b = align16((size_t)ncap * (sizeof(ColStat) + 8));
  const size_t ctx_b = align16(sizeof(WCtx<1>)), col_b = align16((size_t)ncap * 8), codes_b = align16((size_t)codes_smem);
  unsigned char *base = smem_raw + shared_b + (size_t)warp * (ctx_b + col_b + codes_b);
  WCtx<1> *w = reinterpret_cast<WCtx<1> *>(base);
  WScratch S;
  S.col = reinterpret_cast<i64 *>(base + ctx_b);
  S.codes = codes_smem ? base + ctx_b + col_b : D.ws_codes + gw * list_cap;
  S.tgt = D.ws_tgt + gw * list_cap; S.tgt_reason = D.ws_tgt_reason + gw * list_cap;
  S.tgtq = D.ws_tgtq + gw * D.ws_tgtq_cap;
  S.stat0 = sh_stat; S.base0 = sh_base;
  const int n_cells = D.cell_start[D.nRoots * FR];
  int staged = -1;
  while (true) {
    // Guided self-scheduling over the bucket-grouped cell list: a CTA claims a share of what is left (large tasks while
    // there is plenty, KB_CELL_TASK_MIN at the end), so the barrier per task is amortised and the kernel's tail is short.
    __syncthreads();
    if (threadIdx.x == 0) {
      int seen = *(volatile int *)D.cell_cursor;
      int chunk = (n_cells - seen) / (2 * (int)gridDim.x);
      chunk = max(KB_CELL_TASK_MIN, min(KB_CELL_TASK, chunk));
      s_task = atomicAdd(D.cell_cursor, chunk);
      s_task_n = chunk;
    }
    __syncthreads();
    const int lo = s_task, hi = min(lo + s_task_n, n_cells);
    if (lo >= n_cells) break;
    for (int p = lo; p < hi;) {
      const int b = D.cell_bucket[p];
      int q = p + 1;
      while (q < hi && D.cell_bucket[q] == b) q++;  // run of cells in the same bucket (the list is grouped by bucket)
      __syncthreads();  // every warp is done with the previous run and its column
      if (b != staged) {
        const int slot = b / FR, fr = b % FR;
        const int nbase = D.slot_base[slot], nn = D.slot_base[slot + 1] - nbase;
        const size_t o = (size_t)nbase * FR + (size_t)fr * nn;
        const int4 *src = reinterpret_cast<const int4 *>(D.colS + o);
        int4 *dst = reinterpret_cast<int4 *>(sh_stat);
        for (int i = threadIdx.x; i < nn * 2; i += blockDim.x) dst[i] = __ldg(src + i);
        for (int i = threadIdx.x; i < nn; i += blockDim.x) sh_base[i] = D.colU[o + i];
        staged = b;
      }
      if (threadIdx.x == 0) s_next = p;
      __syncthreads();
      while (true) {  // searches differ a lot in length: warps take the run's cells one at a time
        int c = 0;
        if (lane == 0) c = atomicAdd(&s_next, 1);
        c = __shfl_sync(0xffffffffu, c, 0);
        if (c >= q) break;
        const int idx = D.cell_list[c];
        const int item = idx / FR, fr = idx % FR;
        const int wl = D.heads[D.ps_list[item]], cq = D.wl_cq[wl];
        const i64 req = D.memo[idx].val;
        int borrow;
        int pm = ws_simulate<1>(D, w, S, wl, cq, fr, req, &borrow);
        if (lane == 0) { SimMemo mm; mm.val = req; mm.pm = pm; mm.borrow = borrow; D.memo[idx] = mm; }
        __syncwarp();
      }
      p = q;
    }
  }
}

// Oracle policy of k_nominate_walk: every lane of the warp executes the flavor walk; searches are warp-cooperative.
struct NomWarp {
  WCtx<KB_MAX_CELLS> *w;
  WScratch S;
  i64 *col_smem; int col_smem_elems; i64 *col_glob;
  const SimMemo *memo;  // [FR] speculative results of this entry, or nullptr
  __device__ __forceinline__ void pick_col(const DevSnap &D, int cq, int K) {
    int slot = D.root_slot[cq];
    int nn = D.slot_base[slot + 1] - D.slot_base[slot];
    S.col = ((size_t)K * nn <= (size_t)col_smem_elems) ? col_smem : col_glob;
  }
  __device__ inline int simulate(const DevSnap &D, int wl, int cq, int fr, i64 val, int *borrow_after) {
    if (memo) { SimMemo m = memo[fr]; if (m.val == val) { *borrow_after = m.borrow; return m.pm; } }
    if (!candidates_possible(D, cq)) {
      bool may_reclaim;
      *borrow_after = find_height(D, D.usage, cq, fr, val, &may_reclaim);
      return PM_NOCAND;
    }
    pick_col(D, cq, 1);
    return ws_simulate<KB_MAX_CELLS>(D, w, S, wl, cq, fr, val, borrow_after);
  }
  // GetTargets preemption.go:127-146 for the assignment currently in the output rows
  __device__ inline int get_targets(const DevSnap &D, int wl) {
    const int lane = threadIdx.x & 31;
    int cq = D.wl_cq[wl];
    if (!candidates_possible(D, cq)) return 0;
    const int R = D.R;
    __syncwarp();
    if (lane == 0) {
      w->cq = cq; w->prio = D.wl_priority[wl]; w->ts = D.wl_ts[wl];
      bool covers_pods = D.pods_res >= 0 && rg_by_resource(D, cq, D.pods_res) >= 0;
      int K = 0, nn = 0;
      for (int i = 0; i < 32; i++) w->need_bits[i] = 0;
      auto slot_of = [&](int fr) { int j = 0; while (j < K && w->tfr[j] != fr) j++; return j; };
      for (int row = D.wl_ps_start[wl]; row < D.wl_ps_start[wl + 1]; row++)
        for (int r = 0; r < R; r++) {
          int f = D.ps_flavor[(size_t)row * R + r];
          if (f < 0) continue;
          int fr = f * R + r;
          if (D.ps_res_mode[(size_t)row * R + r] == KB_MODE_PREEMPT) {  // flavorResourcesNeedPreemption :480-490
            int j = slot_of(fr);
            if (j == K && K < KB_MAX_CELLS) { w->tfr[K] = (uint16_t)fr; w->tflag[K] = 0; w->tq[K] = 0; K++; }
            if (j < K && !(w->tflag[j] & TC_NEED)) { w->tflag[j] |= TC_NEED; w->need_bits[fr >> 5] |= 1u << (fr & 31); nn++; }
          }
          i64 q = ps_request(D, row, r, D.ps_count_out[row], covers_pods);  // TotalRequestsFor flavorassigner.go:198-218
          if (q == 0) continue;
          int j = slot_of(fr);
          if (j == K) { if (K == KB_MAX_CELLS) continue; w->tfr[K] = (uint16_t)fr; w->tflag[K] = 0; w->tq[K] = 0; K++; }
          w->tflag[j] |= TC_USE; w->tq[j] += q;
        }
      w->K = K; w->n_need = nn;
    }
    __syncwarp();
    const int K = w->K;
    if (w->n_need == 0 || K == 0) return 0;
    pick_col(D, cq, K);
    if (K <= 32) {
      i64 myq[1] = {lane < K ? w->tq[lane] : 0};
      return ws_classical<KB_MAX_CELLS, 1>(D, w, S, myq);
    }
    i64 myq[4];
#pragma unroll
    for (int s = 0; s < 4; s++) myq[s] = lane + 32 * s < K ? w->tq[lane + 32 * s] : 0;
    return ws_classical<KB_MAX_CELLS, 4>(D, w, S, myq);
  }
};

__global__ void __launch_bounds__(256) k_nominate_walk(DevSnap D, int col_smem_elems, int list_cap) {
  extern __shared__ __align__(16) unsigned char smem_raw[];
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, wpb = blockDim.x >> 5;
  const size_t gw = (size_t)blockIdx.x * wpb + warp;
  const size_t ctx_b = align16(sizeof(WCtx<KB_MAX_CELLS>)), col_b = align16((size_t)col_smem_elems * 8);
  unsigned char *base = smem_raw + (size_t)warp * (ctx_b + col_b);
  NomWarp orc;
  orc.w = reinterpret_cast<WCtx<KB_MAX_CELLS> *>(base);
  orc.col_smem = reinterpret_cast<i64 *>(base + ctx_b); orc.col_smem_elems = col_smem_elems;
  orc.col_glob = D.ws_col + gw * D.ws_col_stride;
  orc.S.col = orc.col_glob;
  orc.S.codes = D.ws_codes + gw * list_cap;
  orc.S.tgt = D.ws_tgt + gw * list_cap; orc.S.tgt_reason = D.ws_tgt_reason + gw * list_cap;
  orc.S.tgtq = D.ws_tgtq + gw * D.ws_tgtq_cap;
  const int n_items = *D.ps_n;
  while (true) {
    int item = 0;
    if (lane == 0) item = atomicAdd(D.ps_cursor, 1);
    item = __shfl_sync(0xffffffffu, item, 0);
    if (item >= n_items) break;
    int e = D.ps_list[item];
    int wl = D.heads[e];
    orc.memo = item < D.memo_items ? D.memo + (size_t)item * D.FR : nullptr;
    int borrowing, nt;
    int mode = get_assignments(D, orc, wl, &borrowing, &nt);
    __syncwarp();
    int off = 0;
    if (nt > 0) {
      if (lane == 0) off = atomicAdd(D.tgt_pool_used, nt);
      off = __shfl_sync(0xffffffffu, off, 0);
      if (off + nt <= D.tgt_pool_cap) {
        for (int k = lane; k < nt; k += 32) { D.tgt_pool_adm[off + k] = orc.S.tgt[k]; D.tgt_pool_reason[off + k] = orc.S.tgt_reason[k]; }
      } else { if (lane == 0) atomicOr(D.status, KBS_TARGET_OVERFLOW); nt = 0; }
    }
    if (lane == 0) { D.mode[e] = (uint8_t)mode; D.borrow[e] = borrowing; D.tgt_cnt[e] = nt; D.tgt_off[e] = off; }
    __syncwarp();
  }
}

// Fair-sharing preemption (kb_preempt.cuh): flavor assignment and target searches of one deferred entry run on
// lane 0 of a single-warp CTA on a private copy of the root's whole tree (the DominantResourceShare reads every
// column); the other lanes only stage the tree.
template <bool kSmem>
struct NomSearch {
  const PTab<kSmem> *T;
  PreCtx *c;
  PreScratch S;
  const SimMemo *memo = nullptr;  // [FR] results of k_fair_cells for this entry, or nullptr
  // SimulatePreemption preemption_oracle.go:41-71 on the private tree
  __device__ inline int simulate(const DevSnap &D, int wl, int cq, int fr, i64 val, int *borrow_after) {
    if (memo) { SimMemo m = memo[fr]; if (m.val == val && m.pm >= 0) { *borrow_after = m.borrow; return m.pm; } }
    int hcq = T->handle(cq);
    *borrow_after = T->find_height(hcq, fr, val);  // no candidates: height on the untouched snapshot (:53-56)
    if (!candidates_possible(D, cq)) return PM_NOCAND;
    c->cq = cq; c->prio = D.wl_priority[wl]; c->ts = D.wl_ts[wl];
    c->n_use = 1; c->use_fr[0] = fr; c->use_q[0] = val;
    c->n_need = 1; c->need_fr[0] = fr;
    fair_search<kSmem>(D, *T, c, S);
    int nt = c->n_targets;
    if (nt == 0) return PM_NOCAND;
    for (int k = 0; k < nt; k++) T->remove_adm(S.tgt[k]);
    *borrow_after = T->find_height(hcq, fr, val);
    for (int k = 0; k < nt; k++) T->add_adm(S.tgt[k]);
    for (int k = 0; k < nt; k++) if (D.adm_cq[S.tgt[k]] == cq) return PM_PREEMPT;
    return PM_RECLAIM;
  }
  // GetTargets preemption.go:127-146 for the assignment currently in the output rows
  __device__ inline int get_targets(const DevSnap &D, int wl) {
    int cq = D.wl_cq[wl];
    if (!candidates_possible(D, cq)) return 0;
    const int R = D.R;
    c->cq = cq; c->prio = D.wl_priority[wl]; c->ts = D.wl_ts[wl];
    bool covers_pods = D.pods_res >= 0 && rg_by_resource(D, cq, D.pods_res) >= 0;
    int nu = 0, nn = 0;
    for (int row = D.wl_ps_start[wl]; row < D.wl_ps_start[wl + 1]; row++)
      for (int r = 0; r < R; r++) {
        int f = D.ps_flavor[(size_t)row * R + r];
        if (f < 0) continue;
        int fr = f * R + r;
        if (D.ps_res_mode[(size_t)row * R + r] == KB_MODE_PREEMPT) {  // flavorResourcesNeedPreemption :480-490
          int j = 0; while (j < nn && c->need_fr[j] != fr) j++;
          if (j == nn && nn < KB_MAX_CELLS) c->need_fr[nn++] = fr;
        }
        i64 q = ps_request(D, row, r, D.ps_count_out[row], covers_pods);  // TotalRequestsFor flavorassigner.go:198-218
        if (q == 0) continue;
        int j = 0; while (j < nu && c->use_fr[j] != fr) j++;
        if (j == nu) { if (nu == KB_MAX_CELLS) continue; c->use_fr[nu] = fr; c->use_q[nu] = 0; nu++; }
        c->use_q[j] += q;
      }
    c->n_use = nu; c->n_need = nn;
    fair_search<kSmem>(D, *T, c, S);
    return c->n_targets;
  }
};

// kCells: the searches of the preemption oracle are independent of each other (every SimulatePreemption starts from
// the cycle's snapshot), so they run first, one (entry, flavor-resource) cell per task over the whole grid, and leave
// their results in the memo; the per-entry walk (kCells = false) then replays the flavor assignment against the memo
// and only runs GetTargets itself.
template <bool kSmem, bool kCells>
__global__ void __launch_bounds__(32, 16) k_nominate_search_fair(DevSnap D) {  // <= 128 registers: 16 single-warp CTAs per SM
  extern __shared__ __align__(16) unsigned char smem_raw[];
  __shared__ PreCtx ctx;
  __shared__ int s_item;
  const int FR = D.FR;
  PreScratch S;   // scratch of the CTA's sequential searcher (lane 0)
  {
    size_t b = blockIdx.x;
    S.cand = {D.sc_cand + b * D.sc_adm_cap}; S.variant = {D.sc_variant + b * D.sc_adm_cap};
    S.tgt = {D.sc_tgt + b * D.sc_adm_cap}; S.tgt_reason = {D.sc_tgt_reason + b * D.sc_adm_cap};
    S.cq_class = {D.sc_cq_class + b * D.sc_node_cap}; S.on_path = {D.sc_on_path + b * D.sc_node_cap};
    S.cq_lca = {D.sc_cq_lca + b * D.sc_node_cap};
    S.aux1 = {D.sc_aux1 + b * D.sc_adm_cap}; S.aux2 = {D.sc_aux2 + b * D.sc_adm_cap};
    S.cap = D.sc_adm_cap;
  }
  PTab<kSmem> T;
  T.D = &D; T.FR = FR;
  T.dirty = D.sc_dirty + (size_t)blockIdx.x * D.sc_node_cap; T.drs_ratio = D.sc_drs_ratio + (size_t)blockIdx.x * D.sc_node_cap;
  T.drs_meta = D.sc_drs_meta + (size_t)blockIdx.x * D.sc_node_cap;
  unsigned char *smem_tab = smem_raw;
  if (kSmem) {  // per-node search state next to the tree: [share 8 B][queue head 4 B][on_path][pruned][dirty][share meta]
    const size_t cap = (size_t)D.sc_node_cap;
    T.drs_ratio = (double *)smem_raw;
    S.cq_lca = {(int32_t *)(smem_raw + cap * 8)};
    S.on_path = {(int8_t *)(smem_raw + cap * 12)};
    S.cq_class = {(int8_t *)(smem_raw + cap * 13)};
    T.dirty = smem_raw + cap * 14;
    T.drs_meta = (int8_t *)(smem_raw + cap * 15);
    smem_tab = smem_raw + ((cap * 16 + 15) & ~(size_t)15);
  }
  int cur_slot = -1;
  const int n_items = kCells ? min(*D.ps_n, D.memo_items) : *D.ps_n;
  while (true) {
    __syncthreads();
    if (threadIdx.x == 0) s_item = atomicAdd(kCells ? D.cell_cursor : D.ps_cursor, 1);
    __syncthreads();
    int item = s_item, cell_fr = 0;
    if (kCells) { cell_fr = item % FR; item /= FR; }
    if (item >= n_items) break;
    int e = D.ps_list[item];
    int wl = D.heads[e];
    int cq = D.wl_cq[wl];
    i64 cell_req = 0;
    if (kCells) {  // cells the flavor walk would not ask the oracle about are marked and skipped (uniform over the warp)
      int wl2, cq2;
      bool need = oracle_cell_needed(D, item, cell_fr, &wl2, &cq2, &cell_req);
      if (!need) { if (threadIdx.x == 0) { SimMemo mm; mm.val = -1; mm.pm = -1; mm.borrow = 0; D.memo[(size_t)item * FR + cell_fr] = mm; } continue; }
    }
    int slot = D.root_slot[cq];
    if (slot != cur_slot) {  // stage a private copy of the root's tree (the search restores it after use)
      cur_slot = slot;
      if (slot < D.nLone) { T.nodes = &D.lone_cqs[slot]; T.nn = 1; }
      else { int t = slot - D.nLone; T.nodes = D.tree_nodes + D.tree_start[t]; T.nn = D.tree_start[t + 1] - D.tree_start[t]; }
      size_t tb = (size_t)T.nn * FR;
      if (kSmem) {
        i64 *u = (i64 *)smem_tab, *sb = u + tb, *lq = sb + tb, *bl = lq + tb;
        int *lp = (int *)(bl + tb);
        for (int i = threadIdx.x; i < (int)tb; i += blockDim.x) {
          size_t c = (size_t)T.nodes[i / FR] * FR + i % FR;
          i64 sub = D.subtree[c];
          u[i] = D.usage[c]; sb[i] = sub; lq[i] = local_quota(sub, D.llimit[c]); bl[i] = D.blimit[c];
        }
        for (int i = threadIdx.x; i < T.nn; i += blockDim.x) { int pn = D.parent[T.nodes[i]]; lp[i] = pn < 0 ? -1 : D.local_idx[pn]; }
        T.usage = u; T.sub = sb; T.lq = lq; T.bl = bl; T.lparent = lp;
      } else {
        i64 *u = D.sc_usage + (size_t)blockIdx.x * D.sc_node_cap * FR;
        for (int i = threadIdx.x; i < (int)tb; i += blockDim.x) u[i] = D.usage[(size_t)T.nodes[i / FR] * FR + i % FR];
        T.usage = u;
      }
      __syncthreads();
    }
    if (kCells) {
      if (threadIdx.x == 0) {
        NomSearch<kSmem> orc{&T, &ctx, S};
        int borrow;
        int pm = orc.simulate(D, wl, cq, cell_fr, cell_req, &borrow);
        SimMemo mm; mm.val = cell_req; mm.pm = pm; mm.borrow = borrow;
        D.memo[(size_t)item * FR + cell_fr] = mm;
      }
      continue;
    }
    if (threadIdx.x == 0) {
      NomSearch<kSmem> orc{&T, &ctx, S};
      orc.memo = item < D.memo_items ? D.memo + (size_t)item * FR : nullptr;
      int borrowing, nt;
      int mode = get_assignments(D, orc, wl, &borrowing, &nt);
      D.mode[e] = (uint8_t)mode;
      D.borrow[e] = borrowing;
      int off = 0;
      if (nt > 0) {
        off = atomicAdd(D.tgt_pool_used, nt);
        if (off + nt <= D.tgt_pool_cap) {
          for (int k = 0; k < nt; k++) { D.tgt_pool_adm[off + k] = S.tgt[k]; D.tgt_pool_reason[off + k] = S.tgt_reason[k]; }
        } else { atomicOr(D.status, KBS_TARGET_OVERFLOW); nt = 0; }
      }
      D.tgt_cnt[e] = nt; D.tgt_off[e] = off;
    }
  }
}


// dense request of entry e for column fr (absent = -1); defined before the key computation
__device__ __forceinline__ i64 entry_request_early(const DevSnap &D, int e, int fr) {
  const int R = D.R;
  int f = fr / R, r = fr % R;
  int wl = D.heads[e];
  int cq = D.wl_cq[wl];
  bool covers_pods = D.pods_res >= 0 && rg_by_resource(D, cq, D.pods_res) >= 0;
  i64 q = -1;
  for (int row = D.wl_ps_start[wl]; row < D.wl_ps_start[wl + 1]; row++)
    if (D.ps_flavor[(size_t)row * R + r] == f) q = (q < 0 ? 0 : q) + ps_request(D, row, r, D.ps_count_out[row], covers_pods);
  return q;
}

// Iterator order as a 4 x u64 lexicographic key per entry (D.ekey):
//   classical (scheduler.go:778-817): [Borrowing | priority desc] [queue-order timestamp] [entry index] [0]
//   fair sharing in a FLAT cohort (every ClusterQueue directly under the root): the DominantResourceShare a
//   ClusterQueue would have with its entry admitted depends only on its own usage, which no other pop changes,
//   so the tournament's pop sequence (fair_sharing_iterator.go:120-199) is the order of
//   [requiresBorrowing, zeroWeightBorrows | share hi] [share lo | priority desc] [timestamp] [cq index].
// One term of dominantResourceShare(cq) with the entry's usage added (computeDRS fair_sharing_iterator.go:206-229):
// borrowed[r] * 1000 / lendable[r] (fair_sharing.go:126-156), 0 when nothing is borrowed or lendable.
// borrowed[r] = sum_f max(0, usage + q - SubtreeQuota); only the cells the entry is assigned to differ from the
// ClusterQueue's own over-usage, which k_fair_prep precomputed per (cq, resource) together with lendable[r].
__device__ inline double entry_share_ratio(const DevSnap &D, int e, int r) {
  const int wl = D.heads[e];
  const int cq = D.wl_cq[wl];
  const int hq = nix(D, cq);
  const int P = D.parent[hq];
  const int R = D.R, FR = D.FR;
  const bool covers_pods = D.pods_res >= 0 && rg_by_resource(D, cq, D.pods_res) >= 0;
  i64 b = D.fs_over[(size_t)hq * R + r];
  // flavors this entry uses for resource r (aggregated over its podsets)
  const int ps0 = D.wl_ps_start[wl], ps1 = D.wl_ps_start[wl + 1];
  for (int row = ps0; row < ps1; row++) {
    const int f = D.ps_flavor[(size_t)row * R + r];
    if (f < 0) continue;
    bool first = true;  // count each (f, r) cell once, with the summed request of all podsets on it
    for (int prow = ps0; prow < row; prow++) if (D.ps_flavor[(size_t)prow * R + r] == f) first = false;
    if (!first) continue;
    i64 q = 0;
    for (int prow = row; prow < ps1; prow++)
      if (D.ps_flavor[(size_t)prow * R + r] == f) q += ps_request(D, prow, r, D.ps_count_out[prow], covers_pods);
    const size_t c = (size_t)hq * FR + (size_t)f * R + r;
    const i64 base = D.usage[c] - D.subtree[c];
    b += imax(0, base + (q > 0 ? q : 0)) - imax(0, base);
  }
  const i64 lend = D.fs_lend[(size_t)P * R + r];
  return (b > 0 && lend > 0) ? (double)b * 1000.0 / (double)lend : 0.0;
}
// Is the entry ordered by the flat-cohort fair-sharing key (else: the classical key)?
__device__ __forceinline__ bool entry_key_is_fair_flat(const DevSnap &D, int e) {
  const int cq = D.wl_cq[D.heads[e]];
  const int P = D.parent[nix(D, cq)];
  return (D.flags & KB_F_FAIR_SHARING) && P >= 0 && (D.tab_local == 2 ? D.local_flat != 0 : D.tree_flat[D.root_slot[cq] - D.nLone] != 0);
}
// The 4 x u64 key from the entry's fields: `best` = max over the resources of entry_share_ratio and `weight` the
// ClusterQueue's fair weight (both only read on the fair flat path); `ident` = the ClusterQueue's node id on the fair
// flat path, else the entry id.
__device__ __forceinline__ void entry_key_pack(unsigned flags, bool fair_flat, double best, double weight, int priority, i64 wl_ts,
                                               bool has_qr, int borrow, unsigned ident, u64 *k) {
  unsigned prio = 0;
  if (flags & KB_F_PRIORITY_SORTING_WITHIN_COHORT) prio = ~((unsigned)priority ^ 0x80000000u);  // signed priority, descending
  const u64 ts = (u64)wl_ts ^ 0x8000000000000000ull;
  if (!fair_flat) {
    // workloads that already hold a quota reservation (second pass) first: scheduler.go:781-789
    const u64 no_qr = has_qr ? 0ull : 1ull;
    k[0] = (no_qr << 63) | ((u64)(unsigned)borrow << 32) | prio; k[1] = ts; k[2] = (u64)ident; k[3] = 0;
    return;
  }
  const bool zwb = weight == 0 && best != 0;
  const double value = zwb ? best : (best == 0 ? 0.0 : best / weight);
  const u64 vb = (u64)__double_as_longlong(value);  // value >= 0: the bit pattern is monotone
  const u64 kf = ((flags & KB_F_FS_PRIORITIZE_NON_BORROWING) && borrow > 0 ? 2 : 0) | (zwb ? 1 : 0);
  k[0] = (kf << 32) | (vb >> 32); k[1] = (vb << 32) | prio; k[2] = ts; k[3] = (u64)ident;
}
__device__ inline void entry_key_finish(const DevSnap &D, int e, bool fair_flat, double best, u64 *k) {
  const int wl = D.heads[e];
  const int cq = D.wl_cq[wl];
  const bool has_qr = D.wl_has_qr && D.wl_has_qr[wl];
  const unsigned ident = fair_flat ? (unsigned)(D.node_gid ? D.node_gid[cq] : cq) : (unsigned)(D.ent_gid ? D.ent_gid[e] : e);
  entry_key_pack(D.flags, fair_flat, best, fair_flat ? D.fair_weight[cq] : 0.0, D.wl_priority[wl], D.wl_ts[wl], has_qr, D.borrow[e], ident, k);
}
__device__ inline void compute_entry_key(const DevSnap &D, int e, u64 *k) {
  const bool fair_flat = entry_key_is_fair_flat(D, e);
  double best = 0.0;
  if (fair_flat)
    for (int r = 0; r < D.R; r++) { const double ratio = entry_share_ratio(D, e, r); if (ratio > best) best = ratio; }
  entry_key_finish(D, e, fair_flat, best, k);
}
__device__ __forceinline__ bool key4_less(const u64 *a, const u64 *b) {
  if (a[0] != b[0]) return a[0] < b[0];
  if (a[1] != b[1]) return a[1] < b[1];
  if (a[2] != b[2]) return a[2] < b[2];
  return a[3] < b[3];
}

// ---------------------------------------------------------------------------
// K3: group entries by root (counting sort: count in K2, scan, scatter)
// ---------------------------------------------------------------------------
__global__ void __launch_bounds__(1024) k_scan_roots(DevSnap D) {
  __shared__ int32_t warp_sums[32];
  __shared__ int32_t carry;
  if (threadIdx.x == 0) carry = 0;
  __syncthreads();
  int n = D.nRoots;
  for (int base = 0; base < n; base += blockDim.x) {
    int i = base + threadIdx.x;
    int v = i < n ? D.root_count[i] : 0;
    int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
    int x = v;
    for (int o = 1; o < 32; o <<= 1) { int y = __shfl_up_sync(0xffffffffu, x, o); if (lane >= o) x += y; }
    if (lane == 31) warp_sums[w] = x;
    __syncthreads();
    if (w == 0) {
      int s = warp_sums[lane];
      for (int o = 1; o < 32; o <<= 1) { int y = __shfl_up_sync(0xffffffffu, s, o); if (lane >= o) s += y; }
      warp_sums[lane] = s;
    }
    __syncthreads();
    int excl = carry + (w ? warp_sums[w - 1] : 0) + x - v;
    if (i < n) { D.root_offset[i] = excl; D.root_cursor[i] = 0; }
    __syncthreads();
    if (threadIdx.x == blockDim.x - 1) carry = excl + v;
    __syncthreads();
  }
  if (threadIdx.x == 0) D.root_offset[n] = carry;
}
__global__ void k_scatter(DevSnap D) {
  int e = blockIdx.x * blockDim.x + threadIdx.x;
  if (e >= D.H) return;
  int slot = D.root_slot[D.wl_cq[D.heads[e]]];
  // warp-aggregated cursor bump: one atomic per distinct root in the warp
  unsigned act = __activemask();
  unsigned m = __match_any_sync(act, slot);
  int lane = threadIdx.x & 31, leader = __ffs(m) - 1;
  int base = 0;
  if (lane == leader) base = atomicAdd(&D.root_cursor[slot], __popc(m));
  base = __shfl_sync(m, base, leader);
  D.root_entries[D.root_offset[slot] + base + __popc(m & ((1u << lane) - 1))] = e;
  u64 k[4];
  compute_entry_key(D, e, k);
  ulonglong2 *dst = (ulonglong2 *)(D.ekey + (size_t)e * 4);
  dst[0] = make_ulonglong2(k[0], k[1]); dst[1] = make_ulonglong2(k[2], k[3]);
  int pos = D.root_offset[slot] + base + __popc(m & ((1u << lane) - 1));
  D.pos_slot[pos] = slot;
  ulonglong2 *sd = (ulonglong2 *)(D.skey + (size_t)pos * 4);  // the same key in segment order, for k_rank's scan
  sd[0] = make_ulonglong2(k[0], k[1]); sd[1] = make_ulonglong2(k[2], k[3]);
}

// Fair sharing: per (ClusterQueue, resource) the usage above SubtreeQuota summed over flavors, and per
// (node, resource) the lendable capacity sum_f potentialAvailable(node, f) (calculateLendable fair_sharing.go:160-174).
__global__ void k_fair_prep(DevSnap D) {
  int i = blockIdx.x * blockDim.x + threadIdx.x;
  const int R = D.R, F = D.F, FR = D.FR;
  if (i >= D.N * R) return;
  int n = i / R, r = i % R;
  i64 over = 0, lend = 0;
  for (int f = 0; f < F; f++) {
    size_t c = (size_t)n * FR + (size_t)f * R + r;
    lend += D.potential[c];
    if (n < D.Q) { i64 o = D.usage[c] - D.subtree[c]; if (o > 0) over += o; }
  }
  D.fs_lend[i] = lend;
  if (n < D.Q) D.fs_over[i] = over;
}

// Rank of every entry among the entries of its root (roots with at most KB_RANK_CAP entries): a fully parallel
// all-pairs count.  The segments of the roots a CTA's 256 positions belong to are contiguous in skey; when that
// span fits KB_RANK_STAGE keys it is staged in shared memory with coalesced loads and scanned from there
// (threads of a warp mostly share the root -> broadcast reads), else the scan reads global memory.
// Writes the root's entries in iterator order to D.sorted.
#define KB_RANK_STAGE 1024
__global__ void __launch_bounds__(256) k_rank(DevSnap D) {
  __shared__ ulonglong2 s_key[KB_RANK_STAGE * 2];
  __shared__ int s_lo, s_hi;
  const int p0 = blockIdx.x * blockDim.x;
  const int plast = min(p0 + (int)blockDim.x, D.H) - 1;
  const int pos = p0 + threadIdx.x;
  if (threadIdx.x == 0) {
    s_lo = D.root_offset[D.pos_slot[p0]];
    s_hi = D.root_offset[D.pos_slot[plast] + 1];
  }
  int e = -1, off = 0, n = 0;
  if (pos < D.H) {
    e = D.root_entries[pos];
    int slot = D.pos_slot[pos];
    off = D.root_offset[slot]; n = D.root_offset[slot + 1] - off;
  }
  __syncthreads();
  const int lo = s_lo, span = s_hi - lo;
  const bool staged = span <= KB_RANK_STAGE;
  if (staged) {
    const ulonglong2 *g = (const ulonglong2 *)(D.skey + (size_t)lo * 4);
    for (int i = threadIdx.x; i < span * 2; i += blockDim.x) s_key[i] = g[i];
  }
  __syncthreads();
  if (e < 0 || n > KB_RANK_CAP) return;
  int rank = 0;
  if (staged) {
    ulonglong2 m0 = s_key[2 * (pos - lo)], m1 = s_key[2 * (pos - lo) + 1];
    u64 mine[4] = {m0.x, m0.y, m1.x, m1.y};
    const ulonglong2 *seg = s_key + 2 * (off - lo);
#pragma unroll 4
    for (int j = 0; j < n; j++) {
      ulonglong2 a = seg[2 * j], b = seg[2 * j + 1];
      u64 other[4] = {a.x, a.y, b.x, b.y};
      rank += key4_less(other, mine) ? 1 : 0;
    }
  } else {
    const ulonglong2 *src = (const ulonglong2 *)(D.skey + (size_t)pos * 4);
    ulonglong2 m0 = src[0], m1 = src[1];
    u64 mine[4] = {m0.x, m0.y, m1.x, m1.y};
    const ulonglong2 *seg = (const ulonglong2 *)(D.skey + (size_t)off * 4);
#pragma unroll 4
    for (int j = 0; j < n; j++) {
      ulonglong2 a = seg[2 * j], b = seg[2 * j + 1];
      u64 other[4] = {a.x, a.y, b.x, b.y};
      rank += key4_less(other, mine) ? 1 : 0;
    }
  }
  D.sorted[off + rank] = e;
}

// ---------------------------------------------------------------------------
// K5: ordered admit loop, one CTA per root (scheduler.go:269-401).
//
// Layout of the work inside the CTA:
//   1. sort the root's entries by the classical iterator order (scheduler.go:778-817)
//      with packed keys in shared memory (bitonic network, all threads);
//   2. stage the root's quota tree (usage, SubtreeQuota, localQuota, BorrowingLimit
//      per (node, fr)) in shared memory when it fits — the cohort tree of one root is
//      the whole coupling domain of the admit loop, so the sequential part never
//      touches HBM;
//   3. per tile of KB_TILE entries: all threads expand the assignments into a dense
//      request matrix q[entry][fr] in shared memory (coalesced reads of the podset
//      rows), then warp 0 commits the tile in order — lane l owns the flavor-resource
//      columns l, l+32, ...; columns are independent in the quota tree, so fit checks
//      and addUsage run lane-parallel with one __all_sync per entry.
// ---------------------------------------------------------------------------
#define KB_TILE 128
#define KB_ADMIT_THREADS 256
#define KB_LONE_CAP 256
#define KB_LONE_WARPS 4
#define KB_SORT_CAP 1024  // entries per root sortable in shared memory

// Quota-tree tables of one root, either staged in shared memory (node handle = local
// index inside the tree) or left in global memory (node handle = global node id).
template <bool kSmem>
struct Tab {
  const DevSnap *D;
  i64 *usage; const i64 *sub, *lq, *bl;  // smem mode only
  const int *lparent;                    // smem mode only
  int FR;
  // shadow usage table (global, [N][FR]): the root's usage WITHOUT the workloads preempted so far in this
  // cycle; live once *shadow_on != 0.  fits() (scheduler.go:503-511) evaluates on it instead of removing
  // and re-adding every preempted workload per entry.  Usage is a pure function of the ClusterQueue rows
  // (cohort usage = sum of max(0, child usage - child localQuota), resource_node.go:137-158), so keeping the
  // shadow in step with add/remove is exact.
  i64 *shadow; const int32_t *tnodes; int tnn; int *shadow_on;
  __device__ __forceinline__ i64 U(int nd, int fr) const { return kSmem ? usage[nd * FR + fr] : __ldcg(&D->usage[(size_t)nd * FR + fr]); }
  __device__ __forceinline__ void setU(int nd, int fr, i64 v) const { if (kSmem) usage[nd * FR + fr] = v; else __stcg(&D->usage[(size_t)nd * FR + fr], v); }
  __device__ __forceinline__ size_t scell(int nd, int fr) const { return (size_t)(kSmem ? tnodes[nd] : nd) * FR + fr; }
  template <bool S> __device__ __forceinline__ i64 Ux(int nd, int fr) const { return S ? shadow[scell(nd, fr)] : U(nd, fr); }
  template <bool S> __device__ __forceinline__ void setUx(int nd, int fr, i64 v) const { if (S) shadow[scell(nd, fr)] = v; else setU(nd, fr, v); }
  __device__ __forceinline__ i64 Sub(int nd, int fr) const { return kSmem ? sub[nd * FR + fr] : D->subtree[(size_t)nd * FR + fr]; }
  __device__ __forceinline__ i64 LQ(int nd, int fr) const {
    return kSmem ? lq[nd * FR + fr] : local_quota(D->subtree[(size_t)nd * FR + fr], D->llimit[(size_t)nd * FR + fr]);
  }
  __device__ __forceinline__ i64 BL(int nd, int fr) const { return kSmem ? bl[nd * FR + fr] : D->blimit[(size_t)nd * FR + fr]; }
  __device__ __forceinline__ int parent(int nd) const { return kSmem ? lparent[nd] : D->parent[nd]; }
  __device__ __forceinline__ int handle(int node) const { return kSmem ? D->local_idx[node] : node; }
  // available() resource_node.go:104-118 along a staged path (path[0] = CQ ... path[plen-1] = root)
  // Global-table mode (trees too large for shared memory): every level of a walk costs an L2 round trip, so the
  // operands of ALL levels of the path (<= KB_PF) are requested first and the level-by-level arithmetic of
  // available() / addUsage / removeUsage then runs on registers — one memory latency per walk instead of one per level.
#define KB_PF 6
  template <bool S>
  __device__ __forceinline__ void prefetch(const int *path, int plen, int fr, i64 (&u)[KB_PF], i64 (&sb)[KB_PF], i64 (&ll)[KB_PF], i64 (&b)[KB_PF], bool want_bl) const {
#pragma unroll
    for (int k = 0; k < KB_PF; k++) {
      u[k] = sb[k] = 0; ll[k] = b[k] = KB_NO_LIMIT;
      if (k < plen) {
        size_t c = (size_t)path[k] * FR + fr;
        u[k] = S ? shadow[c] : __ldcg(&D->usage[c]);
        sb[k] = D->subtree[c]; ll[k] = D->llimit[c];
        if (want_bl) b[k] = D->blimit[c];
      }
    }
  }
  // available() on operands already in registers (plen <= KB_PF)
  __device__ __forceinline__ static i64 avail_from(const i64 (&u)[KB_PF], const i64 (&sb)[KB_PF], const i64 (&ll)[KB_PF], const i64 (&b)[KB_PF], int plen) {
    i64 a = 0;
#pragma unroll
    for (int k = KB_PF - 1; k >= 0; k--) {
      if (k >= plen) continue;
      if (k == plen - 1) { a = sb[k] - u[k]; continue; }
      i64 l = local_quota(sb[k], ll[k]);
      i64 pa = a;
      if (b[k] != KB_NO_LIMIT) pa = imin((sb[k] - l) - imax(0, u[k] - l) + b[k], pa);
      a = imax(0, l - u[k]) + pa;
    }
    return a;
  }
  // addUsage on operands already in registers (plen <= KB_PF): stores the new usage of the touched levels
  template <bool S>
  __device__ __forceinline__ void add_from(const int *path, int plen, int fr, const i64 (&u)[KB_PF], const i64 (&sb)[KB_PF], const i64 (&ll)[KB_PF], i64 val) const {
    bool go = true;
#pragma unroll
    for (int k = 0; k < KB_PF; k++) {
      if (k >= plen || !go) continue;
      i64 la = imax(0, local_quota(sb[k], ll[k]) - u[k]);
      setUx<S>(path[k], fr, u[k] + val);
      if (!(k + 1 < plen && val > la)) go = false;
      val -= la;
    }
  }
  template <bool S = false>
  __device__ inline i64 avail(const int *path, int plen, int fr) const {
    if constexpr (!kSmem) {
      if (plen <= KB_PF) {
        i64 u[KB_PF], sb[KB_PF], ll[KB_PF], b[KB_PF];
        prefetch<S>(path, plen, fr, u, sb, ll, b, true);
        return avail_from(u, sb, ll, b, plen);
      }
    }
    int rt = path[plen - 1];
    i64 a = Sub(rt, fr) - Ux<S>(rt, fr);
    for (int k = plen - 2; k >= 0; k--) {
      int nd = path[k];
      i64 u = Ux<S>(nd, fr), l = LQ(nd, fr), b = BL(nd, fr);
      i64 pa = a;
      if (b != KB_NO_LIMIT) pa = imin((Sub(nd, fr) - l) - imax(0, u - l) + b, pa);
      a = imax(0, l - u) + pa;
    }
    return a;
  }
  // addUsage :137-145 / removeUsage :149-158 along an explicit path (path[0] = the ClusterQueue)
  template <bool S = false>
  __device__ inline void add(const int *path, int plen, int fr, i64 val) const {
    if constexpr (!kSmem) {
      if (plen <= KB_PF) {
        i64 u[KB_PF], sb[KB_PF], ll[KB_PF], b[KB_PF];
        prefetch<S>(path, plen, fr, u, sb, ll, b, false);
        bool go = true;
#pragma unroll
        for (int k = 0; k < KB_PF; k++) {
          if (k >= plen || !go) continue;
          i64 la = imax(0, local_quota(sb[k], ll[k]) - u[k]);
          setUx<S>(path[k], fr, u[k] + val);
          if (!(k + 1 < plen && val > la)) go = false;
          val -= la;
        }
        return;
      }
    }
    for (int k = 0; k < plen; k++) {
      int nd = path[k];
      i64 u = Ux<S>(nd, fr);
      i64 la = imax(0, LQ(nd, fr) - u);
      setUx<S>(nd, fr, u + val);
      if (!(k + 1 < plen && val > la)) break;
      val -= la;
    }
  }
  template <bool S = false>
  __device__ inline void remove(const int *path, int plen, int fr, i64 val) const {
    if constexpr (!kSmem) {
      if (plen <= KB_PF) {
        i64 u[KB_PF], sb[KB_PF], ll[KB_PF], b[KB_PF];
        prefetch<S>(path, plen, fr, u, sb, ll, b, false);
        bool go = true;
#pragma unroll
        for (int k = 0; k < KB_PF; k++) {
          if (k >= plen || !go) continue;
          i64 stored = u[k] - local_quota(sb[k], ll[k]);
          setUx<S>(path[k], fr, u[k] - val);
          if (stored <= 0 || k + 1 >= plen) go = false;
          val = imin(val, stored);
        }
        return;
      }
    }
    for (int k = 0; k < plen; k++) {
      int nd = path[k];
      i64 u = Ux<S>(nd, fr), stored = u - LQ(nd, fr);
      setUx<S>(nd, fr, u - val);
      if (stored <= 0 || k + 1 >= plen) break;
      val = imin(val, stored);
    }
  }
  // the same starting from a node (an admitted workload's ClusterQueue): global-table mode reads the node's static
  // path (DevSnap::cq_path), shared-memory mode chases the staged parent handles
  template <bool S = false>
  __device__ inline void add_node(int nd, int fr, i64 val) const {
    if constexpr (!kSmem) add<S>(D->cq_path + (size_t)nd * D->path_stride, D->cq_plen[nd], fr, val);
    else
      while (true) {
        i64 u = Ux<S>(nd, fr), la = imax(0, LQ(nd, fr) - u);
        setUx<S>(nd, fr, u + val);
        int p = parent(nd);
        if (p < 0 || !(val > la)) break;
        val -= la; nd = p;
      }
  }
  template <bool S = false>
  __device__ inline void remove_node(int nd, int fr, i64 val) const {
    if constexpr (!kSmem) remove<S>(D->cq_path + (size_t)nd * D->path_stride, D->cq_plen[nd], fr, val);
    else
      while (true) {
        i64 u = Ux<S>(nd, fr), stored = u - LQ(nd, fr);
        setUx<S>(nd, fr, u - val);
        int p = parent(nd);
        if (stored <= 0 || p < 0) break;
        val = imin(val, stored); nd = p;
      }
  }
};

// Stage the tables of the root's nodes (all threads of the CTA).
template <bool kSmem>
__device__ inline unsigned char *stage_tables(const DevSnap &D, Tab<kSmem> &T, unsigned char *p, const int32_t *nodes, int nn) {
  const int FR = D.FR;
  T.D = &D; T.FR = FR;
  T.shadow = D.usage_shadow; T.tnodes = nodes; T.tnn = nn; T.shadow_on = nullptr;
  if (kSmem) {
    size_t tb = (size_t)nn * FR;
    i64 *u = (i64 *)p, *sb = u + tb, *lq = sb + tb, *bl = lq + tb;
    int *lp = (int *)(bl + tb);
#pragma unroll 4
    for (int i = threadIdx.x; i < nn * FR; i += blockDim.x) {
      int nd = nodes[i / FR], fr = i % FR;
      size_t c = (size_t)nd * FR + fr;
      i64 sub = D.subtree[c];
      u[i] = D.usage[c]; sb[i] = sub; lq[i] = local_quota(sub, D.llimit[c]); bl[i] = D.blimit[c];
    }
    for (int i = threadIdx.x; i < nn; i += blockDim.x) { int pn = D.parent[nodes[i]]; lp[i] = pn < 0 ? -1 : D.local_idx[pn]; }
    T.usage = u; T.sub = sb; T.lq = lq; T.bl = bl; T.lparent = lp;
    p = (unsigned char *)(lp + nn);
    p = (unsigned char *)(((uintptr_t)p + 7) & ~(uintptr_t)7);
  }
  return p;
}
template <bool kSmem>
__device__ inline void publish_usage(const DevSnap &D, const Tab<kSmem> &T, const int32_t *nodes, int nn) {
  if (kSmem)
    for (int i = threadIdx.x; i < nn * D.FR; i += blockDim.x) D.usage[(size_t)nodes[i / D.FR] * D.FR + i % D.FR] = T.usage[i];
}

// One iteration of the admit loop body (scheduler.go:269-401) for entry e, executed by a
// full warp: lane l owns the flavor-resource columns l, l+32, ...  qrow[fr] is the
// aggregated Assignment.Usage.Quota (absent cell = -1).  s_path: KB_MAX_DEPTH+2 ints.
// cq = global id of the entry's ClusterQueue, ntg/toff = its preemption targets in the pool.
// T.shadow_on points at a shared-memory flag (0 at kernel start).
// Global-table mode (trees too large for shared memory): while warp 0 commits one group of KB_SUB entries, the other
// warps stage everything of the NEXT group that does not depend on earlier commits — per entry the ids of its
// preemption targets and their usage cells (quantity, column, ClusterQueue), counting-sorted by column.  Columns are
// independent, so in the commit every lane walks the cells of ITS columns in target order and the lanes' walks
// overlap: the commit warp only ever waits for the usage / shadow values themselves.
struct TgCell { i64 qty; int32_t lh; int16_t fr; int16_t pad; };  // lh: local handle of the target's ClusterQueue
#define KB_SUB 7        // entries per group = staging warps (KB_ADMIT_THREADS / 32 - 1)
#define KB_ECAP 256     // staged cells per entry
#define KB_TCAP 256     // staged targets per entry
struct StagedEntry {
  const TgCell *cells;        // [ncell] sorted by column (fr & 31), target order inside a column
  const uint16_t *col_start;  // [33]
  const int32_t *adm;         // [ntg] target ids
  const int32_t *cq_path;     // [nn][KB_PF] paths of the root's ClusterQueues by local handle (shared memory)
  const int8_t *cq_plen;      // [nn]
};
template <bool kSmem>
__device__ inline void commit_entry(const DevSnap &D, const Tab<kSmem> &T, int *s_path, int lane, int e, int nd, int mode,
                                    int borrowing, const i64 *qrow, int rank, int cq, int ntg, int toff,
                                    const StagedEntry *st = nullptr) {
  const int FR = D.FR;
  if (lane == 0) D.rank[e] = rank;
  if (mode == KB_MODE_NOFIT) { if (lane == 0) D.decision[e] = KB_DEC_NOFIT; return; }
  if (st) {  // path table of the root in shared memory
    const int lh = D.local_idx[nd], pl = st->cq_plen[lh];
    if (lane < pl) s_path[lane] = st->cq_path[lh * KB_PF + lane];
    if (lane == 0) s_path[KB_MAX_DEPTH + 1] = pl;
  } else if constexpr (!kSmem) {  // static path table: one coalesced row instead of a chain of dependent parent loads
    int pl = D.cq_plen[nd];
    if (lane < pl) s_path[lane] = D.cq_path[(size_t)nd * D.path_stride + lane];
    if (lane == 0) s_path[KB_MAX_DEPTH + 1] = pl;
  } else {
    if (lane == 0) { int pl = 0; for (int t = nd; t >= 0; t = T.parent(t)) s_path[pl++] = t; s_path[KB_MAX_DEPTH + 1] = pl; }
  }
  __syncwarp();
  int plen = s_path[KB_MAX_DEPTH + 1];
  bool shadow = *T.shadow_on != 0;
  if (mode == KB_MODE_PREEMPT && ntg == 0) {  // Preempt without targets: scheduler.go:303-318
    if (lane == 0) D.decision[e] = KB_DEC_PREEMPT_NO_TARGETS;
    if (D.cq_reclaim_within[cq] != KB_POLICY_ANY) {  // !CanAlwaysReclaim policy.go:27-29
      for (int fr = lane; fr < FR; fr += 32) {        // quotaResourcesToReserve :530-548
        i64 u = qrow[fr];
        if (u < 0) continue;
        i64 nominal = T.Sub(nd, fr), bl = T.BL(nd, fr), cur = T.U(nd, fr);  // CQ: SubtreeQuota == Nominal
        i64 rsv;
        if (borrowing > 0) rsv = bl == KB_NO_LIMIT ? u : imin(u, nominal + bl - cur);
        else rsv = imax(0, imin(u, nominal - cur));
        T.add(s_path, plen, fr, rsv);
        if (shadow) T.template add<true>(s_path, plen, fr, rsv);
      }
    }
    __syncwarp();
    return;
  }
  // entries with preemption targets: overlap check (:321-325); fits() sees the usage without every
  // workload preempted so far in this root and without the new targets (:503-511) = the shadow table
  if (ntg > 0) {
    bool overlap = false;
    if (st) { for (int k = lane; k < ntg; k += 32) if (D.preempted[st->adm[k]]) overlap = true; }
    else for (int k = lane; k < ntg; k += 32) if (D.preempted[D.tgt_pool_adm[toff + k]]) overlap = true;
    if (__any_sync(0xffffffffu, overlap)) { if (lane == 0) D.decision[e] = KB_DEC_SKIPPED_OVERLAP; __syncwarp(); return; }
    if (!shadow) {  // first targets of this root: the shadow starts as a copy of the current usage
      for (int i = lane; i < T.tnn * FR; i += 32) { int h = kSmem ? i / FR : T.tnodes[i / FR]; T.shadow[T.scell(h, i % FR)] = T.U(h, i % FR); }
      __syncwarp();
      if (lane == 0) *T.shadow_on = 1;
      shadow = true;
      __syncwarp();
    }
  }
  auto apply = [&](int a, bool remove) {  // one admitted workload on the shadow: its cells are distinct columns -> one lane each
    int nd2 = T.handle(D.adm_cq[a]);
    for (int k = D.adm_use_start[a] + lane; k < D.adm_use_start[a + 1]; k += 32) {
      if (remove) T.template remove_node<true>(nd2, D.adm_use_fr[k], D.adm_use_qty[k]);
      else T.template add_node<true>(nd2, D.adm_use_fr[k], D.adm_use_qty[k]);
    }
    __syncwarp();
  };
  auto apply_cells = [&](bool remove) {  // staged cells: lane l walks the cells of columns l, l+32, ... in target order
    if constexpr (!kSmem) {
      const int j1 = st->col_start[lane + 1];
      for (int j = st->col_start[lane]; j < j1; j++) {
        const TgCell c = st->cells[j];
        const int32_t *cp = st->cq_path + c.lh * KB_PF;
        const int pl = st->cq_plen[c.lh];
        if (remove) T.template remove<true>(cp, pl, c.fr, c.qty);
        else T.template add<true>(cp, pl, c.fr, c.qty);
      }
      __syncwarp();
    }
  };
  if (st) apply_cells(true);
  else for (int k = 0; k < ntg; k++) apply(D.tgt_pool_adm[toff + k], true);  // SimulateWorkloadRemoval snapshot.go:67-84
  bool ok = true;  // fits :503-511
  bool fused = false;
  if constexpr (!kSmem) {
    if (FR <= 32 && plen <= KB_PF) {  // one column per lane: fits() and AddUsage share one load of the path's operands
      fused = true;
      const int fr = lane;
      const i64 q = lane < FR ? qrow[fr] : -1;
      i64 um[KB_PF], us[KB_PF], sb[KB_PF], ll[KB_PF], b[KB_PF];
      if (q > 0) {
        T.template prefetch<false>(s_path, plen, fr, um, sb, ll, b, true);
        if (shadow) {
#pragma unroll
          for (int k = 0; k < KB_PF; k++) us[k] = k < plen ? T.shadow[(size_t)s_path[k] * FR + fr] : 0;
          if (imax(0, Tab<kSmem>::avail_from(us, sb, ll, b, plen)) < q) ok = false;
        } else if (imax(0, Tab<kSmem>::avail_from(um, sb, ll, b, plen)) < q) ok = false;
      }
      ok = __all_sync(0xffffffffu, ok);
      if (ok) {
        if (st) { for (int k = lane; k < ntg; k += 32) D.preempted[st->adm[k]] = 1; }
        else for (int k = lane; k < ntg; k += 32) D.preempted[D.tgt_pool_adm[toff + k]] = 1;  // preemptedWorkloads.Insert :335
        if (q > 0) {  // cq.AddUsage :336
          T.template add_from<false>(s_path, plen, fr, um, sb, ll, q);
          if (shadow) T.template add_from<true>(s_path, plen, fr, us, sb, ll, q);
        }
      }
    }
  }
  if (!fused) {
    for (int fr = lane; fr < FR; fr += 32) {
      i64 q = qrow[fr];
      if (q > 0 && imax(0, shadow ? T.template avail<true>(s_path, plen, fr) : T.avail(s_path, plen, fr)) < q) ok = false;
    }
    ok = __all_sync(0xffffffffu, ok);
    if (ok) {
      for (int k = lane; k < ntg; k += 32) D.preempted[D.tgt_pool_adm[toff + k]] = 1;  // preemptedWorkloads.Insert :335 (stay removed in the shadow)
      for (int fr = lane; fr < FR; fr += 32) {  // cq.AddUsage :336
        i64 q = qrow[fr];
        if (q > 0) { T.add(s_path, plen, fr, q); if (shadow) T.template add<true>(s_path, plen, fr, q); }
      }
    }
  }
  if (!ok) {
    if (st) apply_cells(false);
    else for (int k = 0; k < ntg; k++) apply(D.tgt_pool_adm[toff + k], false);
  }
  if (lane == 0) D.decision[e] = ok ? (mode == KB_MODE_PREEMPT ? KB_DEC_PREEMPTING : KB_DEC_ASSUMED) : KB_DEC_SKIPPED_NO_FIT;
  __syncwarp();
}

// Commit loop of one tile for a FLAT cohort tree staged in shared memory (node 0 = root cohort, every other node a
// ClusterQueue whose parent is the root).  Lane l owns columns l and l+32; the root's usage and SubtreeQuota of
// those columns stay in registers for the whole tile, and the operands of entry i+1 that do not depend on earlier
// commits (request row, localQuota, BorrowingLimit, nominal quota of its ClusterQueue) are loaded while entry i
// is being decided, so the dependent chain per entry is one shared-memory load of the ClusterQueue's usage, the
// available() arithmetic (resource_node.go:104-118 for a two-node path), one vote, and the addUsage stores.
// Entries in Preempt mode, with targets, or after the shadow table went live take the generic commit_entry.
template <bool kTwo>  // kTwo: FR > 32, the lane also owns column lane + 32
__device__ inline void commit_tile_flat(const DevSnap &D, const Tab<true> &T, int *s_path, int lane, int tn, int base, const i64 *s_q,
                                        const int *t_e, const int *t_node, int *t_mode, const int *t_borrow,
                                        const int *t_cq, const int *t_ntg, const int *t_toff) {
  const int FR = D.FR;
  const int fr0 = lane, fr1 = lane + 32;
  const bool c0 = fr0 < FR, c1 = kTwo && fr1 < FR;
  i64 urt0 = c0 ? T.usage[fr0] : 0, urt1 = c1 ? T.usage[fr1] : 0;
  const i64 srt0 = c0 ? T.sub[fr0] : 0, srt1 = c1 ? T.sub[fr1] : 0;
  // Per entry and column, everything of available() that does not involve the ROOT's usage is evaluated when the
  // entry is prefetched: A = LocalAvailable of the ClusterQueue, cap = its borrowing cap
  // (storedInParent - usedInParent + BorrowingLimit, resource_node.go:111-116).  The chain from one entry to the
  // next is then  pa = min(SubtreeQuota_root - usage_root, cap); fits = A + pa >= q; usage_root += q - A.
  // Decisions go to t_mode[i] (KB_DEC_* | 0x100) and are flushed to global memory by the whole CTA after the tile.
  struct Ops { int nd, mode, ntg; i64 q0, q1, u0, u1, A0, A1, cap0, cap1; };
  auto prep = [&](Ops &o) {  // reads the ClusterQueue's current usage
    o.u0 = o.A0 = 0; o.cap0 = INT64_MAX;
    if (o.q0 > 0) {
      int r = o.nd * FR + fr0;
      i64 u = T.usage[r], l = T.lq[r], bl = T.bl[r];
      o.u0 = u; o.A0 = imax(0, l - u);
      if (bl != KB_NO_LIMIT) o.cap0 = (T.sub[r] - l) - imax(0, u - l) + bl;
    }
    if (kTwo) {
      o.u1 = o.A1 = 0; o.cap1 = INT64_MAX;
      if (o.q1 > 0) {
        int r = o.nd * FR + fr1;
        i64 u = T.usage[r], l = T.lq[r], bl = T.bl[r];
        o.u1 = u; o.A1 = imax(0, l - u);
        if (bl != KB_NO_LIMIT) o.cap1 = (T.sub[r] - l) - imax(0, u - l) + bl;
      }
    }
  };
  auto load = [&](int i, Ops &o) {
    o.nd = t_node[i]; o.mode = t_mode[i]; o.ntg = t_ntg[i];
    o.q0 = c0 ? s_q[(size_t)i * FR + fr0] : -1;
    if (kTwo) o.q1 = c1 ? s_q[(size_t)i * FR + fr1] : -1;
    prep(o);
  };
  int prev_nd = -1;  // ClusterQueue whose usage row the previous entry may have written after this one was prefetched
  bool shadow = *T.shadow_on != 0;
  auto step = [&](int i, Ops &cur) {
    if (cur.mode == KB_MODE_NOFIT) {
      if (lane == 0) t_mode[i] = KB_DEC_NOFIT | 0x100;
      prev_nd = -1;
    } else if (cur.mode == KB_MODE_PREEMPT || cur.ntg > 0 || shadow) {
      if (c0) T.usage[fr0] = urt0;
      if (c1) T.usage[fr1] = urt1;
      __syncwarp();
      commit_entry<true>(D, T, s_path, lane, t_e[i], cur.nd, cur.mode, t_borrow[i], s_q + (size_t)i * FR, base + i, t_cq[i], cur.ntg, t_toff[i]);
      if (lane == 0) t_mode[i] = -1;  // rank and decision already written
      __syncwarp();
      if (c0) urt0 = T.usage[fr0];
      if (c1) urt1 = T.usage[fr1];
      shadow = *T.shadow_on != 0;
      prev_nd = cur.nd;
    } else {
      if (cur.nd == prev_nd) prep(cur);  // same ClusterQueue as the entry before: its usage row changed after the prefetch
      bool ok = !(cur.q0 > 0 && imax(0, cur.A0 + imin(srt0 - urt0, cur.cap0)) < cur.q0);
      if (kTwo) ok = ok && !(cur.q1 > 0 && imax(0, cur.A1 + imin(srt1 - urt1, cur.cap1)) < cur.q1);
      ok = __all_sync(0xffffffffu, ok);
      if (ok) {  // addUsage resource_node.go:137-145: the part above the ClusterQueue's local availability goes to the root
        if (cur.q0 > 0) { T.usage[cur.nd * FR + fr0] = cur.u0 + cur.q0; if (cur.q0 > cur.A0) urt0 += cur.q0 - cur.A0; }
        if (kTwo) if (cur.q1 > 0) { T.usage[cur.nd * FR + fr1] = cur.u1 + cur.q1; if (cur.q1 > cur.A1) urt1 += cur.q1 - cur.A1; }
      }
      if (lane == 0) t_mode[i] = (ok ? KB_DEC_ASSUMED : KB_DEC_SKIPPED_NO_FIT) | 0x100;
      prev_nd = ok ? cur.nd : -1;
    }
  };
  Ops a, b;  // ping-pong: one is being decided while the other is prefetched
  load(0, a);
  int i = 0;
  for (; i + 1 < tn; i += 2) {
    load(i + 1, b);
    step(i, a);
    if (i + 2 < tn) load(i + 2, a);
    step(i + 1, b);
  }
  if (i < tn) step(i, a);
  if (c0) T.usage[fr0] = urt0;
  if (c1) T.usage[fr1] = urt1;
  __syncwarp();
}

// dense request row of entry e for column fr (absent = -1)
__device__ __forceinline__ i64 entry_request(const DevSnap &D, int e, int fr) {
  const int R = D.R;
  int f = fr / R, r = fr % R;
  int wl = D.heads[e];
  int cq = D.wl_cq[wl];
  bool covers_pods = D.pods_res >= 0 && rg_by_resource(D, cq, D.pods_res) >= 0;
  i64 q = -1;
  for (int row = D.wl_ps_start[wl]; row < D.wl_ps_start[wl + 1]; row++)
    if (D.ps_flavor[(size_t)row * R + r] == f) q = (q < 0 ? 0 : q) + ps_request(D, row, r, D.ps_count_out[row], covers_pods);
  return q;
}

// scatter the aggregated Assignment.Usage.Quota of entry e into a dense row (pre-filled with -1)
__device__ inline void expand_entry(const DevSnap &D, int e, i64 *qrow) {
  const int R = D.R;
  int wl = D.heads[e];
  int ps0 = D.wl_ps_start[wl], ps1 = D.wl_ps_start[wl + 1];
  int cq = D.wl_cq[wl];
  bool covers_pods = D.pods_res >= 0 && rg_by_resource(D, cq, D.pods_res) >= 0;
  for (int row = ps0; row < ps1; row++) {
    int cnt = D.ps_count_out[row];
    for (int r = 0; r < R; r++) {
      int f = D.ps_flavor[(size_t)row * R + r];
      if (f < 0) continue;
      i64 cur = qrow[f * R + r];
      qrow[f * R + r] = (cur < 0 ? 0 : cur) + ps_request(D, row, r, cnt, covers_pods);
    }
  }
}

template <bool kSmemTables>
__global__ void __launch_bounds__(KB_ADMIT_THREADS) k_admit(DevSnap D, int slot_base, int sort_cap, int stage_buffers) {
  extern __shared__ __align__(16) unsigned char smem_raw[];
  const int FR = D.FR;
#ifdef KB_ADMIT_PROBE
  const long long kp0 = clock64();
#endif
  int slot = slot_base + blockIdx.x;
  int off = D.root_offset[slot];
  int n = D.root_offset[slot + 1] - off;
  if (n == 0) return;
  int32_t *ent = D.root_entries + off;
  if (slot < D.nLone && D.lone_fast && n <= KB_RANK_CAP) return;  // handled by k_admit_lone
  if (slot >= D.nLone && (D.flags & KB_F_FAIR_SHARING) && !D.tree_flat[slot - D.nLone]) return;  // tournament kernel
  const int32_t *nodes; int nn;
  if (slot < D.nLone) { nodes = &D.lone_cqs[slot]; nn = 1; }
  else { int t = slot - D.nLone; nodes = D.tree_nodes + D.tree_start[t]; nn = D.tree_start[t + 1] - D.tree_start[t]; }
  // ---- smem carve-up: [tables][sort keys | request tile][tile meta][path] ----
  Tab<kSmemTables> T;
  unsigned char *p = stage_tables<kSmemTables>(D, T, smem_raw, nodes, nn);
  i64 *s_q = (i64 *)p;
  p += (size_t)KB_TILE * FR * 8;
  (void)sort_cap;
  p = (unsigned char *)(((uintptr_t)p + 7) & ~(uintptr_t)7);
  int *t_e = (int *)p, *t_node = t_e + KB_TILE, *t_mode = t_node + KB_TILE, *t_borrow = t_mode + KB_TILE;
  int *t_cq = t_borrow + KB_TILE, *t_ntg = t_cq + KB_TILE, *t_toff = t_ntg + KB_TILE;
  int *s_path = t_toff + KB_TILE;
  int *s_shadow_on = s_path + KB_MAX_DEPTH + 2;
  if (threadIdx.x == 0) *s_shadow_on = 0;
  T.shadow_on = s_shadow_on;
  // global-table mode: staging buffers of the commit pipeline (commit_entry / StagedEntry)
  const bool stage_cells = !kSmemTables && stage_buffers && D.path_stride <= KB_PF && nn <= 32767;  // stage_buffers: the launch provided the shared memory
  int32_t *s_cqpath = nullptr, *s_tadm = nullptr, *s_pref = nullptr, *s_run = nullptr; int8_t *s_cqplen = nullptr, *s_staged = nullptr;
  TgCell *s_cells = nullptr; uint16_t *s_cs = nullptr;
  if (stage_cells) {
    unsigned char *q = (unsigned char *)(((uintptr_t)(s_shadow_on + 2) + 15) & ~(uintptr_t)15);
    s_cells = (TgCell *)q; q += sizeof(TgCell) * 2 * KB_SUB * KB_ECAP;           // [2][KB_SUB][KB_ECAP]
    s_cqpath = (int32_t *)q; q += sizeof(int32_t) * (size_t)nn * KB_PF;           // [nn][KB_PF]
    s_tadm = (int32_t *)q; q += sizeof(int32_t) * 2 * KB_SUB * KB_TCAP;           // [2][KB_SUB][KB_TCAP]
    s_pref = (int32_t *)q; q += sizeof(int32_t) * KB_SUB * (KB_TCAP + 1);         // per staging warp: cells before target k
    s_run = (int32_t *)q; q += sizeof(int32_t) * KB_SUB * 32;                     // per staging warp: per-column cursors
    s_cs = (uint16_t *)q; q += sizeof(uint16_t) * 2 * KB_SUB * 34;                // [2][KB_SUB][33] column offsets
    s_cqplen = (int8_t *)q; q += (size_t)nn;                                      // [nn]
    s_staged = (int8_t *)q;                                                       // [2][KB_SUB]
    for (int i = threadIdx.x; i < nn; i += blockDim.x) {
      int nd = nodes[i];
      int pl = nd < D.Q ? D.cq_plen[nd] : 0;
      s_cqplen[i] = (int8_t)pl;
      for (int k = 0; k < pl; k++) s_cqpath[i * KB_PF + k] = D.cq_path[(size_t)nd * D.path_stride + k];
    }
  }
  // One warp stages one entry: target ids, then the targets' usage cells counting-sorted by column (stable: the cells
  // of a column keep target order).  slot = position of the entry inside its group, b = buffer of the group.
  auto stage_entry = [&](int b, int slot, int ntg, int toff, int sw) {
    const int ln = threadIdx.x & 31;
    int32_t *tadm = s_tadm + ((size_t)b * KB_SUB + slot) * KB_TCAP;
    int32_t *pref = s_pref + (size_t)sw * (KB_TCAP + 1), *run = s_run + sw * 32;
    TgCell *cells = s_cells + ((size_t)b * KB_SUB + slot) * KB_ECAP;
    uint16_t *cs = s_cs + ((size_t)b * KB_SUB + slot) * 34;
    bool ok = ntg <= KB_TCAP;
    int total = 0;
    run[ln] = 0;
    __syncwarp();
    if (ok) {
      for (int k0 = 0; k0 < ntg; k0 += 32) {  // targets: ids, cell counts (prefix), histogram of columns
        int k = k0 + ln, cnt = 0, a = -1, u0 = 0;
        if (k < ntg) { a = D.tgt_pool_adm[toff + k]; u0 = D.adm_use_start[a]; cnt = D.adm_use_start[a + 1] - u0; tadm[k] = a; }
        int inc = cnt;
        for (int o = 1; o < 32; o <<= 1) { int v = __shfl_up_sync(0xffffffffu, inc, o); if (ln >= o) inc += v; }
        if (k < ntg) pref[k] = total + inc - cnt;
        total += __shfl_sync(0xffffffffu, inc, 31);
        for (int j = 0; j < cnt; j++) atomicAdd(&run[D.adm_use_fr[u0 + j] & 31], 1);
      }
      if (ln == 0) pref[ntg] = total;
      ok = total <= KB_ECAP;
    }
    __syncwarp();
    if (ok) {
      int h = run[ln], inc = h;
      for (int o = 1; o < 32; o <<= 1) { int v = __shfl_up_sync(0xffffffffu, inc, o); if (ln >= o) inc += v; }
      __syncwarp();
      run[ln] = inc - h;                     // first free position of column ln
      cs[ln] = (uint16_t)(inc - h);
      if (ln == 31) cs[32] = (uint16_t)inc;
      __syncwarp();
      for (int c0 = 0; c0 < total; c0 += 32) {  // cells in (target, cell) order, 32 at a time
        int c = c0 + ln, col = 32 + ln;
        TgCell cell; cell.qty = 0; cell.lh = 0; cell.fr = 0; cell.pad = 0;
        if (c < total) {
          int lo = 0, hi = ntg;                // last target k with pref[k] <= c
          while (hi - lo > 1) { int mid = (lo + hi) >> 1; if (pref[mid] <= c) lo = mid; else hi = mid; }
          int a = tadm[lo], u = D.adm_use_start[a] + (c - pref[lo]);
          cell.qty = D.adm_use_qty[u]; cell.fr = (int16_t)D.adm_use_fr[u]; cell.lh = D.local_idx[D.adm_cq[a]];
          col = cell.fr & 31;
        }
        unsigned m = __match_any_sync(0xffffffffu, col);
        if (c < total) cells[run[col] + __popc(m & ((1u << ln) - 1u))] = cell;
        __syncwarp();
        if (c < total && (m & ((1u << ln) - 1u)) == 0) run[col] += __popc(m);
        __syncwarp();
      }
    }
    if (ln == 0) s_staged[b * KB_SUB + slot] = ok ? 1 : 0;
  };
  // ---- 1. iterator order: k_rank already produced it for roots up to KB_RANK_CAP entries; larger roots sort here
  //         with an ascending-only bitonic network over the global index array (virtual +inf padding never moves).
  if (n <= KB_RANK_CAP) ent = D.sorted + off;
  else {
    int np2 = 1;
    while (np2 < n) np2 <<= 1;
    auto ce = [&](int i, int l) {  // compare-exchange, minimum to the lower index
      int a = ent[i], b = ent[l];
      if (key4_less(D.ekey + (size_t)b * 4, D.ekey + (size_t)a * 4)) { ent[i] = b; ent[l] = a; }
    };
    for (int k = 2; k <= np2; k <<= 1) {
      for (int i = threadIdx.x; i < n; i += blockDim.x) { int l = i ^ (k - 1); if (l > i && l < n) ce(i, l); }
      __syncthreads();
      for (int j = k >> 2; j > 0; j >>= 1) {
        for (int i = threadIdx.x; i < n; i += blockDim.x) { int l = i ^ j; if (l > i && l < n) ce(i, l); }
        __syncthreads();
      }
    }
  }
  __syncthreads();
  if constexpr (!kSmemTables) {
    // Large tree: if any entry of the root carries preemption targets the shadow table (usage without the workloads
    // preempted so far, commit_entry) will be needed — the whole CTA copies it now instead of warp 0 inside the loop.
    int any = 0;
    for (int i = threadIdx.x; i < n; i += blockDim.x) any |= D.tgt_cnt[ent[i]] > 0;
    if (__syncthreads_or(any)) {
      for (int i = threadIdx.x; i < nn * FR; i += blockDim.x) { size_t c = (size_t)nodes[i / FR] * FR + i % FR; D.usage_shadow[c] = __ldcg(&D.usage[c]); }
      if (threadIdx.x == 0) *s_shadow_on = 1;
    }
    __syncthreads();
  }
  // ---- 2. tiles: expand (all threads), commit (warp 0) ----
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  // flat cohort (every ClusterQueue directly under the root), tables in shared memory, at most two columns per lane
  const bool flat = kSmemTables && FR <= 64 && slot >= D.nLone && D.tree_flat[slot - D.nLone];
  for (int base = 0; base < n; base += KB_TILE) {
    int tn = min(KB_TILE, n - base);
    for (int i = threadIdx.x; i < tn; i += blockDim.x) {
      int e = ent[base + i];
      int cqn = D.wl_cq[D.heads[e]];
      t_e[i] = e; t_node[i] = T.handle(cqn); t_cq[i] = cqn;
      t_mode[i] = D.mode[e]; t_borrow[i] = D.borrow[e]; t_ntg[i] = D.tgt_cnt[e]; t_toff[i] = D.tgt_off[e];
    }
    for (int c = threadIdx.x; c < tn * FR; c += blockDim.x) s_q[c] = -1;
    __syncthreads();
    // one thread per entry walks its podset rows once and scatters the cells of its row
    for (int i = threadIdx.x; i < tn; i += blockDim.x) expand_entry(D, t_e[i], s_q + (size_t)i * FR);
    __syncthreads();
    if (stage_cells) {
      // groups of KB_SUB entries: warp 0 commits group j while warps 1..KB_SUB stage group j + 1
      const int ngrp = (tn + KB_SUB - 1) / KB_SUB;
#ifdef KB_ADMIT_PROBE
#define AP(k, v) do { if (blockIdx.x == 0 && threadIdx.x == 0) atomicAdd(&D.sstat[k], (u64)(v)); } while (0)
      long long ap0 = clock64();
#else
#define AP(k, v) do { } while (0)
#endif
      if (warp >= 1 && warp <= KB_SUB) { int i = warp - 1; if (i < tn) stage_entry(0, i, t_ntg[i], t_toff[i], warp - 1); }
      __syncthreads();
#ifdef KB_ADMIT_PROBE
      AP(0, clock64() - ap0);  // first group staging (exposed)
#endif
      for (int j = 0; j < ngrp; j++) {
        const int b = j & 1, i0 = j * KB_SUB, i1 = min(tn, i0 + KB_SUB);
#ifdef KB_ADMIT_PROBE
        long long ap1 = clock64();
#endif
        if (warp == 0) {
          for (int i = i0; i < i1; i++) {
#ifdef KB_ADMIT_PROBE
            AP(2, 1); AP(3, s_staged[b * KB_SUB + (i - i0)] ? 1 : 0); AP(4, t_ntg[i]); AP(5, s_staged[b * KB_SUB + (i - i0)] ? (s_cs + ((size_t)b * KB_SUB + (i - i0)) * 34)[32] : 0);
#endif
            StagedEntry st;
            const int slot = i - i0;
            st.cells = s_cells + ((size_t)b * KB_SUB + slot) * KB_ECAP; st.col_start = s_cs + ((size_t)b * KB_SUB + slot) * 34;
            st.adm = s_tadm + ((size_t)b * KB_SUB + slot) * KB_TCAP; st.cq_path = s_cqpath; st.cq_plen = s_cqplen;
            commit_entry<kSmemTables>(D, T, s_path, lane, t_e[i], t_node[i], t_mode[i], t_borrow[i], s_q + (size_t)i * FR, base + i,
                                      t_cq[i], t_ntg[i], t_toff[i], s_staged[b * KB_SUB + slot] ? &st : nullptr);
          }
        } else if (warp <= KB_SUB) {
          int i = i1 + warp - 1;
          if (i < tn) stage_entry(b ^ 1, warp - 1, t_ntg[i], t_toff[i], warp - 1);
        }
#ifdef KB_ADMIT_PROBE
        long long ap2 = clock64();
        AP(1, ap2 - ap1);  // commit time of the group (warp 0)
#endif
        __syncthreads();
#ifdef KB_ADMIT_PROBE
        AP(6, clock64() - ap2);  // warp 0 waiting for the stagers
#endif
      }
    } else if (warp == 0) {
      if constexpr (kSmemTables) {
        if (flat) {
          if (FR > 32) commit_tile_flat<true>(D, T, s_path, lane, tn, base, s_q, t_e, t_node, t_mode, t_borrow, t_cq, t_ntg, t_toff);
          else commit_tile_flat<false>(D, T, s_path, lane, tn, base, s_q, t_e, t_node, t_mode, t_borrow, t_cq, t_ntg, t_toff);
        }
      }
      if (!flat)
        for (int i = 0; i < tn; i++)
          commit_entry<kSmemTables>(D, T, s_path, lane, t_e[i], t_node[i], t_mode[i], t_borrow[i], s_q + (size_t)i * FR, base + i,
                                    t_cq[i], t_ntg[i], t_toff[i]);
    }
    __syncthreads();
    if (flat) {  // decisions of the flat commit loop (t_mode[i] = KB_DEC_* | 0x100), written by the whole CTA
      for (int i = threadIdx.x; i < tn; i += blockDim.x) {
        int m = t_mode[i];
        if (m >= 0x100) { D.decision[t_e[i]] = (uint8_t)(m & 0xff); D.rank[t_e[i]] = base + i; }
      }
      __syncthreads();
    }
  }
  publish_usage<kSmemTables>(D, T, nodes, nn);
#ifdef KB_ADMIT_PROBE
  if (threadIdx.x == 0) {
    long long tg = 0; int big = 0;
    for (int i = 0; i < n; i++) { int e = ent[i]; tg += D.tgt_cnt[e]; if (D.tgt_cnt[e] > 100) big++; }
    printf("k_admit root %d: nn %d entries %d targets %lld entries>100tg %d cycles %lld\n", slot, nn, n, tg, big, clock64() - kp0);
  }
#endif
}

// ---------------------------------------------------------------------------
// Fused cycle, one CTA per root cohort (k_cycle_root): tree pass -> nominate -> iterator order -> admit loop with
// the root's quota tables in shared memory from the first load to the last store.  Root cohorts are independent
// coupling domains (resource_node.go:106-108), so the whole cycle of one root needs no other CTA: the node tables
// leave HBM once (nominal / limits / ClusterQueue usage in, final usage out) instead of once per kernel of the chain
// k_tree -> k_nominate -> k_fair_prep -> k_scan_roots -> k_scatter -> k_rank -> k_admit.
// Used when no entry can need a target search (no admitted workloads), every ClusterQueue has a cohort and at most
// one head, the tables of the largest tree fit shared memory, and fair sharing only meets flat cohorts.
// All node tables are indexed by the local handle (DevSnap::tab_local).
// ---------------------------------------------------------------------------
#ifndef KB_ROOT_THREADS
#define KB_ROOT_THREADS 1024
#endif
__global__ void __launch_bounds__(KB_ROOT_THREADS) k_cycle_root(DevSnap D) {
  extern __shared__ __align__(16) unsigned char smem_raw[];
  const int FR = D.FR, R = D.R, Fn = D.F;
  // index -> (row, column): FR is a power of two in every configuration at hand; the shift form saves a ~20-instruction
  // integer division per cell in the phases below (uniform branch)
  const int fr_sh = 31 - __clz(FR); const bool fr_p2 = (1 << fr_sh) == FR;
  auto row_of = [&](int i) { return fr_p2 ? i >> fr_sh : i / FR; };
  auto col_of = [&](int i) { return fr_p2 ? i & (FR - 1) : i % FR; };
  const int t = blockIdx.x;
  long long tk0 = clock64();
#define KB_PHASE(k) do { if (blockIdx.x == 0 && threadIdx.x == 0) { long long now = clock64(); D.sstat[k] = (u64)(now - tk0); tk0 = now; } } while (0)
  const int32_t *nodes = D.tree_nodes + D.tree_start[t];
  const int nn = D.tree_start[t + 1] - D.tree_start[t];
  const int32_t *lvl = D.tree_level + (size_t)t * KB_LEVELS;
  int nlev = 0;
  while (nlev + 1 < KB_LEVELS && lvl[nlev + 1] > lvl[nlev]) nlev++;
  const size_t tb = (size_t)nn * FR;
  // ---- shared memory: [usage][sub][lq][bl][avail | request tile][potential][fs_over][fs_lend][parent][height][entries...]
  i64 *s_u = (i64 *)smem_raw, *s_sub = s_u + tb, *s_lq = s_sub + tb, *s_bl = s_lq + tb, *s_av = s_bl + tb, *s_pot = s_av + tb;
  i64 *s_over = s_pot + tb, *s_lend = s_over + (size_t)nn * R;
  int *s_par = (int *)(s_lend + (size_t)nn * R), *s_hgt = s_par + nn;
  int *s_ent = s_hgt + nn;           // [nn] entries of the root in ClusterQueue order
  int *s_sorted = s_ent + nn;        // [nn] entries in iterator order
  int *t_e = s_sorted + nn, *t_node = t_e + KB_TILE, *t_mode = t_node + KB_TILE, *t_borrow = t_mode + KB_TILE;
  int *t_cq = t_borrow + KB_TILE, *t_ntg = t_cq + KB_TILE, *t_toff = t_ntg + KB_TILE;
  int *s_path = t_toff + KB_TILE;
  int *s_misc = s_path + KB_MAX_DEPTH + 2;  // [0] shadow_on, [1] n entries
  u64 *s_key = (u64 *)(((uintptr_t)(s_misc + 4) + 15) & ~(uintptr_t)15);  // [nn][4]
  // ---- 0. The nominate / key phases below follow, per entry, a chain of dependent loads through the per-cycle tables
  // (head -> workload -> podset rows -> resource group -> flavors), cold in L2 after the upload.  One thread per
  // ClusterQueue walks that chain now and only touches the lines (prefetch), overlapped with the table staging of
  // phase 1, so that the later phases find them in L1/L2.
  if ((int)threadIdx.x < nn) {
    auto touch = [](const void *p) { asm volatile("prefetch.global.L1 [%0];" ::"l"(p)); };
    const int nd = nodes[threadIdx.x];
    const int e = nd < D.Q ? D.cq_entry[nd] : -1;
    if (e >= 0) {
      const int wl = D.heads[e];
      touch(D.wl_cq + wl); touch(D.wl_last_gen + wl); touch(D.wl_priority + wl); touch(D.wl_ts + wl); touch(D.wl_uid + wl);
      touch(D.cq_generation + nd); touch(D.cq_preference + nd); touch(D.cq_when_can_borrow + nd); touch(D.cq_when_can_preempt + nd);
      touch(D.cq_within_cq + nd); touch(D.cq_reclaim_within + nd); touch(D.cq_borrow_within + nd); touch(D.fair_weight + nd);
      const int ps0 = D.wl_ps_start[wl], ps1 = D.wl_ps_start[wl + 1];
      const int g0 = D.cq_rg_start[nd], g1 = D.cq_rg_start[nd + 1];
      for (int row = ps0; row < ps1 && row < ps0 + 4; row++) {
        touch(D.ps_count + row); touch(D.ps_min_count + row); touch(D.ps_req_mask + row); touch(D.ps_flavor_ok + row);
        touch(D.ps_req + (size_t)row * R); touch(D.ps_last_tried + (size_t)row * R);
      }
      for (int g = g0; g < g1 && g < g0 + 4; g++) {
        touch(D.rg_res_mask + g);
        const int f0 = D.rg_flavor_start[g], f1 = D.rg_flavor_start[g + 1];
        for (int k = f0; k < f1; k += 32) touch(D.rg_flavors + k);
      }
    }
  }
  // ---- 1. stage: SubtreeQuota = Nominal, Usage = ClusterQueue usage | 0 (updateCohortResourceNode :184-190)
  for (int i = threadIdx.x; i < (int)tb; i += blockDim.x) {
    int nd = nodes[row_of(i)], fr = col_of(i);
    size_t c = (size_t)nd * FR + fr;
    s_sub[i] = D.nominal[c];
    s_u[i] = nd < D.Q ? D.cq_usage[c] : 0;
    s_bl[i] = D.blimit[c];
    s_lq[i] = D.llimit[c];  // lending limit for now; turned into localQuota once SubtreeQuota is final
  }
  for (int i = threadIdx.x; i < nn; i += blockDim.x) {
    int nd = nodes[i], pn = D.parent[nd];
    s_par[i] = pn < 0 ? -1 : D.local_idx[pn]; s_hgt[i] = D.height[nd];
  }
  if (threadIdx.x == 0) { s_misc[0] = 0; s_misc[1] = 0; }
  __syncthreads();
  KB_PHASE(0);
  // ---- 2. bottom-up accumulateFromChild :210-217 (deepest level first), then localQuota, then available top-down
  if (nlev == 2) {
    // flat cohort: every other node is a child of the root -> one warp per column sums its children (no atomics
    // on the ~100-way contended root cells)
    const int lane_ = threadIdx.x & 31, warp_ = threadIdx.x >> 5, nw = blockDim.x >> 5;
    for (int fr = warp_; fr < FR; fr += nw) {
      i64 dsub = 0, dus = 0;
      for (int h = 1 + lane_; h < nn; h += 32) {
        int c = h * FR + fr;
        i64 sub = s_sub[c];
        i64 lq = local_quota(sub, s_lq[c]);
        dsub += sub - lq;
        dus += imax(0, s_u[c] - lq);
      }
      for (int o = 16; o > 0; o >>= 1) { dsub += __shfl_xor_sync(0xffffffffu, dsub, o); dus += __shfl_xor_sync(0xffffffffu, dus, o); }
      if (lane_ == 0) {  // the root's cell is final: localQuota, available, potentialAvailable of the root (:104-133)
        i64 sub = s_sub[fr] + dsub, u = s_u[fr] + dus;
        s_sub[fr] = sub; s_u[fr] = u;
        s_lq[fr] = local_quota(sub, s_lq[fr]);
        s_av[fr] = sub - u; s_pot[fr] = sub;
      }
    }
    __syncthreads();
    // children in one pass: localQuota, then available / potentialAvailable below the root
    for (int i = FR + threadIdx.x; i < (int)tb; i += blockDim.x) {
      const int fr = col_of(i);
      i64 sub = s_sub[i], u = s_u[i], bl = s_bl[i];
      i64 lq = local_quota(sub, s_lq[i]);
      s_lq[i] = lq;
      i64 pa = s_av[fr], pot = lq + s_pot[fr];
      if (bl != KB_NO_LIMIT) { pa = imin((sub - lq) - imax(0, u - lq) + bl, pa); pot = imin(sub + bl, pot); }
      s_av[i] = imax(0, lq - u) + pa;
      s_pot[i] = pot;
    }
    __syncthreads();
  } else {
  for (int L = nlev - 1; L >= 1; L--) {
    int a = lvl[L], b = lvl[L + 1];
    for (int i = threadIdx.x; i < (b - a) * FR; i += blockDim.x) {
      int h = a + row_of(i), fr = col_of(i);
      int c = h * FR + fr, pc = s_par[h] * FR + fr;
      i64 sub = s_sub[c];
      i64 lq = local_quota(sub, s_lq[c]);
      atomicAdd((u64 *)&s_sub[pc], (u64)(sub - lq));
      i64 spill = imax(0, s_u[c] - lq);
      if (spill) atomicAdd((u64 *)&s_u[pc], (u64)spill);
    }
    __syncthreads();
  }
  for (int i = threadIdx.x; i < (int)tb; i += blockDim.x) s_lq[i] = local_quota(s_sub[i], s_lq[i]);
  __syncthreads();
  for (int L = 0; L < nlev; L++) {
    int a = lvl[L], b = lvl[L + 1];
    for (int i = threadIdx.x; i < (b - a) * FR; i += blockDim.x) {
      int h = a + row_of(i), fr = col_of(i);
      int c = h * FR + fr;
      i64 sub = s_sub[c], u = s_u[c];
      if (L == 0) { s_av[c] = sub - u; s_pot[c] = sub; }
      else {
        int pc = s_par[h] * FR + fr;
        i64 lq = s_lq[c], bl = s_bl[c];
        i64 pa = s_av[pc], pot = lq + s_pot[pc];
        if (bl != KB_NO_LIMIT) { pa = imin((sub - lq) - imax(0, u - lq) + bl, pa); pot = imin(sub + bl, pot); }
        s_av[c] = imax(0, lq - u) + pa;
        s_pot[c] = pot;
      }
    }
    __syncthreads();
  }
  }
  KB_PHASE(1);
  // ---- 3. fair sharing inputs (k_fair_prep): over-usage per (ClusterQueue, resource), lendable per (node, resource)
  const bool fair = D.flags & KB_F_FAIR_SHARING;
  if (fair) {
    for (int i = threadIdx.x; i < nn * R; i += blockDim.x) {
      int h = i / R, r = i % R;
      i64 over = 0, lend = 0;
      for (int f = 0; f < Fn; f++) {
        int c = h * FR + f * R + r;
        lend += s_pot[c];
        i64 o = s_u[c] - s_sub[c];
        if (o > 0) over += o;
      }
      s_lend[i] = lend; s_over[i] = over;
    }
  }
  // ---- 4. the root's entries, in ClusterQueue (= local handle) order
  if (threadIdx.x < 32) {
    int cnt = 0;
    for (int h0 = 0; h0 < nn; h0 += 32) {
      int h = h0 + threadIdx.x;
      int e = -1;
      if (h < nn && nodes[h] < D.Q) e = D.cq_entry[nodes[h]];
      unsigned m = __ballot_sync(0xffffffffu, e >= 0);
      if (e >= 0) s_ent[cnt + __popc(m & ((1u << threadIdx.x) - 1))] = e;
      cnt += __popc(m);
    }
    if (threadIdx.x == 0) s_misc[1] = cnt;
  }
  __syncthreads();
  const int n = s_misc[1];
  if (n == 0) { for (int i = threadIdx.x; i < (int)tb; i += blockDim.x) D.usage[(size_t)nodes[row_of(i)] * FR + col_of(i)] = s_u[i]; return; }
  KB_PHASE(2);
  // local view of the snapshot: node tables in shared memory, indexed by the local handle
  DevSnap L = D;
  L.tab_local = 1; L.parent = s_par; L.height = s_hgt; L.lq = s_lq;
  L.nominal = s_sub;  // only ever read for ClusterQueues: SubtreeQuota == Nominal there (resource_node.go:160-166)
  L.subtree = s_sub; L.usage = s_u; L.avail = s_av; L.potential = s_pot; L.blimit = s_bl;
  L.fs_over = s_over; L.fs_lend = s_lend;
  // ---- 5. nominate: KB_NG lanes per entry (get_assignments_coop), rows written straight to the output tables
  {
    const int lane = threadIdx.x & 31, glane = lane % KB_NG, gbase = lane - glane;
    const unsigned gmask = ((1u << KB_NG) - 1u) << gbase;
    const int groups = blockDim.x / KB_NG;
    for (int i0 = 0; i0 < n; i0 += groups) {
      int i = i0 + threadIdx.x / KB_NG;
      if (i < n) {  // whole KB_NG-lane groups take the branch together
        int e = s_ent[i];
        int wl = D.heads[e];
        bool need_search = false;
        int borrowing;
        int mode = get_assignments_coop(L, &need_search, wl, &borrowing, gmask, gbase, glane);
        if (glane == 0) { D.mode[e] = (uint8_t)mode; D.borrow[e] = borrowing; D.decision[e] = KB_DEC_NOFIT; D.rank[e] = -1; D.tgt_cnt[e] = 0; D.tgt_off[e] = 0; }
      }
    }
  }
  __syncthreads();
  KB_PHASE(3);  // output rows and mode/borrow are read back below by other threads (same CTA: visible after the barrier)
  Tab<true> T;
  T.D = &D; T.FR = FR; T.usage = s_u; T.sub = s_sub; T.lq = s_lq; T.bl = s_bl; T.lparent = s_par;
  T.shadow = D.usage_shadow; T.tnodes = nodes; T.tnn = nn; T.shadow_on = &s_misc[0];
  i64 *s_q = s_av;  // [entries][FR] requests: avail + potential are contiguous and dead after nomination
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const bool flat = FR <= 64 && D.tree_flat[t];
  if (flat && n <= KB_TILE) {
    // ---- 6a. Flat cohort, one entry per ClusterQueue, no preemption targets.  The only state one entry passes to
    // the next is the ROOT's usage per column: everything else of available() (resource_node.go:104-118 on the
    // two-node path) depends on the entry's own ClusterQueue row, which no other entry touches.  So the iterator keys
    // and, per (entry, column), one threshold are computed for all entries in parallel:
    //   fits  <=>  cap >= x  and  usage_root <= SubtreeQuota_root - x,   x = request - LocalAvailable(cq)
    //   admitted: usage_root += max(0, x)            (addUsage :137-145: what exceeds the local availability)
    // and the ordered loop (scheduler.go:269-401) is compare / vote / add on registers.  Entries in Preempt mode
    // without targets reserve unconditionally (:303-318, quotaResourcesToReserve :530-548).
    i64 *s_lim = s_pot;
    const int half = blockDim.x / 2;
    if ((int)threadIdx.x < n) compute_entry_key(L, s_ent[threadIdx.x], s_key + (size_t)threadIdx.x * 4);
    else if ((int)threadIdx.x >= half && (int)threadIdx.x - half < n) {  // tile metadata + dense request row, in entry order
      int i = threadIdx.x - half;
      int e = s_ent[i];
      int cqn = D.wl_cq[D.heads[e]];
      t_e[i] = e; t_node[i] = D.local_idx[cqn]; t_cq[i] = cqn; t_mode[i] = D.mode[e]; t_borrow[i] = D.borrow[e];
      i64 *qrow = s_q + (size_t)i * FR;
      for (int c = 0; c < FR; c++) qrow[c] = -1;
      expand_entry(D, e, qrow);
    }
    __syncthreads();
    KB_PHASE(4);
    if ((int)threadIdx.x < n) {  // position in the iterator order
      const u64 *mine = s_key + (size_t)threadIdx.x * 4;
      int rank = 0;
      for (int j = 0; j < n; j++) rank += key4_less(s_key + (size_t)j * 4, mine) ? 1 : 0;
      s_sorted[rank] = threadIdx.x;  // entry index (position in s_ent) at iterator position `rank`
      t_toff[threadIdx.x] = rank;
    } else if ((int)threadIdx.x >= half) {
      for (int c = threadIdx.x - half; c < n * FR; c += half) {
        int i = row_of(c), fr = col_of(c);
        i64 q = s_q[c];
        int r = t_node[i] * FR + fr;
        i64 u = s_u[r], l = s_lq[r], bl = s_bl[r], sub = s_sub[r];
        i64 A = imax(0, l - u);
        i64 v = INT64_MAX;  // Fit: threshold on the root usage; Preempt: amount added to the root
        int mode = t_mode[i];
        if (mode == KB_MODE_FIT) {
          if (q > 0) {
            i64 x = q - A;
            bool cap_ok = bl == KB_NO_LIMIT || (sub - l) - imax(0, u - l) + bl >= x;
            v = cap_ok ? s_sub[fr] - x : INT64_MIN;
          }
        } else if (mode == KB_MODE_PREEMPT) {
          v = 0;
          if (q >= 0 && D.cq_reclaim_within[t_cq[i]] != KB_POLICY_ANY) {
            i64 rsv = t_borrow[i] > 0 ? (bl == KB_NO_LIMIT ? q : imin(q, sub + bl - u)) : imax(0, imin(q, sub - u));
            v = rsv > A ? rsv - A : 0;
          }
        }
        s_lim[c] = v;
      }
    }
    __syncthreads();
    KB_PHASE(5);
    if (warp == 0) {
      const int fr0 = lane, fr1 = lane + 32;
      const bool c0 = fr0 < FR, c1 = fr1 < FR;
      i64 urt0 = c0 ? s_u[fr0] : 0, urt1 = c1 ? s_u[fr1] : 0;
      const i64 srt0 = c0 ? s_sub[fr0] : 0, srt1 = c1 ? s_sub[fr1] : 0;
      for (int p0 = 0; p0 < n; p0 += 4) {
        i64 v0[4], v1[4]; int md[4], ix[4];
#pragma unroll
        for (int k = 0; k < 4; k++) {
          bool in = p0 + k < n;
          int i = in ? s_sorted[p0 + k] : 0;
          ix[k] = i;
          md[k] = in ? t_mode[i] : -1;
          v0[k] = (in && c0) ? s_lim[(size_t)i * FR + fr0] : INT64_MAX;
          v1[k] = (in && c1) ? s_lim[(size_t)i * FR + fr1] : INT64_MAX;
        }
#pragma unroll
        for (int k = 0; k < 4; k++) {
          if (md[k] < 0) break;
          int dec = KB_DEC_NOFIT;
          if (md[k] == KB_MODE_FIT) {
            bool ok = __all_sync(0xffffffffu, urt0 <= v0[k] && urt1 <= v1[k]);
            if (ok) {
              if (c0 && v0[k] != INT64_MAX && srt0 > v0[k]) urt0 += srt0 - v0[k];
              if (c1 && v1[k] != INT64_MAX && srt1 > v1[k]) urt1 += srt1 - v1[k];
            }
            dec = ok ? KB_DEC_ASSUMED : KB_DEC_SKIPPED_NO_FIT;
          } else if (md[k] == KB_MODE_PREEMPT) {
            if (c0) urt0 += v0[k];
            if (c1) urt1 += v1[k];
            dec = KB_DEC_PREEMPT_NO_TARGETS;
          }
          if (lane == 0) t_ntg[ix[k]] = dec;
        }
      }
      if (c0) s_u[fr0] = urt0;
      if (c1) s_u[fr1] = urt1;
    }
    __syncthreads();
    KB_PHASE(6);
    // ClusterQueue rows of the admitted / reserving entries (cq.AddUsage), decisions and ranks
    for (int c = threadIdx.x; c < n * FR; c += blockDim.x) {
      int i = row_of(c), fr = col_of(c);
      int dec = t_ntg[i];
      i64 q = s_q[c];
      int r = t_node[i] * FR + fr;
      if (dec == KB_DEC_ASSUMED) { if (q > 0) s_u[r] += q; }
      else if (dec == KB_DEC_PREEMPT_NO_TARGETS && q >= 0 && D.cq_reclaim_within[t_cq[i]] != KB_POLICY_ANY) {
        i64 u = s_u[r], bl = s_bl[r], sub = s_sub[r];
        s_u[r] = u + (t_borrow[i] > 0 ? (bl == KB_NO_LIMIT ? q : imin(q, sub + bl - u)) : imax(0, imin(q, sub - u)));
      }
      if (fr == 0) { D.decision[t_e[i]] = (uint8_t)dec; D.rank[t_e[i]] = t_toff[i]; }
    }
    __syncthreads();
    for (int i = threadIdx.x; i < (int)tb; i += blockDim.x) D.usage[(size_t)nodes[row_of(i)] * FR + col_of(i)] = s_u[i];
    KB_PHASE(7);
    return;
  }
  // ---- 6b. general form: iterator order (4 x u64 key per entry, all-pairs rank in shared memory) ...
  for (int i = threadIdx.x; i < n; i += blockDim.x) compute_entry_key(L, s_ent[i], s_key + (size_t)i * 4);
  __syncthreads();
  for (int i = threadIdx.x; i < n; i += blockDim.x) {
    const u64 *mine = s_key + (size_t)i * 4;
    int rank = 0;
    for (int j = 0; j < n; j++) rank += key4_less(s_key + (size_t)j * 4, mine) ? 1 : 0;
    s_sorted[rank] = s_ent[i];
  }
  __syncthreads();
  KB_PHASE(4);
  // ---- 7. ... and the admit loop (scheduler.go:269-401) in tiles of KB_TILE entries
  for (int base = 0; base < n; base += KB_TILE) {
    int tn = min(KB_TILE, n - base);
    for (int i = threadIdx.x; i < tn; i += blockDim.x) {
      int e = s_sorted[base + i];
      int cqn = D.wl_cq[D.heads[e]];
      t_e[i] = e; t_node[i] = D.local_idx[cqn]; t_cq[i] = cqn;
      t_mode[i] = D.mode[e]; t_borrow[i] = D.borrow[e]; t_ntg[i] = 0; t_toff[i] = 0;
    }
    for (int c = threadIdx.x; c < tn * FR; c += blockDim.x) s_q[c] = -1;
    __syncthreads();
    for (int i = threadIdx.x; i < tn; i += blockDim.x) expand_entry(D, t_e[i], s_q + (size_t)i * FR);
    __syncthreads();
    if (warp == 0) {
      if (flat) {
        if (FR > 32) commit_tile_flat<true>(D, T, s_path, lane, tn, base, s_q, t_e, t_node, t_mode, t_borrow, t_cq, t_ntg, t_toff);
        else commit_tile_flat<false>(D, T, s_path, lane, tn, base, s_q, t_e, t_node, t_mode, t_borrow, t_cq, t_ntg, t_toff);
      } else {
        for (int i = 0; i < tn; i++)
          commit_entry<true>(D, T, s_path, lane, t_e[i], t_node[i], t_mode[i], t_borrow[i], s_q + (size_t)i * FR, base + i, t_cq[i], 0, 0);
      }
    }
    __syncthreads();
    if (flat)
      for (int i = threadIdx.x; i < tn; i += blockDim.x) {
        int m = t_mode[i];
        if (m >= 0x100) { D.decision[t_e[i]] = (uint8_t)(m & 0xff); D.rank[t_e[i]] = base + i; }
      }
    __syncthreads();
  }
  KB_PHASE(5);
  for (int i = threadIdx.x; i < (int)tb; i += blockDim.x) D.usage[(size_t)nodes[row_of(i)] * FR + col_of(i)] = s_u[i];
  KB_PHASE(6);
}
__global__ void k_cq_entry(DevSnap D, int32_t *cq_entry) {  // ClusterQueue -> its single head of this cycle
  int e = blockIdx.x * blockDim.x + threadIdx.x;
  if (e < D.H) cq_entry[D.wl_cq[D.heads[e]]] = e;
}

// ---------------------------------------------------------------------------
// K5b: admit loop for ClusterQueues WITHOUT a cohort (every such CQ is its own root): one
// WARP per ClusterQueue, four per CTA.  The quota "tree" is one row: lane l keeps the usage
// and nominal quota of its flavor-resource columns l, l+32 in REGISTERS, so the ordered
// commit loop (scheduler.go:269-401) touches memory only for the entries themselves.  Entries
// arrive in iterator order (k_rank) and are expanded 32 at a time into a dense request matrix
// (one lane per entry).
// Roots with more than KB_RANK_CAP entries, or with preemption targets in play, are left
// to the general kernel.
// ---------------------------------------------------------------------------
__global__ void __launch_bounds__(KB_LONE_WARPS * 32) k_admit_lone(DevSnap D) {
  extern __shared__ __align__(16) unsigned char smem_raw[];
  const int FR = D.FR;
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  int slot = blockIdx.x * KB_LONE_WARPS + warp;
  if (slot >= D.nLone) return;
  int off = D.root_offset[slot];
  int n = D.root_offset[slot + 1] - off;
  if (n == 0 || n > KB_RANK_CAP) return;
  const int32_t *order = D.sorted + off;  // iterator order from k_rank
  int cq = D.lone_cqs[slot];
  // per-warp shared memory: dense request chunk (32 x FR x 8 B)
  i64 *qm = (i64 *)(smem_raw + (size_t)warp * 32 * FR * 8);
  // ---- the CQ's row in registers (two columns per lane: FR <= 64) ----
  const bool two = FR > 32;
  const int c0 = lane, c1 = lane + 32;
  i64 u0 = 0, u1 = 0, nom0 = 0, nom1 = 0;
  if (c0 < FR) { u0 = D.usage[(size_t)cq * FR + c0]; nom0 = D.subtree[(size_t)cq * FR + c0]; }
  if (two && c1 < FR) { u1 = D.usage[(size_t)cq * FR + c1]; nom1 = D.subtree[(size_t)cq * FR + c1]; }
  const bool reserve_ok = D.cq_reclaim_within[cq] != KB_POLICY_ANY;  // !CanAlwaysReclaim policy.go:27-29
  // ---- chunks of 32 entries: expand (lane = entry), then commit in order (lane = column) ----
  for (int basei = 0; basei < n; basei += 32) {
    int cn = min(32, n - basei);
    for (int c = lane; c < cn * FR; c += 32) qm[c] = -1;
    __syncwarp();
    int my_e = lane < cn ? order[basei + lane] : -1;
    int my_mode = 0, my_dec = 0;
    if (my_e >= 0) { expand_entry(D, my_e, qm + (size_t)lane * FR); my_mode = D.mode[my_e]; }
    __syncwarp();
    for (int jb = 0; jb < cn; jb += 8) {
      // batch the state-independent loads of 8 entries, then walk them with a short dependent chain
      i64 q0[8], q1[8]; int md[8];
#pragma unroll
      for (int t = 0; t < 8; t++) {
        int j = jb + t;
        bool in = j < cn;
        md[t] = __shfl_sync(0xffffffffu, my_mode, j & 31);
        q0[t] = (in && c0 < FR) ? qm[(size_t)j * FR + c0] : -1;
        q1[t] = (in && two && c1 < FR) ? qm[(size_t)j * FR + c1] : -1;
        if (!in) md[t] = -1;
      }
#pragma unroll
      for (int t = 0; t < 8; t++) {
        int mode = md[t];
        if (mode < 0) break;
        int dec;
        if (mode == KB_MODE_NOFIT) dec = KB_DEC_NOFIT;
        else if (mode == KB_MODE_PREEMPT) {  // Preempt without targets (entries with targets never reach this kernel): :303-318
          dec = KB_DEC_PREEMPT_NO_TARGETS;
          if (reserve_ok) {  // quotaResourcesToReserve :530-548 with Borrowing == 0 (no cohort)
            if (q0[t] >= 0) u0 += imax(0, imin(q0[t], nom0 - u0));
            if (q1[t] >= 0) u1 += imax(0, imin(q1[t], nom1 - u1));
          }
        } else {
          bool ok = !(q0[t] > 0 && imax(0, nom0 - u0) < q0[t]) && !(q1[t] > 0 && imax(0, nom1 - u1) < q1[t]);  // Fits :121-136
          ok = __all_sync(0xffffffffu, ok);
          if (ok) { if (q0[t] > 0) u0 += q0[t]; if (q1[t] > 0) u1 += q1[t]; }
          dec = ok ? KB_DEC_ASSUMED : KB_DEC_SKIPPED_NO_FIT;
        }
        if (lane == jb + t) my_dec = dec;
      }
    }
    if (my_e >= 0) { D.decision[my_e] = (uint8_t)my_dec; D.rank[my_e] = basei + lane; }
    __syncwarp();
  }
  if (c0 < FR) D.usage[(size_t)cq * FR + c0] = u0;
  if (two && c1 < FR) D.usage[(size_t)cq * FR + c1] = u1;
}

// ---------------------------------------------------------------------------
// K4: fair-sharing iterator + admit (fair_sharing_iterator.go:36-229), one CTA per
// cohort tree.  Each pop: (1) every remaining entry recomputes, one thread per entry,
// the DominantResourceShare of each node on its CQ->root path as if its own usage were
// admitted (computeDRS :206-229, without mutating the tree: the usage bubbling of
// addUsage is replayed functionally per column); (2) the tournament (runTournament
// :120-153) runs bottom-up over the cohort levels, one warp per cohort with a
// shuffle reduction over its children; (3) warp 0 commits the winner.
// ---------------------------------------------------------------------------
// Per-entry state of one cohort tree's tournament, staged once per cycle (slot = position of
// the entry in the root's entry list).  Shared memory when it fits, else a global scratch of
// the same layout.
struct FsState {
  double2 *drs;     // [n][nlev] (unweightedRatio, fairWeight) per path level
  i64 *e_ts;        // [n]
  int *e_id;        // [n] global entry index
  int *e_cq;        // [n] ClusterQueue (global node id)
  int *e_prio;      // [n]
  int *e_flags;     // [n] bit0 requiresBorrowing, bit1 alive, bit2 dirty (DRS must be recomputed)
  int *e_top;       // [n] local index of the ancestor directly below the root (the CQ itself in a flat cohort)
  int *e_depth;     // [n] depth of the ClusterQueue
  int *e_mode;      // [n] RepresentativeMode | Borrowing << 8
  int nlev;
};
#define KB_FS_ENTRY_BYTES (48 + 16 * KB_MAX_DEPTH)

// entryComparer.less fair_sharing_iterator.go:166-199 for slots a, b under a parent cohort of depth dP
__device__ __forceinline__ bool fs_less(const DevSnap &D, const FsState &F, int a, int b, int dP) {
  if (D.flags & KB_F_FS_PRIORITIZE_NON_BORROWING) {
    bool ab = F.e_flags[a] & 1, bb = F.e_flags[b] & 1;
    if (ab != bb) return !ab;
  }
  int ka = F.e_depth[a] - dP - 1, kb = F.e_depth[b] - dP - 1;
  double2 va = F.drs[(size_t)a * F.nlev + ka], vb = F.drs[(size_t)b * F.nlev + kb];
  DevDRS da{va.y, va.x, -1, false}, db{vb.y, vb.x, -1, false};
  int c = drs_compare(da, db);
  if (c != 0) return c < 0;
  if (D.flags & KB_F_PRIORITY_SORTING_WITHIN_COHORT) {
    int pa = F.e_prio[a], pb = F.e_prio[b];
    if (pa != pb) return pa > pb;
  }
  return F.e_ts[a] < F.e_ts[b];
}

template <bool kSmemTables>
__global__ void __launch_bounds__(128) k_admit_fair(DevSnap D, int slot_base, int state_in_smem) {
  extern __shared__ __align__(16) unsigned char smem_raw[];
  const int FR = D.FR, R = D.R, Fn = D.F;
  int slot = slot_base + blockIdx.x;
  int off = D.root_offset[slot];
  int n = D.root_offset[slot + 1] - off;
  if (n == 0) return;
  int32_t *ent = D.root_entries + off;
  int t = slot - D.nLone;
  if (D.tree_flat[t]) return;  // flat cohorts: the pop order is a static key order -> k_rank + k_admit
  const int32_t *nodes = D.tree_nodes + D.tree_start[t];
  int nn = D.tree_start[t + 1] - D.tree_start[t];
  const int32_t *lvl = D.tree_level + (size_t)t * KB_LEVELS;
  int nlev = 0;
  while (nlev + 1 < KB_LEVELS && lvl[nlev + 1] > lvl[nlev]) nlev++;
  Tab<kSmemTables> T;
  unsigned char *p = stage_tables<kSmemTables>(D, T, smem_raw, nodes, nn);
  int *s_path = (int *)p; p += (KB_MAX_DEPTH + 2) * 4;
  int *s_shadow_on = (int *)p; p += 8;
  if (threadIdx.x == 0) *s_shadow_on = 0;
  T.shadow_on = s_shadow_on;
  // tree index arrays in LOCAL node ids (always shared memory): children CSR, waiting slot of a CQ, winner of a cohort
  int *s_cstart = (int *)p; p += (size_t)(nn + 1) * 4;
  int *s_child = (int *)p; p += (size_t)nn * 4;
  int *s_slot = (int *)p; p += (size_t)nn * 4;
  int *s_winner = (int *)p; p += (size_t)nn * 4;
  p = (unsigned char *)(((uintptr_t)p + 15) & ~(uintptr_t)15);
  FsState F;
  F.nlev = nlev > 1 ? nlev - 1 : 1;  // a CQ at depth d has d path levels; d <= nlev-1
  {
    unsigned char *q = state_in_smem ? p : D.fs_state + (size_t)off * KB_FS_ENTRY_BYTES;
    F.drs = (double2 *)q; q += (size_t)n * F.nlev * 16;
    F.e_ts = (i64 *)q; q += (size_t)n * 8;
    F.e_id = (int *)q; q += (size_t)n * 4; F.e_cq = (int *)q; q += (size_t)n * 4; F.e_prio = (int *)q; q += (size_t)n * 4;
    F.e_flags = (int *)q; q += (size_t)n * 4; F.e_top = (int *)q; q += (size_t)n * 4;
    F.e_depth = (int *)q; q += (size_t)n * 4; F.e_mode = (int *)q; q += (size_t)n * 4;
  }
  for (int i = threadIdx.x; i < nn; i += blockDim.x) {
    int nd = nodes[i];
    (void)nd;
    s_slot[i] = -1; s_winner[i] = -1;
  }
  __syncthreads();
  // children CSR in local ids: count, scan (thread 0; nn is small), fill
  if (threadIdx.x == 0) {
    int acc = 0;
    for (int i = 0; i < nn; i++) { int nd = nodes[i]; s_cstart[i] = acc; acc += D.child_start[nd + 1] - D.child_start[nd]; }
    s_cstart[nn] = acc;
  }
  __syncthreads();
  for (int i = threadIdx.x; i < nn; i += blockDim.x) {
    int nd = nodes[i];
    int c0 = D.child_start[nd], cn = D.child_start[nd + 1] - c0;
    for (int k = 0; k < cn; k++) s_child[s_cstart[i] + k] = D.local_idx[D.child_list[c0 + k]];
  }
  for (int i = threadIdx.x; i < n; i += blockDim.x) {
    int e = ent[i];
    int wl = D.heads[e];
    int cq = D.wl_cq[wl];
    F.e_id[i] = e; F.e_cq[i] = cq; F.e_prio[i] = D.wl_priority[wl]; F.e_ts[i] = D.wl_ts[wl];
    int bw = D.borrow[e];
    F.e_flags[i] = (bw > 0 ? 1 : 0) | 2 | 4;
    F.e_mode[i] = (int)D.mode[e] | (bw << 8);
    F.e_depth[i] = D.depth[cq];
    int top = cq;
    while (D.parent[top] >= 0 && D.parent[D.parent[top]] >= 0) top = D.parent[top];
    F.e_top[i] = D.local_idx[top];
    s_slot[D.local_idx[cq]] = i;
  }
  for (int c = threadIdx.x; c < n * FR; c += blockDim.x) { int e = ent[c / FR]; D.q_scratch[(size_t)e * FR + c % FR] = entry_request(D, e, c % FR); }
  __syncthreads();
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, nwarps = blockDim.x >> 5;

  // computeDRS (:206-229) for the dirty entries: DRS of every node on the CQ->root path as if the entry were admitted
  auto compute_drs = [&]() {
    for (int i = threadIdx.x; i < n; i += blockDim.x) {
      int fl = F.e_flags[i];
      if ((fl & 6) != 6) continue;  // popped or clean
      F.e_flags[i] = fl & ~4;
      int e = F.e_id[i], cq = F.e_cq[i];
      const i64 *q = D.q_scratch + (size_t)e * FR;
      int X = cq;
      for (int k = 0; D.parent[X] >= 0; k++, X = D.parent[X]) {
        int P = D.parent[X];
        int hX = T.handle(X);
        double best = 0.0;
        for (int r = 0; r < R; r++) {
          i64 b = 0, lend = 0;
          for (int f = 0; f < Fn; f++) {
            int fr = f * R + r;
            // usage that the entry adds at node X in column fr: replay addUsage from the CQ up to X
            i64 d = q[fr] > 0 ? q[fr] : 0;
            int Y = cq;
            for (int j = 0; j < k && d > 0; j++, Y = D.parent[Y]) {
              int hY = T.handle(Y);
              i64 la = imax(0, T.LQ(hY, fr) - T.U(hY, fr));
              d = d > la ? d - la : 0;
            }
            i64 over = T.U(hX, fr) + d - T.Sub(hX, fr);
            if (over > 0) b += over;
            lend += D.potential[(size_t)P * FR + fr];  // calculateLendable fair_sharing.go:160-174
          }
          if (b > 0 && lend > 0) {
            double ratio = (double)b * 1000.0 / (double)lend;
            if (ratio > best) best = ratio;
          }
        }
        F.drs[(size_t)i * F.nlev + k] = make_double2(best, D.fair_weight[X]);
      }
    }
  };

  for (int it = 0; it < n; it++) {
    compute_drs();  // (1)
    __syncthreads();
    // (2) tournament (runTournament :120-153), bottom-up over cohort levels, one warp per cohort
    for (int L = nlev - 1; L >= 0; L--) {
      for (int idx = lvl[L] + warp; idx < lvl[L + 1]; idx += nwarps) {
        if (nodes[idx] < D.Q) continue;  // CQs carry entries, cohorts run the tournament
        int c0 = s_cstart[idx], c1 = s_cstart[idx + 1];
        int best = -1, bestpos = INT32_MAX;
        for (int c = c0 + lane; c < c1; c += 32) {
          int ch = s_child[c];
          int cand = nodes[ch] < D.Q ? s_slot[ch] : s_winner[ch];
          if (cand < 0) continue;
          if (best < 0 || fs_less(D, F, cand, best, L)) { best = cand; bestpos = c; }  // the earlier candidate keeps ties
        }
        for (int o = 16; o > 0; o >>= 1) {
          int ob = __shfl_xor_sync(0xffffffffu, best, o), op = __shfl_xor_sync(0xffffffffu, bestpos, o);
          if (ob >= 0) {
            bool take;
            if (best < 0) take = true;
            else if (fs_less(D, F, ob, best, L)) take = true;
            else if (fs_less(D, F, best, ob, L)) take = false;
            else take = op < bestpos;
            if (take) { best = ob; bestpos = op; }
          }
        }
        if (lane == 0) s_winner[idx] = best;
      }
      __syncthreads();
    }
    // (3) pop + commit (warp 0), then mark the entries whose DRS inputs changed
    int w = s_winner[0];
    int wcq = F.e_cq[w], we = F.e_id[w];
    if (warp == 0) {
      int md = F.e_mode[w];
      commit_entry<kSmemTables>(D, T, s_path, lane, we, T.handle(wcq), md & 0xff, md >> 8, D.q_scratch + (size_t)we * FR, it,
                                wcq, D.tgt_cnt[we], D.tgt_off[we]);
      __syncwarp();
      if (lane == 0) {
        int dec = D.decision[we];  // every branch that may have touched the tree's usage
        bool changed = dec == KB_DEC_ASSUMED || dec == KB_DEC_PREEMPTING || dec == KB_DEC_PREEMPT_NO_TARGETS;
        s_slot[D.local_idx[wcq]] = -1; F.e_flags[w] &= ~2; s_path[KB_MAX_DEPTH] = changed;
      }
    }
    __syncthreads();
    if (s_path[KB_MAX_DEPTH]) {  // usage changed along path(wcq): entries below the same child-of-root share nodes with it
      int top = F.e_top[w];
      if (top != D.local_idx[wcq])  // directly under the root: shares no non-root node with anyone else
        for (int i = threadIdx.x; i < n; i += blockDim.x) if (F.e_top[i] == top) F.e_flags[i] |= 4;
    }
    __syncthreads();
  }
  publish_usage<kSmemTables>(D, T, nodes, nn);
}

#include "kb_flat.cuh"
