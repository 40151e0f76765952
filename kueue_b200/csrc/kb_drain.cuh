// kb_drain.cuh — the queue layer of kb_run_drain on the device (SURVEY.md §8 f1).
//
// Reference: pkg/cache/queue/cluster_queue.go:362-425 (requeueIfNotPresent, handleInadmissibleHash), :494-510 (Pop),
// :609-685 (RequeueIfNotPresent, queueOrderingFunc); manager.go:770-794 (heads); pkg/scheduler/scheduler.go:405-418,
// 823-850 (requeueAndUpdate); pkg/workload/workload.go:161-191 (PendingFlavors, NextFlavorToTryForPodSetResource).
//
// The heaps of the reference become, per ClusterQueue, one segment of the pending workloads sorted once by
// queueOrderingFunc (priority desc, queue-order timestamp, UID) plus a cursor, and one state byte per workload
// (KB_WS_QUEUED / KB_WS_SET_ASIDE: the inadmissible set / KB_WS_HELD: holds quota).  "Pop the heap" is "first QUEUED
// workload in the static order": the cursor of a segment always points at it (no QUEUED workload lies before it).
// Every cycle: pick the heads (ordered compaction over ClusterQueues), run the unchanged cycle kernels on them, then
// apply the decisions — admissions extend the admitted tables and the ClusterQueue usage on the device, the others
// keep their LastAssignment and move per the Strict / BestEffort FIFO rules.
//
// Eviction replay (kb_snapshot.adm_wl != NULL, a preemption policy somewhere): after the decisions and k_drain_admit,
// k_drain_evict takes every target of every Preempting entry out of the ClusterQueue usage, flags its row dead and
// requeues its pending record (LastAssignment nil; the cursor moves back to it if it lies before).  k_drain_requeue
// then returns every set-aside workload of the ClusterQueues of the victims' root cohort trees to its queue, moving the
// cursor back to the first of them (first_aside tracks that position per segment).  k_drain_live + two exclusive scans
// + k_drain_compact copy the live rows, in order, into the other half of a double buffer: the rows the cycle started
// with, then the admissions k_drain_admit appended after them.  A workload holds at most one live row, so the rows
// never exceed the capacity drain_impl reserves (kb_api.cu).
//
// AdmissionFairSharing (kb_snapshot.wl_lq != NULL): the queue of a ClusterQueue with cq_afs set is one SEGMENT per
// LocalQueue (each sorted as above, each with its own cursor); every other ClusterQueue is one segment.  Segments are
// numbered ClusterQueue-major (seg_start[Q+1]).  The head of an AFS ClusterQueue is the minimum of (LocalQueue usage by
// cmp.Compare, -priority, timestamp, UID) over the heads of its segments (one warp per ClusterQueue, k_drain_afs_heads);
// an admission adds its entry penalty to its LocalQueue and recomputes that LocalQueue's usage (k_drain_admit).  In event
// mode with lq_last_update_ns the consumed usage decays (include/kueue_b200.h): k_drain_afs_decay takes the samples due
// at the start and at every boundary, k_drain_admit decays to t_c and puts the penalty into consumed, k_drain_finish
// takes finished rows out of the LocalQueue's admitted usage (adm.lq, carried by the compaction).
//
// Event mode (kb_snapshot.wl_create_ns / wl_run_ns / adm_finish_ns / wl_evict_ns; include/kueue_b200.h): two more states,
// KB_WS_ABSENT (not created yet) and KB_WS_FINISHED.  Every admitted row carries its finish time (adm.finish, written by
// k_drain_admit, carried by the compaction) and its record (adm.wl, -1 for a row of the snapshot without one).  The
// boundary is the replay's, with the clock between the evictions and the requeue: k_drain_ev_min reduces E (the
// earliest finish of a live row and the next creation), k_drain_ev_next (one thread) computes t_{c+1} and the end
// flag, k_drain_finish stamps the finished rows dead with the eviction stamp and takes their cells out (a row admitted
// in this cycle that finishes by t_{c+1} dies before any cycle sees it), k_drain_arrive walks the arrived prefix of the
// (create, index) order; then k_drain_requeue visits the marked roots and the compaction follows.  A cycle without heads
// is replaced by the same boundary with t_{c+1} = E and a negative stamp (no cycle is counted).  The NoFit set of a
// ClusterQueue is one byte per (ClusterQueue, scheduling hash) class: k_drain_apply sets it, k_drain_requeue clears the
// bytes of the queues it visits.  With eviction latency (wl_evict_ns) k_drain_evict only issues: it sets adm_evicted and
// the byte column adm.evicting (carried by the compaction) and writes the end time into the finish column, so E and the
// compaction see it unchanged; k_drain_finish releases the row at its end time through the replay's requeue path.
//
// Sticky workload (kb_snapshot.cq_sticky; include/kueue_b200.h): one slot per ClusterQueue.  k_drain_heads takes a QUEUED
// sticky workload as the head instead of the one at the cursor, so the head may lie past the cursor: k_drain_apply moves
// the queue from the head's own position (wl_pos), excludes the head from the scheduling-hash move by identity, and sets
// (a Preempting head of a BestEffortFIFO ClusterQueue) or clears (its admission) the slot.  One head per ClusterQueue per
// cycle: one writer per slot.  Never set on an AFS ClusterQueue (refused, and no preemption there), so k_drain_afs_heads
// does not read it.
//
// Admission checks (kb_snapshot.wl_check_ns; include/kueue_b200.h): the row-phase byte column adm.phase (both halves,
// carried by the compaction) marks a row whose checks run (KB_PH_CHECK); its verdict time lives in the finish column, so
// k_drain_ev_min sees it unchanged.  k_drain_admit starts the attempt, k_drain_evict drops it (a preempted row without pods is released at the
// next boundary), k_drain_finish applies the verdicts before the completions.  The DevSnap's wl_ts is the mutable
// queue-order timestamp the cycle kernels read (wl_ts0 keeps the creation timestamps).  k_drain_backoff (one pass over
// the records per boundary) requeues the BACKOFF records whose RequeueAt has come and reduces the next RequeueAt into
// clock[2], which k_drain_ev_next folds into E.  A record that enters its queue with a timestamp other than the key the
// order was built with (wl_sort_ts) stamps KB_DC_RESORT with the boundary; the host then rebuilds the order (kb_api.cu).
//
// WaitForPodsReady (kb_snapshot.wl_pods_ready_ns) runs on the same machinery.  drain_admitted starts an attempt
// (kb_pr_attempt) at Admitted (k_drain_admit, or a Ready verdict in k_drain_finish): a ready one only moves the finish column, a failing one
// is KB_PH_WAIT with its timeout T in the finish column.  k_drain_finish applies the timeout after the verdicts: Count,
// RequeueAt and the queue timestamp on the record, and the row is KB_PH_TIMED_OUT, released at once or, with latency, at
// T + latency as an evicting row; its release sends the record to BACKOFF (k_drain_backoff queues it) or DEACTIVATED.
// k_drain_evict drops a waiting attempt.
//
// MaximumExecutionTimeSeconds (kb_snapshot.wl_max_exec_s) adds one int64 row column, adm.since (the Admitted time;
// both halves, carried by the compaction), and the per-record limit and accumulated time.  kb_exec_clip puts the
// effective deadline into the finish column where it comes before the row's own event (KB_PH_EXPIRE): in drain_admitted,
// after the PodsReady attempt.  k_drain_finish applies an expiry after the timeouts: the record is
// deactivated and the row becomes KB_PH_TIMED_OUT, whose release sends a deactivated record to DEACTIVATED.
// drain_exec_release adds an attempt's seconds at every release of a row with an Admitted time (k_drain_finish, and
// k_drain_evict without latency) and deactivates a record whose deadline passed before the release.
//
// Reclaim steps (kb_snapshot.wl_rc_start) add two row columns (both halves, carried by the compaction): adm.rc_next, the
// time of the row's next step, and adm.rc_cur, its index.  drain_rc_begin starts a run (k_drain_admit, and a Ready
// verdict in k_drain_finish), which also records the admission's PodSetAssignment per podset (ps_adm_*; the snapshot's
// rows bring theirs).  k_drain_ev_min folds the next step of a running row into E, and k_drain_finish applies the steps
// due (drain_reclaim) before a row's completion, its stop or its expiry: a thread per row, integer atomics on the usage
// tables, one writer for the record's ps_count / ps_req / wl_sched_hash (a record holds at most one row).
#pragma once

#include <cub/device/device_scan.cuh>

#include "kb_device.cuh"

// Backoff.WaitTime (pkg/util/wait/backoff.go:35-60) without jitter: wait.Backoff.Step `iteration` times (the duration
// grows by `factor` in float64 and is capped at cap, after which Step returns cap), stopping at the cap.  cap 0 =
// MaxInt64 / ceil(factor).  Restated by kueue_b200/drain.py wait_time.
__host__ __device__ inline i64 kb_backoff_wait(i64 base, i64 cap, double factor, int iteration) {
  if (base == 0) return 0;  // every Step returns 0: no loop over a large iteration count
  if (cap == 0) cap = (i64)(9223372036854775807.0 / ceil(factor));
  i64 dur = base, out = 0;
  bool capped = false;
  for (int i = 0; i < iteration; i++) {
    out = dur;
    if (!capped) {
      const double x = (double)dur * factor;
      if (x >= 9223372036854775808.0 || (i64)x > cap) { dur = cap; capped = true; }  // past int64 is past the cap too
      else dur = (i64)x;
    }
    if (out == cap) break;
  }
  return out;
}
// RequeueAfterSeconds of admission-check attempt k: WaitTime(k) of wait.NewBackoff(base, max, 2, 0.0001) truncated to
// whole seconds, exact below 10,000 s (kb_run_drain refuses a reachable backoff at or above it).  With base > max > 0 the
// first Step returns the base uncapped.  Restated by kueue_b200/drain.py check_wait_s.
__host__ __device__ inline i64 kb_check_wait_ns(int k, i64 base_s, i64 max_s) {
  return kb_backoff_wait(base_s * 1000000000ll, max_s * 1000000000ll, 2.0, k) / 1000000000ll * 1000000000ll;
}
// WaitTime of PodsReady requeue k (UpdateRequeueState workload.go:707-722): wait.NewBackoff(base, max, 2, 0.0001)
// without jitter, in nanoseconds (RequeueAt = T + it).  Restated by kueue_b200/drain.py pods_ready_wait_ns.
__host__ __device__ inline i64 kb_pods_ready_wait_ns(int k, i64 base_s, i64 max_s) {
  return kb_backoff_wait(base_s * 1000000000ll, max_s * 1000000000ll, 2.0, k);
}
// Seconds of an Admitted span of d >= 0 ns as SyncAdmittedCondition adds them (admissionchecks.go:73-80):
// int32(Duration.Seconds()) with Seconds() = float64(d / 1e9) + float64(d % 1e9) / 1e9, so from about 2^24 s the sum can
// round up to the next second.  -1 when the value leaves int32 (Go's conversion is then undefined).  Restated by
// kueue_b200/drain.py exec_seconds.
__host__ __device__ inline i64 kb_exec_seconds(i64 d) {
  const double x = (double)(d / 1000000000ll) + (double)(d % 1000000000ll) / 1e9;
  return x >= 2147483648.0 ? -1 : (i64)x;
}
__host__ __device__ inline i64 drain_sat_add(i64 t, i64 d) { return t > INT64_MAX - d ? INT64_MAX : t + d; }  // d >= 0
// the MaximumExecutionTimeSeconds deadline A + (max - acc) s of a row Admitted at A (acc -1 = nil, read as 0), saturating
// both ways.  Restated by kueue_b200/drain.py exec_deadline.
__host__ __device__ inline i64 kb_exec_deadline(i64 A, int32_t max_s, int32_t acc_s) {
  const i64 left = ((i64)max_s - (acc_s < 0 ? 0 : acc_s)) * 1000000000ll;
  if (left >= 0) return A > INT64_MAX - left ? INT64_MAX : A + left;
  return A < INT64_MIN - left ? INT64_MIN : A + left;
}
// adm.phase: what the finish column of a row holds.  RUN: its finish (or its eviction's end when adm.evicting); CHECK: its
// checks' verdict; WAIT: the timeout T of a PodsReady attempt that fails; TIMED_OUT: the end of its eviction by that
// timeout or by an expiry; EXPIRE: its effective MaximumExecutionTimeSeconds deadline, which comes before its own event
enum { KB_PH_RUN = 0, KB_PH_CHECK = 1, KB_PH_WAIT = 2, KB_PH_TIMED_OUT = 3, KB_PH_EXPIRE = 4 };
struct DrainFin { i64 fin; uint8_t ph; };  // a row's finish column and phase
// WaitForPodsReady: the attempt of a row Admitted at t.  A failing one (failures left, or a delay d past the timeout)
// waits for its timeout T = t + timeout; a ready one reaches PodsReady at t + d, and its finish is PodsReady + run (run
// < 0 never finishes).
__host__ __device__ inline DrainFin kb_pr_attempt(i64 t, i64 d, bool failing, i64 timeout, i64 run) {
  if (failing || d > timeout) return {drain_sat_add(t, timeout), KB_PH_WAIT};
  return {run < 0 ? INT64_MAX : drain_sat_add(drain_sat_add(t, d), run), KB_PH_RUN};
}
// MaximumExecutionTimeSeconds of a row Admitted at A whose own next event is f: the effective deadline max(D, A, floor)
// when it comes first, as KB_PH_EXPIRE (a tie goes to the own event).  floor: now_ns for the snapshot's rows.
__host__ __device__ inline DrainFin kb_exec_clip(DrainFin f, i64 A, int32_t max_s, int32_t acc_s, i64 floor) {
  if (max_s <= 0) return f;
  i64 dl = kb_exec_deadline(A, max_s, acc_s);
  dl = dl < A ? A : dl;
  dl = dl < floor ? floor : dl;
  return dl < f.fin ? DrainFin{dl, KB_PH_EXPIRE} : f;
}

// ---- resource.Quantity in the int64Amount form (value * 10^scale), as AdmissionFairSharing sums it -----------------
// Pow10 for |n| <= 22: 10^n is exact in a double, and Go's math.Pow10(-n) is 1 / 10^n (not a multiplication by 1e-n).
__host__ __device__ inline double afs_pow10(int n) {
  double p = 1.0;
  for (int i = 0; i < (n < 0 ? -n : n); i++) p *= 10.0;
  return n < 0 ? 1.0 / p : p;
}
#define AFS_MAX_SCALE 22
// positiveScaleInt64 (apimachinery math.go:140-165): v * 10^k, false on int64 overflow
__host__ __device__ inline bool afs_scale_up(i64 v, int k, i64 *out) {
  for (int i = 0; i < k; i++) {
    if (v > 922337203685477580ll || v < -922337203685477580ll) return false;
    v *= 10;
  }
  *out = v;
  return true;
}
// int64Add (math.go): false when the sum leaves int64
__host__ __device__ inline bool afs_add64(i64 a, i64 b, i64 *out) {
  i64 c = (i64)((u64)a + (u64)b);
  if ((a > 0 && b > 0 && c < 0) || (a < 0 && b < 0 && c >= 0)) return false;
  *out = c;
  return true;
}
// int64Amount.Add (amount.go:162-199): a zero operand keeps the other's scale, otherwise the smaller scale wins
__host__ __device__ inline bool afs_qty_add(i64 av, int as, i64 bv, int bs, i64 *rv, int *rs) {
  if (bv == 0) { *rv = av; *rs = as; return true; }
  if (av == 0) { *rv = bv; *rs = bs; return true; }
  i64 c;
  if (as == bs) { if (!afs_add64(av, bv, &c)) return false; *rv = c; *rs = as; return true; }
  if (as > bs) { if (!afs_scale_up(av, as - bs, &c) || !afs_add64(c, bv, &c)) return false; *rv = c; *rs = bs; return true; }
  if (!afs_scale_up(bv, bs - as, &c) || !afs_add64(av, c, &c)) return false;
  *rv = c; *rs = as;
  return true;
}
// Quantity.AsApproximateFloat64 (quantity.go:468-483)
__host__ __device__ inline double afs_qty_float(i64 v, int s) { return s == 0 ? (double)v : (double)v * afs_pow10(s); }
// Info.CalcLocalQueueFSUsage (workload.go:391-427) for one LocalQueue, resources in index order (the reference sums over
// a map: its order is random; this order is the library's canonical choice).  A zero quantity adds nothing, like an
// absent key.  Built with -fmad=false: each product is rounded before the sum.  false = int64 overflow.
__host__ __device__ inline bool afs_lq_usage(const i64 *consumed, const int32_t *scale, const i64 *penalty_milli,
                                             const double *res_weight, double lq_weight, int R, double *out) {
  double usage = 0.0;
  for (int r = 0; r < R; r++) {
    i64 v; int s;
    if (!afs_qty_add(consumed[r], scale[r], penalty_milli ? penalty_milli[r] : 0, -3, &v, &s)) return false;
    if (v == 0) continue;
    usage += res_weight[r] * afs_qty_float(v, s);
  }
  *out = usage / lq_weight;
  return true;
}

// ---- decay of consumed usage (CalculateDecayedConsumed, admission_fair_sharing.go:39-66) ---------------------------
// 0.5^x for x >= 0 in plain fp64 operations, restated operation for operation by kueue_b200/drain.py half_pow, so the
// device and the host definition agree bit for bit (Go's math.Pow bits depend on the platform).  Go's Pow for base 0.5:
// x = yi + yf with |yf| <= 0.5, 0.5^yf = exp(yf * Log(0.5)) by the fdlibm reduction and polynomial of Go's exp, then
// ldexp by -yi.  Exactly 1 at 0 and 2^-n at an integer n.  Built with -fmad=false (host: -ffp-contract=off).
__host__ __device__ inline double afs_half_pow(double x) {
  double yi = trunc(x), yf = x - yi;
  if (yf > 0.5) { yf -= 1.0; yi += 1.0; }
  if (yi >= 2048.0) return 0.0;
  const double v = yf * -0.6931471805599453;
  double a;
  if (-3.725290298461914e-09 < v && v < 3.725290298461914e-09) {
    a = 1.0 + v;  // |v| < 2^-28
  } else {
    const double Ln2Hi = 6.93147180369123816490e-01, Ln2Lo = 1.90821492927058770002e-10, Log2e = 1.44269504088896338700e+00;
    const double P1 = 1.66666666666666657415e-01, P2 = -2.77777777770155933842e-03, P3 = 6.61375632143793436117e-05,
                 P4 = -1.65339022054652515390e-06, P5 = 4.13813679705723846039e-08;
    const int k = v < 0 ? (int)(Log2e * v - 0.5) : (int)(Log2e * v + 0.5);
    const double hi = v - (double)k * Ln2Hi, lo = (double)k * Ln2Lo;
    const double r = hi - lo, t = r * r;
    const double c = r - t * (P1 + t * (P2 + t * (P3 + t * (P4 + t * P5))));
    a = ldexp(1.0 - ((lo - (r * c) / (2.0 - c)) - hi), k);
  }
  return ldexp(a, -(int)yi);
}
// Duration.Seconds(): whole seconds and the remainder converted separately
__host__ __device__ inline double afs_seconds(i64 d) { return (double)(d / 1000000000ll) + (double)(d % 1000000000ll) / 1e9; }
// calculateAlphaRate(elapsed, halfLife) on durations in ns: 1 - 0.5^(elapsed / halfLife), 0 when halfLife is 0
__host__ __device__ inline double afs_alpha_of(i64 elapsed_ns, i64 half_life_ns) {
  return half_life_ns == 0 ? 0.0 : 1.0 - afs_half_pow(afs_seconds(elapsed_ns) / afs_seconds(half_life_ns));
}
// Quantity.MilliValue of (v, s) (int64Amount.AsScaledInt64(-3)): a coarser scale multiplies (false on overflow), a finer
// one divides and rounds away from zero (negativeScaleInt64, apimachinery math.go:166-198)
__host__ __device__ inline bool afs_milli(i64 v, int s, i64 *out) {
  if (s >= -3) return afs_scale_up(v, s + 3, out);
  i64 q = v;
  bool frac = false;
  for (int i = 0; i < -3 - s; i++) { frac |= q % 10 != 0; q /= 10; }
  *out = frac ? (v > 0 ? q + 1 : q - 1) : q;
  return true;
}
// consumed = MulByFloat(consumed, 1 - alpha) (+) MulByFloat(admitted, alpha) for one LocalQueue, every resource written
// back as (milli, -3); admitted usage in library units, MilliValue = adm * milli_mul.  *changed: some pair differs.
// false = int64 overflow.
__host__ __device__ inline bool afs_decay(i64 *cons, int32_t *scale, const i64 *adm, const i64 *milli_mul, double alpha, int R,
                                          bool *changed) {
  const double keep = 1.0 - alpha;
  bool ok = true;
  for (int r = 0; r < R; r++) {
    i64 old_m = 0, new_m = 0, sum = 0;
    if (!afs_milli(cons[r], scale[r], &old_m)) { ok = false; continue; }
    const i64 mul = milli_mul[r];
    if (adm[r] > INT64_MAX / mul || adm[r] < -INT64_MAX / mul) { ok = false; continue; }
    new_m = adm[r] * mul;
    if (!afs_add64((i64)((double)old_m * keep), (i64)((double)new_m * alpha), &sum)) { ok = false; continue; }
    if (sum != cons[r] || scale[r] != -3) *changed = true;
    cons[r] = sum; scale[r] = -3;
  }
  return ok;
}

// The admitted-row columns: one half of the double buffer k_drain_compact copies the live rows between ([A_cap] each).
// The first nine are the DevSnap's admitted tables (the first half borrows those upload_impl laid out); every other
// column exists with its block and is null otherwise.
struct AdmRows {
  int32_t *cq, *priority; i64 *ts, *qr_ts, *uid; uint8_t *evicted; int32_t *use_start, *use_fr; i64 *use_qty;
  int32_t *wl;        // pending record of the row, -1 = none (eviction replay or event mode)
  i64 *finish;        // finish time, INT64_MAX = never (event mode); phase says what it holds
  int32_t *lq;        // LocalQueue, -1 = none (decay)
  uint8_t *evicting;  // 1 while the row's eviction is under way, its end in finish (eviction latency)
  uint8_t *phase;     // KB_PH_*: what finish holds (admission checks, WaitForPodsReady, MaximumExecutionTimeSeconds)
  i64 *since;         // Admitted time, INT64_MIN while the checks run (MaximumExecutionTimeSeconds)
  i64 *rc_next;       // time of the row's next reclaim step, INT64_MAX = none (reclaim steps)
  int32_t *rc_cur;    // index of that step
};

struct DrainDev {
  // queues
  int32_t *q_order, *q_start, *cursor; uint8_t *wl_state;  // wl_state: KB_WS_* per pending workload
  int32_t *first_aside;                      // [S] smallest KB_WS_SET_ASIDE position of a segment (its length = none)
  int32_t *flag, *pos;                       // [Q+1] ClusterQueues with work left / their entry position
  int32_t *e_assumed, *e_ncells, *e_adm_off, *e_cell_off;  // [Hcap+1]
  int32_t *counters;                          // [0] entries of the next cycle
  // per pending workload
  int32_t *wl_admit_cycle, *wl_evals; uint8_t *wl_last_decision;
  int32_t *trace_wl; uint8_t *trace_dec; long long trace_off, trace_cap;
  // mutable views of the snapshot tables
  i64 *cq_usage, *wl_last_gen; int8_t *ps_last_tried;
  AdmRows adm;       // the admitted rows (current half)
  int A, AU, cycle;  // admitted workloads / usage cells before this cycle's admissions
  int A_cap, AU_cap; // capacity of the admitted tables (rows / usage cells)
  // eviction replay; adm.wl == nullptr: off
  int32_t *wl_seg, *wl_pos;        // [W] segment of a pending workload / its position in the segment
  int32_t *adm_dead;               // [A_cap] cycle + 1 when the row was evicted in that cycle
  int32_t *root_mark;              // [nRoots] cycle + 1 when the root cohort tree had a victim in that cycle
  int32_t *wl_evictions;           // [W]
  int32_t *row_live, *row_cells, *row_new, *cell_new;  // [A_cap + 1] compaction: flags / cells of live rows / their scans
  uint8_t *wl_has_qr;              // mutable view of wl_has_quota_reservation (may be null)
  // AdmissionFairSharing; seg_start == nullptr: no AFS tables, segment = ClusterQueue
  const int32_t *seg_start;   // [Q+1] first segment of every ClusterQueue
  const int32_t *lq_seg;      // [n_lq] segment of a LocalQueue of an AFS ClusterQueue
  const int32_t *seg_lq;      // [S] LocalQueue of a segment of an AFS ClusterQueue
  const int32_t *afs_cqs;     // [n_afs_cq] ClusterQueues with cq_afs set
  int32_t *head_seg;          // [Q] segment of this cycle's head
  const int32_t *wl_lq; const uint8_t *cq_afs; const double *lq_weight, *res_weight;
  const i64 *milli_mul;
  i64 *lq_consumed; int32_t *lq_consumed_scale;  // device copies: decay rewrites them
  i64 *lq_penalty; double *lq_usage;
  double alpha;
  int n_afs_cq;
  // decay of consumed usage (event mode); lq_last == nullptr: off
  i64 *lq_last;               // [n_lq] LastUpdate of the consumed usage
  i64 *lq_adm;                // [n_lq][R] admitted usage in library units: cells of the LocalQueue's live rows
  unsigned long long *afs_samples;  // [1] samples taken
  i64 half_life_ns, sampling_ns;
  // event mode; adm.finish == nullptr: off
  const i64 *wl_run;               // [W] run time once admitted (< 0 never finishes); null = none finishes
  i64 *wl_admit_ns, *wl_finish_ns; // [W]
  i64 *clock;                      // [0] t_{c+1} of the boundary, [1] E (INT64_MAX = none; reset by k_drain_ev_next)
  const u64 *arr_key;              // [n_arr] creation times (sign flipped) of the ABSENT workloads, ascending
  const int32_t *arr_order;        // [n_arr] their indices, ties by index
  int n_arr;
  int32_t *wl_class;               // [W] (ClusterQueue, hash) class of a BestEffortFIFO workload with a known hash, -1
  const int32_t *cq_class_start;   // [Q+1] classes of a ClusterQueue
  uint8_t *class_nofit;            // [classes] in the ClusterQueue's NoFit set; null = no arrivals or no hashes
  // eviction latency (event mode); wl_evict == nullptr: off
  const i64 *wl_evict;             // [W] time from a workload's eviction until its quota is released
  // sticky workload; cq_sticky == nullptr: off
  int32_t *cq_sticky;              // [Q] pending index of each ClusterQueue's sticky workload, -1 = none
  // admission checks (event mode); wl_check == nullptr: off
  const i64 *wl_check;             // [W] time from a reservation to the attempt's verdict
  int32_t *wl_fail, *wl_retries;   // [W] failures left (INT32_MAX = all) / RetryCount
  i64 *wl_qts;                     // [W] queue-order timestamps: the DevSnap's wl_ts
  const i64 *wl_ts0;               // [W] creation timestamps
  i64 *wl_sort_ts;                 // [W] the keys the current order was built with
  i64 *wl_requeue_at;              // [W] RequeueAt of a BACKOFF record
  i64 *wl_ready_ns; uint8_t *wl_deactivated;  // [W]
  i64 check_base_s, check_max_s; int check_limit;
  // WaitForPodsReady (event mode; the requeue state above is allocated with it); wl_pr == nullptr: off
  const i64 *wl_pr;                // [W] Admitted -> PodsReady delay of a ready attempt
  int32_t *wl_pr_fail, *wl_pr_count;  // [W] failures left (INT32_MAX = all) / RequeueState.Count
  i64 *wl_pr_at, *wl_pr_prev;      // [W] PodsReady time of the last attempt that reaches it / the value before it
  i64 pr_timeout, pr_base_s, pr_max_s; int pr_limit, pr_creation;
  // MaximumExecutionTimeSeconds (event mode; adm.phase and wl_deactivated are allocated with it); wl_max_exec == nullptr:
  // off.  wl_deactivated then holds the reason (KB_DR_*).
  const int32_t *wl_max_exec;      // [W] limit in seconds, 0 = nil
  int32_t *wl_exec_acc;            // [W] accumulated seconds, -1 = nil
  // quota changes (event mode); qc_ns == nullptr: off.  The host works out which edits change nothing, the root and
  // the tree of every other one (the rows change only through the edits, in table order).
  const i64 *qc_ns;                // [n_qc] edit times, non-decreasing
  const int32_t *qc_node;          // [n_qc] edited node
  const i64 *qc_nominal, *qc_blimit, *qc_llimit;  // [n_qc][FR] the node's new rows
  const int32_t *qc_root;          // [n_qc] root slot of the node's tree, -1 = the edit changes nothing
  const int32_t *qc_tree;          // [n_qc] cohort tree of the tree-local tables to refresh, -1 = none
  const int32_t *qc_tree_next;     // [n_qc] the next edit that refreshes the same tree (n_qc = none): one refresh per tree
  const int32_t *qc_cq_start, *qc_cq;  // [nRoots+1] / [Q] the ClusterQueues of every root tree
  const int32_t *qc_blob_gen;      // [Q] byte offset of the ClusterQueue's generation in tree_blob, -1 = not in a tree
  int n_qc;
  // deactivation / reactivation edits (event mode); ac_ns == nullptr: off.  wl_deactivated holds the reason (KB_DR_*).
  const i64 *ac_ns;                // [n_ac] edit times, non-decreasing
  const int32_t *ac_wl;            // [n_ac] record
  const uint8_t *ac_on;            // [n_ac] 0 = stop, 1 = resume
  const int32_t *ac_next, *ac_prev;  // [n_ac] the record's next / previous edit (n_ac / -1 = none)
  int32_t *wl_ac_from;             // [W] the edit a deferred record continues from (values before the boundary: none)
  i64 *wl_stop;                    // [W] stop time of an active row-holding record at this boundary, INT64_MAX = none
  i64 *wl_gone;                    // [W] time its row went at this boundary, INT64_MIN = none
  int n_ac;
  // reclaim steps (event mode); wl_rc_start == nullptr: off.  D.ps_count / ps_req / wl_sched_hash are the records'
  // mutable counts and requests after reclaim.
  const int32_t *wl_rc_start;      // [W+1] CSR of each record's steps
  const i64 *rc_after;             // [n_rc] time of the step after the run starts
  const int32_t *rc_ps, *rc_remaining;  // [n_rc] podset row / its count after the step
  const i64 *rc_hash;              // [n_rc] the record's scheduling hash after the step; null = 0
  const int32_t *rc_class;         // [n_rc] NoFit class of that hash (wl_class), -1 = none
  int32_t *ps_adm_cnt;             // [P] the held row's PodSetAssignment.Count
  int8_t *ps_adm_fl;               // [P][R] its flavors, -1 = none
  i64 *ps_adm_use;                 // [P][R] its ResourceUsage
  const int32_t *rc_blob_gen;      // [Q] byte offset of the ClusterQueue's generation in tree_blob, -1 = not in a tree
};
// wl_deactivated: 0, or the reason a record was deactivated (kb_drain_out.wl_deactivation_reason)
enum { KB_DR_REJECTED = 1, KB_DR_REQUEUING_LIMIT = 2, KB_DR_MAX_EXEC = 3, KB_DR_USER = 4 };
// counters of a boundary: [1] evictions (issued, with latency), [2] / [3] rows / cells after the compaction, [4]
// evictions completed (latency), [5] capacity flag; event mode: [6] completions, [7] arrivals, [8] end flag, [9] / [10]
// arrived prefix of arr_order [lo, hi); admission checks: [11] the stamp (cycle + 1) of the last boundary that needs a
// re-sort, [12] / [13] / [14] Ready / Retry / Rejected verdicts since the start (the host takes differences: no memset);
// WaitForPodsReady: [15] / [16] timeouts that requeue / deactivate since the start, likewise; MaximumExecutionTimeSeconds:
// [17] deactivations since the start, [18] KBS_EXEC_OVERFLOW once an accumulated time leaves int32 (never cleared);
// quota changes: [19] / [20] the edits of this boundary [lo, hi) (hi = edits applied since the start); deactivation:
// [21] / [22] stops / resumes that changed the state since the start, [23] / [24] the edits of this boundary [lo, hi);
// reclaim steps: [25] steps that lowered a count since the start
enum { KB_DC_EVICTED = 1, KB_DC_ROWS = 2, KB_DC_CELLS = 3, KB_DC_EVICT_DONE = 4, KB_DC_FULL = 5,
       KB_DC_FINISHED = 6, KB_DC_ARRIVED = 7, KB_DC_END = 8, KB_DC_ARR_LO = 9, KB_DC_ARR_HI = 10,
       KB_DC_RESORT = 11, KB_DC_CHECK_READY = 12, KB_DC_CHECK_RETRY = 13, KB_DC_CHECK_REJECTED = 14,
       KB_DC_PR_TIMEOUT = 15, KB_DC_PR_DEACTIVATED = 16, KB_DC_EXEC_DEACTIVATED = 17, KB_DC_EXEC_STATUS = 18,
       KB_DC_QC_LO = 19, KB_DC_QC_HI = 20, KB_DC_STOPPED = 21, KB_DC_RESUMED = 22, KB_DC_AC_LO = 23, KB_DC_AC_HI = 24,
       KB_DC_RECLAIMS = 25 };

__device__ __forceinline__ int drain_seg0(const DrainDev &X, int cq) { return X.seg_start ? X.seg_start[cq] : cq; }
__device__ __forceinline__ int drain_seg1(const DrainDev &X, int cq) { return X.seg_start ? X.seg_start[cq + 1] : cq + 1; }

// sort keys of queueOrderingFunc (cluster_queue.go:636-685): LSD passes uid, timestamp, (ClusterQueue | priority desc)
__global__ void k_drain_keys_uid(DevSnap D, u64 *keys, int32_t *vals) {
  int w = blockIdx.x * blockDim.x + threadIdx.x;
  if (w >= D.W) return;
  keys[w] = (u64)D.wl_uid[w] ^ 0x8000000000000000ull;
  vals[w] = w;
}
__global__ void k_drain_keys_ts(DevSnap D, const int32_t *vals, u64 *keys) {
  int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= D.W) return;
  keys[i] = (u64)D.wl_ts[vals[i]] ^ 0x8000000000000000ull;
}
// the segment of workload w: its ClusterQueue's, or its LocalQueue's where the ClusterQueue's queue is split by LocalQueue
__device__ __forceinline__ int drain_wl_seg(const DevSnap &D, const DrainDev &X, int w) {
  const int cq = D.wl_cq[w];
  return (X.seg_start && X.cq_afs[cq]) ? X.lq_seg[X.wl_lq[w]] : drain_seg0(X, cq);
}
// third pass: (segment | priority desc)
__global__ void k_drain_keys_cq(DevSnap D, DrainDev X, const int32_t *vals, u64 *keys, int32_t *q_count) {
  int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= D.W) return;
  const int w = vals[i], seg = drain_wl_seg(D, X, w);
  keys[i] = ((u64)seg << 32) | (u64)(~((unsigned)D.wl_priority[w] ^ 0x80000000u));  // higher priority first
  atomicAdd(&q_count[seg], 1);
}
enum { KB_WS_QUEUED = 0, KB_WS_SET_ASIDE = 1, KB_WS_HELD = 2, KB_WS_ABSENT = 3, KB_WS_FINISHED = 4, KB_WS_BACKOFF = 5,
       KB_WS_DEACTIVATED = 6 };
__global__ void k_drain_init(DevSnap D, DrainDev X, int S) {
  int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < D.W) { X.wl_state[i] = KB_WS_QUEUED; X.wl_admit_cycle[i] = -1; X.wl_evals[i] = 0; X.wl_last_decision[i] = 0xff; }
  if (i < D.W && X.wl_evictions) X.wl_evictions[i] = 0;
  if (i < S) { X.cursor[i] = 0; X.first_aside[i] = X.q_start[i + 1] - X.q_start[i]; }
}
// replay: the records named by adm_wl hold quota (out of every queue); segment and position of every workload
__global__ void k_drain_init_replay(DevSnap D, DrainDev X, int n_adm) {
  int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n_adm) X.wl_state[X.adm.wl[i]] = KB_WS_HELD;
  if (i < D.W) {
    const int w = X.q_order[i], seg = drain_wl_seg(D, X, w);
    X.wl_seg[w] = seg; X.wl_pos[w] = i - X.q_start[seg];
  }
}
// the cursor of segment s past the workloads that left the queue, at its first QUEUED one
__device__ __forceinline__ void drain_advance(const DrainDev &X, int s) {
  const int qs = X.q_start[s], qn = X.q_start[s + 1] - qs;
  int cur = X.cursor[s];
  while (cur < qn && X.wl_state[X.q_order[qs + cur]] != KB_WS_QUEUED) cur++;
  X.cursor[s] = cur;
}
// every segment's cursor (the start of a drain, after a re-sort or the edits of a boundary)
__global__ void k_drain_advance(DrainDev X, int S) {
  int s = blockIdx.x * blockDim.x + threadIdx.x;
  if (s < S) drain_advance(X, s);
}

// heads of the next cycle (queues.Heads manager.go:770-794): one per ClusterQueue with work left, in ClusterQueue order.
// Thread per ClusterQueue of one segment; the AFS ClusterQueues are k_drain_afs_heads'.
__global__ void k_drain_flag(DevSnap D, DrainDev X) {
  int q = blockIdx.x * blockDim.x + threadIdx.x;
  if (q >= D.Q) return;
  if (X.seg_start && X.cq_afs[q]) return;
  int s = drain_seg0(X, q);
  X.flag[q] = X.cursor[s] < X.q_start[s + 1] - X.q_start[s];
  if (X.head_seg) X.head_seg[q] = s;
}

// (usage, -priority, timestamp, UID) of a segment head; seg < 0 = no candidate
struct AfsHead { double u; i64 ts, uid; int prio, seg; };
__device__ __forceinline__ bool afs_before(const AfsHead &a, const AfsHead &b) {
  if (a.seg < 0 || b.seg < 0) return a.seg >= 0 && b.seg < 0;
  const bool an = isnan(a.u), bn = isnan(b.u);  // cmp.Compare: NaN sorts first, two NaNs are equal
  if (an != bn) return an;
  if (!an && a.u != b.u) return a.u < b.u;
  if (a.prio != b.prio) return a.prio > b.prio;
  if (a.ts != b.ts) return a.ts < b.ts;
  if (a.uid != b.uid) return a.uid < b.uid;
  return a.seg < b.seg;
}
// head of an AFS ClusterQueue (queueOrderingFunc with enableAdmissionFs, cluster_queue.go:636-685): one warp per
// ClusterQueue, lanes stride its LocalQueue segments and reduce by shuffles
__global__ void k_drain_afs_heads(DevSnap D, DrainDev X) {
  const int wid = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, lane = threadIdx.x & 31;
  if (wid >= X.n_afs_cq) return;
  const int q = X.afs_cqs[wid];
  AfsHead best{0.0, 0, 0, 0, -1};
  for (int s = X.seg_start[q] + lane; s < X.seg_start[q + 1]; s += 32) {
    const int c = X.cursor[s];
    if (c >= X.q_start[s + 1] - X.q_start[s]) continue;
    const int w = X.q_order[X.q_start[s] + c];
    AfsHead h{X.lq_usage[X.seg_lq[s]], D.wl_ts[w], D.wl_uid[w], D.wl_priority[w], s};
    if (afs_before(h, best)) best = h;
  }
  for (int o = 16; o > 0; o >>= 1) {
    AfsHead h;
    h.u = __shfl_xor_sync(0xffffffffu, best.u, o);
    h.ts = __shfl_xor_sync(0xffffffffu, best.ts, o);
    h.uid = __shfl_xor_sync(0xffffffffu, best.uid, o);
    h.prio = __shfl_xor_sync(0xffffffffu, best.prio, o);
    h.seg = __shfl_xor_sync(0xffffffffu, best.seg, o);
    if (afs_before(h, best)) best = h;
  }
  if (lane == 0) { X.flag[q] = best.seg >= 0; X.head_seg[q] = best.seg; }
}

__global__ void k_drain_heads(DevSnap D, DrainDev X, int32_t *heads) {
  int q = blockIdx.x * blockDim.x + threadIdx.x;
  if (q >= D.Q) return;
  if (X.flag[q]) {  // a queued sticky workload implies cursor < length: the flag is set
    int s = X.head_seg ? X.head_seg[q] : q;
    int w = X.q_order[X.q_start[s] + X.cursor[s]];
    if (X.cq_sticky) { const int sw = X.cq_sticky[q]; if (sw >= 0 && X.wl_state[sw] == KB_WS_QUEUED) w = sw; }
    heads[X.pos[q]] = w;
  }
  if (q == 0) X.counters[0] = X.pos[D.Q];
}

__device__ __forceinline__ bool drain_covers_pods(const DevSnap &D, int cq) {
  if (D.pods_res < 0) return false;
  for (int g = D.cq_rg_start[cq]; g < D.cq_rg_start[cq + 1]; g++) if (D.rg_res_mask[g] & (1u << D.pods_res)) return true;
  return false;
}
__device__ __forceinline__ i64 drain_request(const DevSnap &D, int row, int r, int count, bool covers_pods) {  // ScaledTo workload.go:258-275
  if (covers_pods && r == D.pods_res) return count;
  i64 q = D.ps_req[(size_t)row * D.R + r];
  int full = D.ps_count[row];
  if (full != 0 && full != count) q = q / full * count;
  return q;
}

// decisions of the cycle -> LastAssignment, queue movement, per-entry admission bookkeeping
__global__ void k_drain_apply(DevSnap D, DrainDev X) {
  int e = blockIdx.x * blockDim.x + threadIdx.x;
  if (e >= D.H) return;
  const int R = D.R;
  int wl = D.heads[e], cq = D.wl_cq[wl];
  int dec = D.decision[e];
  X.wl_last_decision[wl] = (uint8_t)dec;
  X.wl_evals[wl]++;
  if (X.trace_wl && X.trace_off + e < X.trace_cap) { X.trace_wl[X.trace_off + e] = wl; X.trace_dec[X.trace_off + e] = (uint8_t)dec; }
  const bool ok = dec == KB_DEC_ASSUMED;
  const int ps0 = D.wl_ps_start[wl], ps1 = D.wl_ps_start[wl + 1];
  int ncell = 0;
  bool pending_flavors = false;
  if (ok) {
    X.wl_admit_cycle[wl] = X.cycle;
    X.wl_state[wl] = KB_WS_HELD;
    for (int row = ps0; row < ps1; row++)  // distinct flavor-resource cells of Assignment.Usage
      for (int r = 0; r < R; r++) {
        int f = D.ps_flavor[(size_t)row * R + r];
        if (f < 0) continue;
        bool first = true;  // same cell = same resource and same flavor in an earlier podset
        for (int prow = ps0; prow < row; prow++) if (D.ps_flavor[(size_t)prow * R + r] == f) { first = false; break; }
        if (first) ncell++;
      }
  } else if (dec == KB_DEC_PREEMPTING) {
    X.wl_last_gen[wl] = -1;  // "the next attempt should try all the flavors" scheduler.go:345
  } else {
    X.wl_last_gen[wl] = D.cq_generation[cq];  // e.LastAssignment = &e.assignment.LastState scheduler.go:494
    for (int i = ps0 * R; i < ps1 * R; i++) { int8_t t = D.ps_tried[i]; X.ps_last_tried[i] = t; if (t != -1) pending_flavors = true; }  // PendingFlavors workload.go:163-176
  }
  X.e_assumed[e] = ok; X.e_ncells[e] = ncell;
  // ---- queue movement (cluster_queue.go:362-425,609-633)
  const bool strict = D.cq_strategy[cq] == KB_QUEUE_STRICT_FIFO;
  if (X.cq_sticky) {  // delete (cluster_queue.go:330-340) on admission; RequeueIfNotPresent with PendingPreemption (:609-619)
    if (ok) { if (X.cq_sticky[cq] == wl) X.cq_sticky[cq] = -1; }
    else if (dec == KB_DEC_PREEMPTING && !strict) X.cq_sticky[cq] = wl;
  }
  const bool inadmissible = (dec == KB_DEC_NOFIT || dec == KB_DEC_PREEMPT_NO_TARGETS) && !pending_flavors;
  const int hs = X.head_seg ? X.head_seg[cq] : cq, s0 = drain_seg0(X, cq), s1 = drain_seg1(X, cq);
  const int hp = X.cq_sticky ? X.wl_pos[wl] : X.cursor[hs];  // the head's position: a sticky head may lie past the cursor
  const bool bulk = dec == KB_DEC_NOFIT && !strict && D.wl_sched_hash && D.wl_sched_hash[wl] != 0;
  if (bulk) {  // handleInadmissibleHash :408-425: every queued workload of the class but the head, in every segment
    const i64 hsh = D.wl_sched_hash[wl];
    if (X.class_nofit) X.class_nofit[X.wl_class[wl]] = 1;  // noFitSchedulingHashes.Insert (:414)
    for (int s = s0; s < s1; s++) {
      const int qs = X.q_start[s], qn = X.q_start[s + 1] - qs;
      for (int p = X.cursor[s]; p < qn; p++) {
        const int w2 = X.q_order[qs + p];
        if (w2 != wl && D.wl_sched_hash[w2] == hsh && X.wl_state[w2] == KB_WS_QUEUED) { X.wl_state[w2] = KB_WS_SET_ASIDE; X.first_aside[s] = min(X.first_aside[s], p); }
      }
    }
  }
  if (inadmissible && !strict) { X.wl_state[wl] = KB_WS_SET_ASIDE; X.first_aside[hs] = min(X.first_aside[hs], hp); }
  for (int s = s0; s < s1; s++)  // the cursor past the workloads that left the queue, the head among them
    if (s == hs || bulk) drain_advance(X, s);
}

// RequeueState cleared: Count 0, no RequeueAt
__device__ __forceinline__ void drain_clear_requeue(const DrainDev &X, int w) {
  if (X.wl_pr) X.wl_pr_count[w] = 0;
  if (X.wl_requeue_at) X.wl_requeue_at[w] = INT64_MIN;
}
// a PodsReady attempt of record w still waiting at t is dropped: not counted, no failure used
__device__ __forceinline__ void drain_drop_attempt(const DrainDev &X, int w, i64 t) {
  if (X.wl_pr && X.wl_pr_at[w] > t) X.wl_pr_at[w] = X.wl_pr_prev[w];
}
// deactivation for MaximumExecutionTimeExceeded: acc nil, RequeueState cleared (a BACKOFF-bound record is DEACTIVATED
// at its release instead)
__device__ __forceinline__ void drain_exec_deactivate(const DrainDev &X, int w) {
  X.wl_deactivated[w] = KB_DR_MAX_EXEC;
  X.wl_exec_acc[w] = -1;
  drain_clear_requeue(X, w);
  atomicAdd(&X.counters[KB_DC_EXEC_DEACTIVATED], 1);
}
// release at t of row a (record w): with an Admitted time, a deadline at or before t deactivates a record not
// deactivated yet (rule 4), then the attempt's seconds join acc.  Returns whether it deactivated the record.
__device__ __forceinline__ bool drain_exec_release(const DrainDev &X, int a, int w, i64 t) {
  const i64 A = X.adm.since[a];
  if (A == INT64_MIN) return false;
  const bool deact = X.wl_max_exec[w] > 0 && X.wl_deactivated[w] == 0 && kb_exec_deadline(A, X.wl_max_exec[w], X.wl_exec_acc[w]) <= t;
  if (deact) drain_exec_deactivate(X, w);
  const i64 d = kb_exec_seconds(t - A), acc = X.wl_exec_acc[w];
  const i64 sum = acc < 0 ? d : acc + d;
  if (d < 0 || sum > INT32_MAX) atomicOr((unsigned *)&X.counters[KB_DC_EXEC_STATUS], KBS_EXEC_OVERFLOW);
  else X.wl_exec_acc[w] = (int32_t)sum;
  return deact;
}

// ---- reclaim steps ------------------------------------------------------------------------------------------------
// the run of row a (record w) starts at S: its steps replay from the first
__device__ __forceinline__ void drain_rc_begin(const DrainDev &X, int a, int w, i64 S) {
  const int i = X.wl_rc_start[w];
  X.adm.rc_cur[a] = i;
  X.adm.rc_next[a] = i < X.wl_rc_start[w + 1] ? drain_sat_add(S, X.rc_after[i]) : INT64_MAX;
}
// row a can take a step: not evicting, phase running (its run started: adm.rc_next is INT64_MAX otherwise)
__device__ __forceinline__ bool drain_rc_live(const DrainDev &X, int a) {
  if (X.adm.evicting && X.adm.evicting[a]) return false;
  return !X.adm.phase || X.adm.phase[a] == KB_PH_RUN || X.adm.phase[a] == KB_PH_EXPIRE;
}
// the steps of running row a due at or before lim, in time order (rule 4 of kb_run_drain): a step that lowers podset p
// from c to r scales the record's requests to r pods and the row's usage of p to U0 / n * min(r, n) per resource; the
// difference leaves the row's cells, the ClusterQueue usage and the LocalQueue's admitted usage (integer atomics).  The
// steps of one instant are one update: generation + 1 (the cycle's copy and the tree block's), root tree marked.
__device__ void drain_reclaim(const DevSnap &D, const DrainDev &X, int a, i64 lim) {
  i64 t = X.adm.rc_next[a];
  if (t > lim) return;
  const int w = X.adm.wl[a], cq = X.adm.cq[a], R = D.R, i1 = X.wl_rc_start[w + 1];
  int i = X.adm.rc_cur[a], n = 0;
  const i64 S = t - X.rc_after[i];  // t <= lim < INT64_MAX: not saturated
  int32_t *cnt = const_cast<int32_t *>(D.ps_count);
  i64 *req = const_cast<i64 *>(D.ps_req), *hash = const_cast<i64 *>(D.wl_sched_hash);
  while (i < i1 && t <= lim) {
    bool lowered = false;
    for (; i < i1 && drain_sat_add(S, X.rc_after[i]) == t; i++) {
      const int p = X.rc_ps[i], rem = X.rc_remaining[i], c = cnt[p];
      if (rem >= c) continue;  // counts only go down
      for (int r = 0; r < R; r++) req[(size_t)p * R + r] = req[(size_t)p * R + r] / c * rem;
      const int na = X.ps_adm_cnt[p];
      for (int r = 0; r < R && na > 0; r++) {
        const int f = X.ps_adm_fl[(size_t)p * R + r];
        if (f < 0) continue;
        const i64 u = X.ps_adm_use[(size_t)p * R + r] / na, d = u * min(rem, na) - u * min(c, na);
        if (d == 0) continue;
        const int fr = f * R + r;
        for (int k = X.adm.use_start[a]; k < X.adm.use_start[a + 1]; k++)
          if (X.adm.use_fr[k] == fr) { X.adm.use_qty[k] += d; break; }
        atomicAdd((unsigned long long *)&X.cq_usage[(size_t)cq * D.FR + fr], (unsigned long long)d);
        if (X.lq_last && X.adm.lq[a] >= 0 && X.cq_afs[cq])
          atomicAdd((unsigned long long *)&X.lq_adm[(size_t)X.adm.lq[a] * R + r], (unsigned long long)d);
      }
      cnt[p] = rem;
      if (hash) { hash[w] = X.rc_hash ? X.rc_hash[i] : 0; if (X.wl_class) X.wl_class[w] = X.rc_class[i]; }
      lowered = true;
      n++;
    }
    if (lowered) {  // AddOrUpdateWorkload -> deleteWorkload: AllocatableResourceGeneration + 1; the root tree requeued
      atomicAdd((unsigned long long *)&D.cq_generation[cq], 1ull);
      if (X.rc_blob_gen[cq] >= 0) atomicAdd((unsigned long long *)(D.tree_blob + X.rc_blob_gen[cq]), 1ull);
      X.root_mark[D.root_slot[cq]] = X.cycle + 1;
    }
    t = i < i1 ? drain_sat_add(S, X.rc_after[i]) : INT64_MAX;
  }
  X.adm.rc_cur[a] = i; X.adm.rc_next[a] = t;
  if (n) atomicAdd(&X.counters[KB_DC_RECLAIMS], n);
}

// row a (record w) is Admitted at t (the reservation without a check delay, or a Ready verdict): the run clock or the
// PodsReady attempt starts (kb_pr_attempt; a ready one moves the PodsReady time), the reclaim steps with the run (at
// PodsReady of a ready attempt), and the MaximumExecutionTimeSeconds deadline may come first
__device__ __forceinline__ void drain_admitted(const DrainDev &X, int a, int w, i64 t) {
  if (X.wl_ready_ns) X.wl_ready_ns[w] = t;
  const i64 run = X.wl_run ? X.wl_run[w] : -1;
  DrainFin f{run < 0 ? INT64_MAX : drain_sat_add(t, run), KB_PH_RUN};
  if (X.wl_pr) {
    const i64 d = X.wl_pr[w];
    f = kb_pr_attempt(t, d, X.wl_pr_fail[w] > 0, X.pr_timeout, run);
    if (f.ph == KB_PH_RUN) { X.wl_pr_prev[w] = X.wl_pr_at[w]; X.wl_pr_at[w] = drain_sat_add(t, d); }
  }
  if (X.wl_rc_start) {
    if (f.ph == KB_PH_RUN) drain_rc_begin(X, a, w, X.wl_pr ? X.wl_pr_at[w] : t);
    else X.adm.rc_next[a] = INT64_MAX;
  }
  if (X.wl_max_exec) {
    X.adm.since[a] = t;
    f = kb_exec_clip(f, t, X.wl_max_exec[w], X.wl_exec_acc[w], INT64_MIN);
  }
  if (X.adm.phase) X.adm.phase[a] = f.ph;
  X.adm.finish[a] = f.fin;
}
// admitted entries join the admitted tables (cache.AssumeWorkload), appended at X.A / X.AU, and the ClusterQueue usage
__global__ void k_drain_admit(DevSnap D, DrainDev X, i64 qr_ts) {
  int e = blockIdx.x * blockDim.x + threadIdx.x;
  if (e >= D.H || !X.e_assumed[e]) return;
  const int R = D.R;
  int wl = D.heads[e], cq = D.wl_cq[wl];
  int a = X.A + X.e_adm_off[e];
  int c0 = X.AU + X.e_cell_off[e];
  if (a >= X.A_cap || c0 + X.e_ncells[e] > X.AU_cap) { atomicOr(&X.counters[KB_DC_FULL], 1); return; }  // nothing past the end
  if (X.adm.wl) X.adm.wl[a] = wl;
  if (X.adm.lq) X.adm.lq[a] = X.wl_lq[wl];
  X.adm.cq[a] = cq; X.adm.priority[a] = D.wl_priority[wl]; X.adm.ts[a] = X.wl_ts0 ? X.wl_ts0[wl] : D.wl_ts[wl]; X.adm.qr_ts[a] = qr_ts;
  X.adm.uid[a] = D.wl_uid[wl]; X.adm.evicted[a] = 0;
  if (X.adm.evicting) X.adm.evicting[a] = 0;
  X.adm.use_start[a] = c0;
  if (X.adm.finish) {  // checks or PodsReady: the reservation resets Evicted; a check delay starts an attempt, 0 is Ready at once
    if (X.wl_qts) X.wl_qts[wl] = X.wl_ts0[wl];
    const i64 chk = X.wl_check ? X.wl_check[wl] : 0;
    if (chk > 0) {  // not Admitted while the checks run: the verdict time in the finish column
      X.adm.phase[a] = KB_PH_CHECK;
      X.adm.finish[a] = drain_sat_add(qr_ts, chk);
      if (X.wl_rc_start) X.adm.rc_next[a] = INT64_MAX;
      if (X.wl_max_exec) X.adm.since[a] = INT64_MIN;
    } else {
      drain_admitted(X, a, wl, qr_ts);
    }
    X.wl_admit_ns[wl] = qr_ts;
  }
  const bool covers_pods = drain_covers_pods(D, cq);
  const int ps0 = D.wl_ps_start[wl], ps1 = D.wl_ps_start[wl + 1];
  int n = 0;
  for (int row = ps0; row < ps1; row++)
    for (int r = 0; r < R; r++) {
      int f = D.ps_flavor[(size_t)row * R + r];
      if (X.wl_rc_start) {  // the admission's PodSetAssignment, read by the reclaim steps
        if (r == 0) X.ps_adm_cnt[row] = D.ps_count_out[row];
        X.ps_adm_fl[(size_t)row * R + r] = (int8_t)f;
        X.ps_adm_use[(size_t)row * R + r] = f < 0 ? 0 : drain_request(D, row, r, D.ps_count_out[row], covers_pods);
      }
      if (f < 0) continue;
      int fr = f * R + r;
      i64 q = drain_request(D, row, r, D.ps_count_out[row], covers_pods);
      int j = 0;
      while (j < n && X.adm.use_fr[c0 + j] != fr) j++;
      if (j == n) { X.adm.use_fr[c0 + n] = fr; X.adm.use_qty[c0 + n] = 0; n++; }
      X.adm.use_qty[c0 + j] += q;
    }
  X.adm.use_start[a + 1] = c0 + n;
  for (int j = 0; j < n; j++) X.cq_usage[(size_t)cq * D.FR + X.adm.use_fr[c0 + j]] += X.adm.use_qty[c0 + j];  // one entry per ClusterQueue
  if (X.seg_start && X.cq_afs[cq]) {
    // entry penalty (scheduler.go:727-742,946-960; CalculateEntryPenalty + MulByFloat): per resource of SumTotalRequests
    // (the full TotalRequests, partial admission does not reduce it), int64(float64(MilliValue) * alpha) milli-units,
    // pushed into the LocalQueue's penalties (AfsEntryPenalties.Push: Quantity.Add at scale -3).  A ClusterQueue admits
    // one entry per cycle and a LocalQueue belongs to one ClusterQueue: one writer per LocalQueue, no atomics.
    // With decay (workload_controller.go:965-971,1030-1056): the cells join the LocalQueue's admitted usage, consumed
    // decays over t_c - LastUpdate, LastUpdate = t_c, and the penalty goes into consumed instead of the pending ones.
    const int lq = X.wl_lq[wl];
    i64 *pen = X.lq_penalty + (size_t)lq * R;
    i64 *cons = X.lq_consumed + (size_t)lq * R;
    int32_t *csc = X.lq_consumed_scale + (size_t)lq * R;
    bool bad = false;
    if (X.lq_last) {
      i64 *adm = X.lq_adm + (size_t)lq * R;
      for (int j = 0; j < n; j++) adm[X.adm.use_fr[c0 + j] % R] += X.adm.use_qty[c0 + j];
      bool changed = false;
      bad |= !afs_decay(cons, csc, adm, X.milli_mul, afs_alpha_of(qr_ts - X.lq_last[lq], X.half_life_ns), R, &changed);
      X.lq_last[lq] = qr_ts;
    }
    for (int r = 0; r < R; r++) {
      i64 total = 0;
      for (int row = ps0; row < ps1; row++)
        if (D.ps_req_mask[row] & (1u << r)) bad |= !afs_add64(total, D.ps_req[(size_t)row * R + r], &total);
      if (total == 0) continue;
      const i64 mul = X.milli_mul[r];
      if (total > INT64_MAX / mul || total < -INT64_MAX / mul) { bad = true; continue; }
      const i64 delta = (i64)((double)(total * mul) * X.alpha);
      if (X.lq_last) { int s; bad |= !afs_qty_add(cons[r], csc[r], delta, -3, &cons[r], &s); csc[r] = s; }
      else bad |= !afs_add64(pen[r], delta, &pen[r]);
    }
    double u = 0.0;
    bad |= !afs_lq_usage(cons, csc, pen, X.res_weight, X.lq_weight[lq], R, &u);
    X.lq_usage[lq] = u;
    if (bad) atomicOr(D.status, KBS_AFS_OVERFLOW);
  }
}

// ---- eviction replay ---------------------------------------------------------------------------------------------
// the record of an evicted row returns to its queue with LastAssignment nil (the eviction completed)
// (a released record: LastAssignment nil, no reservation)
__device__ __forceinline__ void drain_forget(const DevSnap &D, const DrainDev &X, int w) {
  X.wl_last_gen[w] = -1;
  for (int i = D.wl_ps_start[w] * D.R; i < D.wl_ps_start[w + 1] * D.R; i++) X.ps_last_tried[i] = -1;
  if (X.wl_has_qr) X.wl_has_qr[w] = 0;
  X.wl_admit_cycle[w] = -1;
}
// a record entering its queue with a queue-order timestamp other than the key its position was sorted by stamps the
// boundary for a re-sort
__device__ __forceinline__ void drain_mark_resort(const DrainDev &X, int w) {
  if (X.wl_sort_ts && X.wl_sort_ts[w] != X.wl_qts[w]) X.counters[KB_DC_RESORT] = X.cycle + 1;
}
__device__ __forceinline__ void drain_release(const DevSnap &D, const DrainDev &X, int w) {
  X.wl_state[w] = KB_WS_QUEUED;
  drain_forget(D, X, w);
  atomicMin(&X.cursor[X.wl_seg[w]], X.wl_pos[w]);
  drain_mark_resort(X, w);
}
// record w joins its queue (PushOrUpdate, cluster_queue.go:288-293): the cursor moves back to it, or in a BestEffortFIFO
// ClusterQueue a known hash in the NoFit set sets it aside
__device__ __forceinline__ void drain_enqueue(const DrainDev &X, int w) {
  const int s = X.wl_seg[w], p = X.wl_pos[w];
  if (X.class_nofit && X.wl_class[w] >= 0 && X.class_nofit[X.wl_class[w]]) {
    X.wl_state[w] = KB_WS_SET_ASIDE;
    atomicMin(&X.first_aside[s], p);
  } else {
    X.wl_state[w] = KB_WS_QUEUED;
    atomicMin(&X.cursor[s], p);
  }
}
// the cells of row a leave its ClusterQueue's usage (cache.DeleteWorkload) and, with lq and decay, its LocalQueue's
// admitted usage: integer atomics, the order does not matter (several rows of one LocalQueue can go together).  lq is
// false where no AFS row can be: evictions (AFS drains cannot preempt) and check verdicts (checks exclude decay).
__device__ __forceinline__ void drain_uncharge(const DevSnap &D, const DrainDev &X, int a, bool lq) {
  const int cq = X.adm.cq[a], c0 = X.adm.use_start[a], c1 = X.adm.use_start[a + 1];
  for (int c = c0; c < c1; c++)
    atomicAdd((unsigned long long *)&X.cq_usage[(size_t)cq * D.FR + X.adm.use_fr[c]], (unsigned long long)(-X.adm.use_qty[c]));
  if (lq && X.lq_last && X.adm.lq[a] >= 0 && X.cq_afs[cq]) {
    i64 *adm = X.lq_adm + (size_t)X.adm.lq[a] * D.R;
    for (int c = c0; c < c1; c++) atomicAdd((unsigned long long *)&adm[X.adm.use_fr[c] % D.R], (unsigned long long)(-X.adm.use_qty[c]));
  }
}
// row a (record w) becomes an evicting row at t0: it holds its cells until t0 + latency
__device__ __forceinline__ void drain_evict_row(const DrainDev &X, int a, int w, i64 t0) {
  X.adm.evicted[a] = 1;
  X.adm.evicting[a] = 1;
  X.adm.finish[a] = drain_sat_add(t0, X.wl_evict[w]);
}
// sets byte i of a byte column (256-byte aligned, padded) and returns whether it was set: atomicOr on its aligned word
__device__ __forceinline__ bool drain_claim_byte(uint8_t *col, int i) {
  const uintptr_t p = (uintptr_t)(col + i);
  const unsigned bit = 1u << (8 * (unsigned)(p & 3));
  return (atomicOr((unsigned *)(p & ~(uintptr_t)3), bit) & bit) != 0;
}
// every target of every Preempting entry (thread per entry): cells out of its ClusterQueue's usage, row dead, pending record QUEUED with LastAssignment nil, its root tree marked.  With
// latency (wl_evict) the eviction is only issued: a row not evicting yet is claimed once, gets adm_evicted and its end
// time t_c + latency (saturating) in its finish column, and keeps its cells and its record; k_drain_finish releases it.
__global__ void k_drain_evict(DevSnap D, DrainDev X) {
  int e = blockIdx.x * blockDim.x + threadIdx.x;
  if (e >= D.H || D.decision[e] != KB_DEC_PREEMPTING) return;
  const int stamp = X.cycle + 1;
  const int off = D.tgt_off[e], n = D.tgt_cnt[e];
  for (int k = 0; k < n; k++) {
    const int a = D.tgt_pool_adm[off + k], w = X.adm.wl[a];
    if (X.wl_evict) {
      if (drain_claim_byte(X.adm.evicting, a)) continue;  // under way: "Preemption ongoing" (preemption.go:183-186)
      X.adm.evicted[a] = 1;
      X.adm.finish[a] = drain_sat_add(D.now_ns, X.wl_evict[w]);
      if (X.adm.phase) {  // checks running: no pods, the next boundary; a PodsReady attempt waiting for T is dropped
        if (X.adm.phase[a] == KB_PH_CHECK) X.adm.finish[a] = D.now_ns;
        X.adm.phase[a] = KB_PH_RUN;
      }
    } else {
      if (atomicExch(&X.adm_dead[a], stamp) == stamp) continue;  // one eviction per row
      drain_uncharge(D, X, a, false);
      if (X.wl_max_exec && drain_exec_release(X, a, w, D.now_ns)) { drain_forget(D, X, w); X.wl_state[w] = KB_WS_DEACTIVATED; }
      else drain_release(D, X, w);
      X.root_mark[D.root_slot[X.adm.cq[a]]] = stamp;
    }
    drain_drop_attempt(X, w, D.now_ns);  // dropped before PodsReady
    X.wl_evictions[w]++;  // a workload holds at most one row: one writer
    atomicAdd(&X.counters[KB_DC_EVICTED], 1);
  }
}
// inadmissible requeue (thread per ClusterQueue of a marked root): set aside -> queued, cursor back to the first of them
__global__ void k_drain_requeue(DevSnap D, DrainDev X) {
  int q = blockIdx.x * blockDim.x + threadIdx.x;
  if (q >= D.Q || X.root_mark[D.root_slot[q]] != X.cycle + 1) return;
  if (X.class_nofit) for (int k = X.cq_class_start[q]; k < X.cq_class_start[q + 1]; k++) X.class_nofit[k] = 0;  // inadmissible_workloads.go:174
  for (int s = drain_seg0(X, q); s < drain_seg1(X, q); s++) {
    const int qs = X.q_start[s], qn = X.q_start[s + 1] - qs, fa = X.first_aside[s];
    for (int p = fa; p < qn; p++) { const int w = X.q_order[qs + p]; if (X.wl_state[w] == KB_WS_SET_ASIDE) X.wl_state[w] = KB_WS_QUEUED; }
    X.cursor[s] = min(X.cursor[s], fa);
    X.first_aside[s] = qn;
  }
}
// compaction: live flags and cell counts of the rows [0, bound) ([bound] = 0 closes the scans).  The rows are the
// tables the cycle started with, less those stamped dead at this boundary, and the *n_new admissions appended after
// them; rows past those only pad the range.  After a capacity overflow no row is live: not every admission was written.
__global__ void k_drain_live(DrainDev X, int bound, const int32_t *n_new) {
  int a = blockIdx.x * blockDim.x + threadIdx.x;
  if (a > bound) return;
  const bool live = a < bound && a < X.A + (n_new ? *n_new : 0) && !X.counters[KB_DC_FULL] && X.adm_dead[a] != X.cycle + 1;
  X.row_live[a] = live;
  X.row_cells[a] = live ? X.adm.use_start[a + 1] - X.adm.use_start[a] : 0;
}
// row a of I into row n of O, its cells excepted (the caller moves them and writes O.use_start)
__device__ __forceinline__ void drain_copy_row(const AdmRows &I, int a, const AdmRows &O, int n) {
  O.cq[n] = I.cq[a]; O.priority[n] = I.priority[a]; O.ts[n] = I.ts[a]; O.qr_ts[n] = I.qr_ts[a];
  O.uid[n] = I.uid[a]; O.evicted[n] = I.evicted[a]; O.wl[n] = I.wl[a];
  if (I.finish) O.finish[n] = I.finish[a];
  if (I.lq) O.lq[n] = I.lq[a];
  if (I.evicting) O.evicting[n] = I.evicting[a];
  if (I.phase) O.phase[n] = I.phase[a];
  if (I.since) O.since[n] = I.since[a];
  if (I.rc_next) { O.rc_next[n] = I.rc_next[a]; O.rc_cur[n] = I.rc_cur[a]; }
}
// live rows of [0, bound), in order, into the other half O of the double buffer; thread bound writes the totals
__global__ void k_drain_compact(DrainDev X, AdmRows O, int bound) {
  int a = blockIdx.x * blockDim.x + threadIdx.x;
  if (a > bound) return;
  if (a == bound) { O.use_start[X.row_new[a]] = X.cell_new[a]; X.counters[KB_DC_ROWS] = X.row_new[a]; X.counters[KB_DC_CELLS] = X.cell_new[a]; return; }
  if (!X.row_live[a]) return;
  const int n = X.row_new[a], c0 = X.cell_new[a], u0 = X.adm.use_start[a], nc = X.adm.use_start[a + 1] - u0;
  drain_copy_row(X.adm, a, O, n);
  O.use_start[n] = c0;
  for (int c = 0; c < nc; c++) { O.use_fr[c0 + c] = X.adm.use_fr[u0 + c]; O.use_qty[c0 + c] = X.adm.use_qty[u0 + c]; }
}

// ---- event mode ---------------------------------------------------------------------------------------------------
__device__ __forceinline__ i64 ev_time(u64 key) { return (i64)(key ^ 0x8000000000000000ull); }
// first i in [lo, hi) with key[i] > k (the keys up to k are [.., i)); key ascending
template <class K> __device__ __forceinline__ int drain_upper_bound(const K *key, int lo, int hi, K k) {
  while (lo < hi) { const int m = lo + (hi - lo) / 2; if (key[m] <= k) lo = m + 1; else hi = m; }
  return lo;
}
__device__ __forceinline__ int ev_upper_bound(const u64 *key, int lo, int n, i64 t) {  // the creations up to t
  return drain_upper_bound(key, lo, n, (u64)t ^ 0x8000000000000000ull);
}
// sort keys of the arrival order: creation time, then index (the radix sort is stable)
__global__ void k_drain_keys_create(int W, const i64 *create, u64 *keys, int32_t *vals) {
  int w = blockIdx.x * blockDim.x + threadIdx.x;
  if (w >= W) return;
  keys[w] = (u64)create[w] ^ 0x8000000000000000ull;
  vals[w] = w;
}
// start of an event drain: workloads created after now_ns are ABSENT, no admission or finish yet, E = none, and the
// arrived prefix of the arrival order holds the workloads present at the start
__global__ void k_drain_init_events(DevSnap D, DrainDev X, const i64 *create, i64 now_ns) {
  int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i == 0) {
    X.clock[0] = now_ns; X.clock[1] = INT64_MAX; X.clock[2] = INT64_MAX;
    const int lo = X.arr_key ? ev_upper_bound(X.arr_key, 0, X.n_arr, now_ns) : 0;
    X.counters[KB_DC_ARR_LO] = lo; X.counters[KB_DC_ARR_HI] = lo;
  }
  if (i >= D.W) return;
  if (create && create[i] > now_ns) X.wl_state[i] = KB_WS_ABSENT;
  X.wl_admit_ns[i] = INT64_MIN; X.wl_finish_ns[i] = INT64_MAX;
}
// E: the earliest finish of a live row (rows [0, A + *n_new), the ones stamped this boundary excluded) and the next
// creation; warp minimum, one atomic per warp
__global__ void k_drain_ev_min(DrainDev X, int bound, const int32_t *n_new) {
  const int a = blockIdx.x * blockDim.x + threadIdx.x;
  const int n_rows = X.A + (n_new ? *n_new : 0);
  i64 v = INT64_MAX;
  if (a < bound && a < n_rows && X.adm_dead[a] != X.cycle + 1) {
    v = X.adm.finish[a];
    if (X.adm.rc_next && drain_rc_live(X, a)) v = min(v, X.adm.rc_next[a]);  // the row's next reclaim step
  }
  if (a == 0 && X.counters[KB_DC_ARR_HI] < X.n_arr) v = min(v, ev_time(X.arr_key[X.counters[KB_DC_ARR_HI]]));
  if (a == 0 && X.qc_ns && X.counters[KB_DC_QC_HI] < X.n_qc) v = min(v, X.qc_ns[X.counters[KB_DC_QC_HI]]);  // the next edit
  if (a == 0 && X.ac_ns && X.counters[KB_DC_AC_HI] < X.n_ac) v = min(v, X.ac_ns[X.counters[KB_DC_AC_HI]]);
  for (int o = 16; o > 0; o >>= 1) v = min(v, (i64)__shfl_xor_sync(0xffffffffu, (long long)v, o));
  if ((threadIdx.x & 31) == 0 && v < INT64_MAX) atomicMin((long long *)&X.clock[1], (long long)v);
}
// t_{c+1} and the end flag (one thread).  jump: no heads, the clock goes to E.  Otherwise a cycle that admitted or
// evicted steps, a quiet one waits for E; no E ends the drain.  Then the arrived prefix up to t_{c+1}, and the edits
// with a time in (t_c, t_{c+1}] (k_drain_quota applies them).
__global__ void k_drain_ev_next(DrainDev X, i64 t_c, i64 step, int jump, const int32_t *n_new) {
  const i64 E = min(X.clock[1], X.clock[2]);  // [2]: the next RequeueAt (admission checks), INT64_MAX otherwise
  X.clock[2] = INT64_MAX;
  const i64 stepped = drain_sat_add(t_c, step);
  const bool active = !jump && ((n_new && *n_new > 0) || X.counters[KB_DC_EVICTED] > 0);
  i64 tn;
  bool end = false;
  if (jump) { end = E == INT64_MAX; tn = E; }
  else if (active) tn = stepped;
  else { end = E == INT64_MAX; tn = max(stepped, E); }
  X.clock[0] = end ? t_c : tn;
  X.clock[1] = INT64_MAX;
  X.counters[KB_DC_END] = end;
  const int lo = X.counters[KB_DC_ARR_HI];
  X.counters[KB_DC_ARR_LO] = lo;
  X.counters[KB_DC_ARR_HI] = (end || !X.arr_key) ? lo : ev_upper_bound(X.arr_key, lo, X.n_arr, tn);
  if (X.qc_ns) {
    const int qlo = X.counters[KB_DC_QC_HI];
    X.counters[KB_DC_QC_LO] = qlo;
    X.counters[KB_DC_QC_HI] = drain_upper_bound(X.qc_ns, qlo, end ? qlo : X.n_qc, tn);
  }
  if (X.ac_ns) {  // the deactivation / reactivation edits (k_drain_active applies them)
    const int alo = X.counters[KB_DC_AC_HI];
    X.counters[KB_DC_AC_LO] = alo;
    X.counters[KB_DC_AC_HI] = drain_upper_bound(X.ac_ns, alo, end ? alo : X.n_ac, tn);
  }
}
// a stop at d of active record w holding row a (before the row leaves): RequeueState cleared, a waiting PodsReady
// attempt dropped, the Admitted seconds into acc up to the QuotaReserved unset (the end of an eviction under way, else
// d + latency), reason KB_DR_USER
__device__ __forceinline__ void drain_stop_row(const DrainDev &X, int a, int w, i64 d) {
  X.wl_deactivated[w] = KB_DR_USER;
  drain_clear_requeue(X, w);
  drain_drop_attempt(X, w, d);
  if (X.wl_max_exec) {
    const bool rel = X.adm.evicting && X.adm.evicting[a];
    drain_exec_release(X, a, w, rel ? X.adm.finish[a] : X.wl_evict ? drain_sat_add(d, X.wl_evict[w]) : d);
  }
  X.wl_gone[w] = d;
}
// a stop at sd (INT64_MAX = none) of row a's record comes before the row's own event while the record is active
__device__ __forceinline__ bool drain_stop_due(const DrainDev &X, int a, i64 sd) {
  return sd < X.adm.finish[a] && X.wl_deactivated[X.adm.wl[a]] == 0;
}
// whether a stop at sd or the own event of running row a is due at this boundary (stop: the stop), after the reclaim
// steps before it: strictly before its finish column, at or before a stop (an own event first)
__device__ __forceinline__ bool drain_row_due(const DevSnap &D, const DrainDev &X, int a, i64 sd, bool &stop) {
  stop = drain_stop_due(X, a, sd);
  if (X.wl_rc_start && drain_rc_live(X, a)) drain_reclaim(D, X, a, stop ? sd : min(X.clock[0], X.adm.finish[a] - 1));
  return stop || X.adm.finish[a] <= X.clock[0];
}
// completions (thread per row): a live row with finish <= t_{c+1} gets the dead stamp, its cells leave its ClusterQueue's
// usage (cache.DeleteWorkload, integer atomics), its record becomes FINISHED and its root tree is marked.  An evicting
// row's finish column holds its end time: it completes the eviction instead, its record returns to its queue.  Rows in
// [A + *n_new, bound) only pad the compaction's range.  Verdicts (admission checks), PodsReady timeouts and
// MaximumExecutionTimeSeconds expiries come first; a timed-out or expired row releases its record to BACKOFF or
// DEACTIVATED, and counts as neither a completion nor an eviction.
__global__ void k_drain_finish(DevSnap D, DrainDev X, int bound, const int32_t *n_new) {
  const int a = blockIdx.x * blockDim.x + threadIdx.x;
  if (a >= bound || a >= X.A + (n_new ? *n_new : 0) || X.counters[KB_DC_FULL]) return;
  const int stamp = X.cycle + 1;
  if (X.counters[KB_DC_END] || X.adm_dead[a] == stamp) return;
  const i64 sd = X.wl_stop ? X.wl_stop[X.adm.wl[a]] : INT64_MAX;  // a stop edit of the record at this boundary
  bool stop;
  if (!drain_row_due(D, X, a, sd, stop)) return;
  const int cq = X.adm.cq[a], w = X.adm.wl[a];
  int ph = X.adm.phase ? X.adm.phase[a] : KB_PH_RUN;
  if (!stop && ph == KB_PH_CHECK) {  // a verdict (ProvisioningRequest controller.go:536-580)
    const i64 tv = X.adm.finish[a];
    if (X.wl_fail[w] == 0) {  // Ready: Admitted, the run clock (or the PodsReady attempt) starts; it may end in this boundary
      drain_admitted(X, a, w, tv);
      atomicAdd(&X.counters[KB_DC_CHECK_READY], 1);
      if (!drain_row_due(D, X, a, sd, stop)) return;
      ph = X.adm.phase[a];
    } else {  // Retry or Rejected: the workload holds no pods, its quota goes at once
      if (X.wl_fail[w] != INT32_MAX) X.wl_fail[w]--;
      const int k = X.wl_retries[w] + 1;
      X.adm_dead[a] = stamp;
      drain_uncharge(D, X, a, false);
      drain_forget(D, X, w);
      if (k <= X.check_limit) {  // Retry: RequeueAt = verdict + WaitTime(k), queue-order timestamp = the eviction time
        X.wl_retries[w] = k;
        X.wl_requeue_at[w] = drain_sat_add(tv, kb_check_wait_ns(k, X.check_base_s, X.check_max_s));
        X.wl_qts[w] = tv;
        X.wl_state[w] = KB_WS_BACKOFF;
        atomicAdd(&X.counters[KB_DC_CHECK_RETRY], 1);
      } else {  // Rejected: deactivated
        X.wl_state[w] = KB_WS_DEACTIVATED;
        X.wl_deactivated[w] = KB_DR_REJECTED;
        atomicAdd(&X.counters[KB_DC_CHECK_REJECTED], 1);
      }
      X.root_mark[D.root_slot[cq]] = stamp;
      return;
    }
  }
  const i64 T = X.adm.finish[a];  // the time of a timeout or an expiry
  if (!stop && ph == KB_PH_WAIT) {  // PodsReady timeout at T (workload_controller.go:805-855, UpdateRequeueState workload.go:707-722)
    if (X.wl_pr_fail[w] > 0 && X.wl_pr_fail[w] != INT32_MAX) X.wl_pr_fail[w]--;
    const int n = X.wl_pr_count[w];
    if (X.pr_limit >= 0 && n >= X.pr_limit) {  // Count + 1 > limit: deactivated, RequeueState cleared
      X.wl_pr_count[w] = 0;
      X.wl_deactivated[w] = KB_DR_REQUEUING_LIMIT;
      atomicAdd(&X.counters[KB_DC_PR_DEACTIVATED], 1);
    } else {  // BACKOFF at release: RequeueAt = T + WaitTime(Count); under Eviction the queue timestamp is T
      const int k = n == INT32_MAX ? n : n + 1;
      X.wl_pr_count[w] = k;
      X.wl_requeue_at[w] = drain_sat_add(T, kb_pods_ready_wait_ns(k, X.pr_base_s, X.pr_max_s));
      if (!X.pr_creation) X.wl_qts[w] = T;
      atomicAdd(&X.counters[KB_DC_PR_TIMEOUT], 1);
    }
  } else if (!stop && ph == KB_PH_EXPIRE) {  // MaximumExecutionTimeExceeded at the effective deadline T (workload_controller.go:619-646)
    drain_exec_deactivate(X, w);
    drain_drop_attempt(X, w, T);  // a PodsReady attempt still waiting is dropped
  }
  if (!stop && (ph == KB_PH_WAIT || ph == KB_PH_EXPIRE)) {
    ph = KB_PH_TIMED_OUT;
    X.adm.phase[a] = ph;
    if (X.wl_evict) {  // the pods terminate: the row holds its cells until T + latency, as an evicting row (no steps)
      drain_evict_row(X, a, w, T);
      stop = drain_stop_due(X, a, sd);  // an expiry deactivated the record: no stop is due
      if (!stop && X.adm.finish[a] > X.clock[0]) return;
    }
  }
  if (stop) drain_stop_row(X, a, w, sd);
  else if (X.wl_gone) X.wl_gone[w] = X.adm.finish[a];
  X.adm_dead[a] = stamp;
  drain_uncharge(D, X, a, true);
  const bool timed_out = !stop && ph == KB_PH_TIMED_OUT;
  const bool released = !stop && X.adm.evicting && X.adm.evicting[a];
  const bool expired = X.wl_max_exec && (timed_out || released) && drain_exec_release(X, a, w, X.adm.finish[a]);
  if (stop || timed_out || expired) { drain_forget(D, X, w); X.wl_state[w] = X.wl_deactivated[w] ? KB_WS_DEACTIVATED : KB_WS_BACKOFF; }
  else if (released) drain_release(D, X, w);
  else if (w >= 0) { X.wl_state[w] = KB_WS_FINISHED; X.wl_admit_cycle[w] = -1; X.wl_finish_ns[w] = X.adm.finish[a]; }
  X.root_mark[D.root_slot[cq]] = stamp;
  if (!timed_out) atomicAdd(&X.counters[stop ? KB_DC_STOPPED : released ? KB_DC_EVICT_DONE : KB_DC_FINISHED], 1);
}
// decay samples (thread per LocalQueue of an AFS ClusterQueue): every sample due in (t, t'] with t' = clock[0], in time
// order, each with alpha = afs_alpha (one interval elapsed), or a reset to empty with half-life 0; LastUpdate moves to
// each due time.  Launched after k_drain_ev_next and before k_drain_finish, so the samples see the admitted usage the
// cycle left.  Nothing is due at or before t (the previous boundary took those samples, an admission at t sets
// LastUpdate = t), so a drain that ends (clock[0] = t) takes none.  The admitted usage is constant here: once a sample
// leaves consumed unchanged so do the later ones, and LastUpdate jumps to the last due time.  AFS drains cannot evict
// (the preemption guard), so k_drain_evict never changes the admitted usage.
__global__ void k_drain_afs_decay(DevSnap D, DrainDev X, int L) {
  const int l = blockIdx.x * blockDim.x + threadIdx.x;
  if (l >= L || X.lq_seg[l] < 0) return;
  const int R = D.R;
  const i64 last = X.lq_last[l];
  const u64 gap = (u64)X.clock[0] - (u64)last, samp = (u64)X.sampling_ns;  // t' >= LastUpdate
  if (gap < samp) return;
  const u64 due = gap / samp;
  i64 *cons = X.lq_consumed + (size_t)l * R;
  int32_t *csc = X.lq_consumed_scale + (size_t)l * R;
  bool bad = false, any = false;
  for (u64 k = 0; k < due; k++) {
    bool changed = false;
    if (X.half_life_ns == 0) {
      for (int r = 0; r < R; r++) { changed |= cons[r] != 0 || csc[r] != 0; cons[r] = 0; csc[r] = 0; }
    } else {
      bad |= !afs_decay(cons, csc, X.lq_adm + (size_t)l * R, X.milli_mul, X.alpha, R, &changed);
    }
    if (!changed || bad) break;
    any = true;
  }
  X.lq_last[l] = last + (i64)(due * samp);
  atomicAdd(X.afs_samples, (unsigned long long)due);
  if (any) {
    double u = 0.0;
    bad |= !afs_lq_usage(cons, csc, X.lq_penalty + (size_t)l * R, X.res_weight, X.lq_weight[l], R, &u);
    X.lq_usage[l] = u;
  }
  if (bad) atomicOr(D.status, KBS_AFS_OVERFLOW);
}
// arrivals (grid-stride over the arrived prefix [lo, hi)): each workload joins its queue (drain_enqueue)
__global__ void k_drain_arrive(DrainDev X) {
  const int lo = X.counters[KB_DC_ARR_LO], hi = X.counters[KB_DC_ARR_HI];
  if (blockIdx.x == 0 && threadIdx.x == 0) X.counters[KB_DC_ARRIVED] = hi - lo;
  for (int i = lo + blockIdx.x * blockDim.x + threadIdx.x; i < hi; i += gridDim.x * blockDim.x) drain_enqueue(X, X.arr_order[i]);
}

// ---- quota changes -----------------------------------------------------------------------------------------------------
// the edits of this boundary (one block, after k_drain_ev_next and before k_drain_finish: step 5 before the verdicts), in
// table order: the node's three rows, +1 on the generation of every ClusterQueue of its root tree (D.cq_generation and
// the copy in the tree's static block, TreeBlobHdr.gen), the root marked for k_drain_requeue; then the tree-local quota
// tables of the edited trees, rebuilt from the new rows as the static upload builds them, once per tree (by the tree's
// last edit of the boundary).  An edit that changes nothing (qc_root -1) is only counted.
__global__ void k_drain_quota(DevSnap D, DrainDev X) {
  const int lo = X.counters[KB_DC_QC_LO], hi = X.counters[KB_DC_QC_HI];
  if (lo == hi) return;
  const int FR = D.FR;
  i64 *nom = const_cast<i64 *>(D.nominal), *bl = const_cast<i64 *>(D.blimit), *ll = const_cast<i64 *>(D.llimit);
  i64 *gen = const_cast<i64 *>(D.cq_generation);
  unsigned char *blob = const_cast<unsigned char *>(D.tree_blob);
  for (int i = lo; i < hi; i++) {
    const int slot = X.qc_root[i];
    if (slot < 0) continue;
    const size_t src = (size_t)i * FR, dst = (size_t)X.qc_node[i] * FR;
    for (int c = threadIdx.x; c < FR; c += blockDim.x) { nom[dst + c] = X.qc_nominal[src + c]; bl[dst + c] = X.qc_blimit[src + c]; ll[dst + c] = X.qc_llimit[src + c]; }
    for (int k = X.qc_cq_start[slot] + threadIdx.x; k < X.qc_cq_start[slot + 1]; k += blockDim.x) {
      const int q = X.qc_cq[k];
      const i64 g = gen[q] + 1;
      gen[q] = g;
      if (X.qc_blob_gen[q] >= 0) *(i64 *)(blob + X.qc_blob_gen[q]) = g;
    }
    if (threadIdx.x == 0) X.root_mark[slot] = X.cycle + 1;
    __syncthreads();  // the next edit may write the same rows and generations
  }
  if (!D.tl_subtree) return;
  i64 *sub = const_cast<i64 *>(D.tl_subtree), *tbl = const_cast<i64 *>(D.tl_blimit), *lq = const_cast<i64 *>(D.tl_lquota);
  for (int i = lo; i < hi; i++) {
    const int t = X.qc_tree[i];
    if (t < 0 || X.qc_tree_next[i] < hi) continue;
    const int c0 = D.tree_start[t] * FR, c1 = D.tree_start[t + 1] * FR;
    for (int c = c0 + threadIdx.x; c < c1; c += blockDim.x) tl_static_cell(D, sub, tbl, lq, c);
    __syncthreads();
    for (int fr = threadIdx.x; fr < FR; fr += blockDim.x) tl_root_cell(D, sub, lq, t, fr);
    __syncthreads();
  }
}

// ---- deactivation and reactivation --------------------------------------------------------------------------------------
// edit j on record w (rules 2, 4 and 5 of kb_run_drain); held: the record holds a row at the edit's time (nothing changes).
// A stop deactivates an active record without a row; a resume returns a DEACTIVATED record to its queue as an arrival
// does (NoFit rule included), with LastAssignment nil, and raises the re-sort flag when its queue-order timestamp is not
// its sort key.  One thread per record: no atomics on the record's state.
__device__ __forceinline__ void drain_active_edit(const DevSnap &D, const DrainDev &X, int j, int w, bool held) {
  if (held) return;
  const uint8_t st = X.wl_state[w];
  if (X.ac_on[j] == 0) {
    if (X.wl_deactivated[w] != 0 || (st != KB_WS_QUEUED && st != KB_WS_SET_ASIDE && st != KB_WS_BACKOFF)) return;
    X.wl_state[w] = KB_WS_DEACTIVATED;
    X.wl_deactivated[w] = KB_DR_USER;
    drain_clear_requeue(X, w);
    const int cq = D.wl_cq[w];
    if (X.cq_sticky && X.cq_sticky[cq] == w) X.cq_sticky[cq] = -1;  // delete (cluster_queue.go:330-340)
    X.root_mark[D.root_slot[cq]] = X.cycle + 1;
    drain_forget(D, X, w);
    atomicAdd(&X.counters[KB_DC_STOPPED], 1);
  } else if (st == KB_WS_DEACTIVATED) {
    X.wl_deactivated[w] = 0;
    drain_forget(D, X, w);
    drain_enqueue(X, w);
    drain_mark_resort(X, w);
    atomicAdd(&X.counters[KB_DC_RESUMED], 1);
  }
}
// the edits of this boundary [lo, hi), one thread per record (grid-stride over the edits; the record's first edit of the
// boundary walks its edits in table order).  pass 0, after k_drain_ev_next and before k_drain_finish: the edits of records
// without a row; a record that is ABSENT or holds a row stops at its edit (wl_ac_from) to meet its own events first, and
// the first stop of an active row-holding record writes its time to wl_stop for k_drain_finish.  pass 1, after the
// arrivals and before k_drain_backoff (so a record that its own timeout or Retry put in BACKOFF and a stop then
// deactivated leaves no RequeueAt in the next E): the deferred edits; an edit before the time the record's row went (wl_gone) met a
// held record.  It clears wl_stop and wl_gone.
__global__ void k_drain_active(DevSnap D, DrainDev X, int pass) {
  const int lo = X.counters[KB_DC_AC_LO], hi = X.counters[KB_DC_AC_HI];
  for (int i = lo + blockIdx.x * blockDim.x + threadIdx.x; i < hi; i += gridDim.x * blockDim.x) {
    const int w = X.ac_wl[i];
    if (pass == 0) {
      if (X.ac_prev[i] >= lo) continue;
      for (int j = i; j < hi; j = X.ac_next[j]) {
        const uint8_t st = X.wl_state[w];
        const bool inactive = X.wl_deactivated[w] != 0;
        if (st == KB_WS_ABSENT || (st == KB_WS_HELD && (inactive || X.ac_on[j] == 0))) {
          if (st == KB_WS_HELD && !inactive) X.wl_stop[w] = X.ac_ns[j];
          X.wl_ac_from[w] = j;
          break;
        }
        drain_active_edit(D, X, j, w, st == KB_WS_HELD);
      }
    } else {
      if (X.wl_ac_from[w] != i) continue;
      for (int j = i; j < hi; j = X.ac_next[j]) drain_active_edit(D, X, j, w, X.wl_state[w] == KB_WS_HELD || X.wl_gone[w] > X.ac_ns[j]);
      X.wl_stop[w] = INT64_MAX; X.wl_gone[w] = INT64_MIN;
    }
  }
}
// start of a drain with the block: no edit deferred, no stop; records with wl_inactive start DEACTIVATED with its reason,
// in no queue, without RequeueAt (after k_drain_init_checks, before k_drain_backoff)
__global__ void k_drain_init_active(DrainDev X, int W, const uint8_t *inactive) {
  const int w = blockIdx.x * blockDim.x + threadIdx.x;
  if (w >= W) return;
  if (X.wl_ac_from) { X.wl_ac_from[w] = -1; X.wl_stop[w] = INT64_MAX; X.wl_gone[w] = INT64_MIN; }
  if (!inactive || !inactive[w]) return;
  X.wl_state[w] = KB_WS_DEACTIVATED;
  X.wl_deactivated[w] = inactive[w];
  if (X.wl_requeue_at) X.wl_requeue_at[w] = INT64_MIN;
}

// ---- admission checks ------------------------------------------------------------------------------------------------
// BACKOFF records (thread per record), after k_drain_finish and k_drain_ev_next: RequeueAt <= t_{c+1} joins its queue as
// an arrival does (PushOrUpdate, NoFit rule included) and raises the re-sort flag when its queue-order timestamp is not
// the key its position was sorted by; a later RequeueAt joins clock[2], the next boundary's E.  At the start (clock[0] =
// now_ns) it only reduces clock[2].
__global__ void k_drain_backoff(DrainDev X, int W) {
  const int w = blockIdx.x * blockDim.x + threadIdx.x;
  if (w >= W || X.wl_state[w] != KB_WS_BACKOFF) return;
  const i64 at = X.wl_requeue_at[w];
  if (at > X.clock[0]) { atomicMin((long long *)&X.clock[2], (long long)at); return; }
  drain_enqueue(X, w);
  drain_mark_resort(X, w);
}
// re-sort: every cursor back to 0 and no set-aside position, then the SET_ASIDE positions of the new order
__global__ void k_drain_resort_reset(DrainDev X, int S) {
  const int s = blockIdx.x * blockDim.x + threadIdx.x;
  if (s < S) { X.cursor[s] = 0; X.first_aside[s] = X.q_start[s + 1] - X.q_start[s]; }
}
__global__ void k_drain_resort_aside(DrainDev X, int W) {
  const int w = blockIdx.x * blockDim.x + threadIdx.x;
  if (w < W && X.wl_state[w] == KB_WS_SET_ASIDE) atomicMin(&X.first_aside[X.wl_seg[w]], X.wl_pos[w]);
}
// start of a drain with admission checks: records in check backoff (RequeueAt after now_ns) are BACKOFF; nothing is Admitted
__global__ void k_drain_init_checks(DrainDev X, int W, i64 now_ns) {
  const int w = blockIdx.x * blockDim.x + threadIdx.x;
  if (w >= W) return;
  if (X.wl_requeue_at[w] > now_ns) X.wl_state[w] = KB_WS_BACKOFF;
  X.wl_ready_ns[w] = INT64_MIN; X.wl_deactivated[w] = 0;
}
