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
// takes finished rows out of the LocalQueue's admitted usage (adm_lq, carried by the compaction).
//
// Event mode (kb_snapshot.wl_create_ns / wl_run_ns / adm_finish_ns; include/kueue_b200.h): two more states,
// KB_WS_ABSENT (not created yet) and KB_WS_FINISHED.  Every admitted row carries its finish time (adm_finish, written by
// k_drain_admit, carried by the compaction) and its record (adm_wl, -1 for a row of the snapshot without one).  The
// boundary is the replay's, with the clock between the evictions and the requeue: k_drain_ev_min reduces E (the
// earliest finish of a live row and the next creation), k_drain_ev_next (one thread) computes t_{c+1} and the end
// flag, k_drain_finish stamps the finished rows dead with the eviction stamp and takes their cells out (a row admitted
// in this cycle that finishes by t_{c+1} dies before any cycle sees it), k_drain_arrive walks the arrived prefix of the
// (create, index) order; then k_drain_requeue visits the marked roots and the compaction follows.  A cycle without heads
// is replaced by the same boundary with t_{c+1} = E and a negative stamp (no cycle is counted).  The NoFit set of a
// ClusterQueue is one byte per (ClusterQueue, scheduling hash) class: k_drain_apply sets it, k_drain_requeue clears the
// bytes of the queues it visits.
#pragma once

#include <cub/device/device_scan.cuh>

#include "kb_device.cuh"

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
  int32_t *adm_cq, *adm_priority; i64 *adm_ts, *adm_qr_ts, *adm_uid; uint8_t *adm_evicted; int32_t *adm_use_start, *adm_use_fr; i64 *adm_use_qty;
  int A, AU, cycle;  // admitted workloads / usage cells before this cycle's admissions
  int A_cap, AU_cap; // capacity of the admitted tables (rows / usage cells)
  // eviction replay; adm_wl == nullptr: off
  int32_t *adm_wl;                 // [A_cap] pending record of each admitted row (current half)
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
  int32_t *adm_lq;            // [A_cap] LocalQueue of each admitted row (current half), -1 = none
  unsigned long long *afs_samples;  // [1] samples taken
  i64 half_life_ns, sampling_ns;
  // event mode; adm_finish == nullptr: off
  i64 *adm_finish;                 // [A_cap] finish time of each admitted row (current half), INT64_MAX = never
  const i64 *wl_run;               // [W] run time once admitted (< 0 never finishes); null = none finishes
  i64 *wl_admit_ns, *wl_finish_ns; // [W]
  i64 *clock;                      // [0] t_{c+1} of the boundary, [1] E (INT64_MAX = none; reset by k_drain_ev_next)
  const u64 *arr_key;              // [n_arr] creation times (sign flipped) of the ABSENT workloads, ascending
  const int32_t *arr_order;        // [n_arr] their indices, ties by index
  int n_arr;
  const int32_t *wl_class;         // [W] (ClusterQueue, hash) class of a BestEffortFIFO workload with a known hash, -1
  const int32_t *cq_class_start;   // [Q+1] classes of a ClusterQueue
  uint8_t *class_nofit;            // [classes] in the ClusterQueue's NoFit set; null = no arrivals or no hashes
};
// counters of a boundary: [1] evictions, [2] / [3] rows / cells after the compaction, [5] capacity flag; event mode:
// [6] completions, [7] arrivals, [8] end flag, [9] / [10] arrived prefix of arr_order [lo, hi)
enum { KB_DC_EVICTED = 1, KB_DC_ROWS = 2, KB_DC_CELLS = 3, KB_DC_FULL = 5,
       KB_DC_FINISHED = 6, KB_DC_ARRIVED = 7, KB_DC_END = 8, KB_DC_ARR_LO = 9, KB_DC_ARR_HI = 10 };

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
// third pass: (segment | priority desc); the segment is the ClusterQueue unless its queue is split by LocalQueue
__global__ void k_drain_keys_cq(DevSnap D, DrainDev X, const int32_t *vals, u64 *keys, int32_t *q_count) {
  int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= D.W) return;
  int w = vals[i];
  int cq = D.wl_cq[w];
  int seg = (X.seg_start && X.cq_afs[cq]) ? X.lq_seg[X.wl_lq[w]] : drain_seg0(X, cq);
  keys[i] = ((u64)seg << 32) | (u64)(~((unsigned)D.wl_priority[w] ^ 0x80000000u));  // higher priority first
  atomicAdd(&q_count[seg], 1);
}
enum { KB_WS_QUEUED = 0, KB_WS_SET_ASIDE = 1, KB_WS_HELD = 2, KB_WS_ABSENT = 3, KB_WS_FINISHED = 4 };
__global__ void k_drain_init(DevSnap D, DrainDev X, int S) {
  int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < D.W) { X.wl_state[i] = KB_WS_QUEUED; X.wl_admit_cycle[i] = -1; X.wl_evals[i] = 0; X.wl_last_decision[i] = 0xff; }
  if (i < D.W && X.wl_evictions) X.wl_evictions[i] = 0;
  if (i < S) { X.cursor[i] = 0; X.first_aside[i] = X.q_start[i + 1] - X.q_start[i]; }
}
// replay: the records named by adm_wl hold quota (out of every queue); segment and position of every workload
__global__ void k_drain_init_replay(DevSnap D, DrainDev X, int n_adm) {
  int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n_adm) X.wl_state[X.adm_wl[i]] = KB_WS_HELD;
  if (i < D.W) {
    const int w = X.q_order[i];
    const int cq = D.wl_cq[w];
    const int seg = (X.seg_start && X.cq_afs[cq]) ? X.lq_seg[X.wl_lq[w]] : drain_seg0(X, cq);
    X.wl_seg[w] = seg; X.wl_pos[w] = i - X.q_start[seg];
  }
}
// the cursor of every segment at its first QUEUED workload (the start of a drain)
__global__ void k_drain_advance(DrainDev X, int S) {
  int s = blockIdx.x * blockDim.x + threadIdx.x;
  if (s >= S) return;
  const int qs = X.q_start[s], qn = X.q_start[s + 1] - qs;
  int cur = X.cursor[s];
  while (cur < qn && X.wl_state[X.q_order[qs + cur]] != KB_WS_QUEUED) cur++;
  X.cursor[s] = cur;
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
  if (X.flag[q]) { int s = X.head_seg ? X.head_seg[q] : q; heads[X.pos[q]] = X.q_order[X.q_start[s] + X.cursor[s]]; }
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
  const bool inadmissible = (dec == KB_DEC_NOFIT || dec == KB_DEC_PREEMPT_NO_TARGETS) && !pending_flavors;
  const int hs = X.head_seg ? X.head_seg[cq] : cq, s0 = drain_seg0(X, cq), s1 = drain_seg1(X, cq);
  const bool bulk = dec == KB_DEC_NOFIT && !strict && D.wl_sched_hash && D.wl_sched_hash[wl] != 0;
  if (bulk) {  // handleInadmissibleHash :408-425: every queued workload of the class, in every segment of the queue
    const i64 hsh = D.wl_sched_hash[wl];
    if (X.class_nofit) X.class_nofit[X.wl_class[wl]] = 1;  // noFitSchedulingHashes.Insert (:414)
    for (int s = s0; s < s1; s++) {
      const int qs = X.q_start[s], qn = X.q_start[s + 1] - qs;
      for (int p = X.cursor[s] + (s == hs); p < qn; p++) {
        const int w2 = X.q_order[qs + p];
        if (D.wl_sched_hash[w2] == hsh && X.wl_state[w2] == KB_WS_QUEUED) { X.wl_state[w2] = KB_WS_SET_ASIDE; X.first_aside[s] = min(X.first_aside[s], p); }
      }
    }
  }
  if (inadmissible && !strict) { X.wl_state[wl] = KB_WS_SET_ASIDE; X.first_aside[hs] = min(X.first_aside[hs], X.cursor[hs]); }
  if (ok || (inadmissible && !strict)) X.cursor[hs]++;
  for (int s = s0; s < s1; s++) {
    if (s != hs && !bulk) continue;
    const int qs = X.q_start[s], qn = X.q_start[s + 1] - qs;
    int cur = X.cursor[s];
    while (cur < qn && X.wl_state[X.q_order[qs + cur]] != KB_WS_QUEUED) cur++;
    X.cursor[s] = cur;
  }
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
  if (X.adm_wl) X.adm_wl[a] = wl;
  if (X.adm_lq) X.adm_lq[a] = X.wl_lq[wl];
  X.adm_cq[a] = cq; X.adm_priority[a] = D.wl_priority[wl]; X.adm_ts[a] = D.wl_ts[wl]; X.adm_qr_ts[a] = qr_ts;
  X.adm_uid[a] = D.wl_uid[wl]; X.adm_evicted[a] = 0;
  X.adm_use_start[a] = c0;
  if (X.adm_finish) {  // finish = QuotaReserved time + run time, saturating; run < 0 never finishes
    const i64 run = X.wl_run ? X.wl_run[wl] : -1;
    X.adm_finish[a] = run < 0 ? INT64_MAX : (qr_ts > INT64_MAX - run ? INT64_MAX : qr_ts + run);
    X.wl_admit_ns[wl] = qr_ts;
  }
  const bool covers_pods = drain_covers_pods(D, cq);
  const int ps0 = D.wl_ps_start[wl], ps1 = D.wl_ps_start[wl + 1];
  int n = 0;
  for (int row = ps0; row < ps1; row++)
    for (int r = 0; r < R; r++) {
      int f = D.ps_flavor[(size_t)row * R + r];
      if (f < 0) continue;
      int fr = f * R + r;
      i64 q = drain_request(D, row, r, D.ps_count_out[row], covers_pods);
      int j = 0;
      while (j < n && X.adm_use_fr[c0 + j] != fr) j++;
      if (j == n) { X.adm_use_fr[c0 + n] = fr; X.adm_use_qty[c0 + n] = 0; n++; }
      X.adm_use_qty[c0 + j] += q;
    }
  X.adm_use_start[a + 1] = c0 + n;
  for (int j = 0; j < n; j++) X.cq_usage[(size_t)cq * D.FR + X.adm_use_fr[c0 + j]] += X.adm_use_qty[c0 + j];  // one entry per ClusterQueue
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
      for (int j = 0; j < n; j++) adm[X.adm_use_fr[c0 + j] % R] += X.adm_use_qty[c0 + j];
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
// every target of every Preempting entry (thread per entry): cells out of its ClusterQueue's usage (integer atomics:
// the order does not matter), row dead, pending record QUEUED with LastAssignment nil, its root tree marked
__global__ void k_drain_evict(DevSnap D, DrainDev X) {
  int e = blockIdx.x * blockDim.x + threadIdx.x;
  if (e >= D.H || D.decision[e] != KB_DEC_PREEMPTING) return;
  const int R = D.R, stamp = X.cycle + 1;
  const int off = D.tgt_off[e], n = D.tgt_cnt[e];
  for (int k = 0; k < n; k++) {
    const int a = D.tgt_pool_adm[off + k];
    if (atomicExch(&X.adm_dead[a], stamp) == stamp) continue;  // one eviction per row
    const int cq = X.adm_cq[a];
    for (int c = X.adm_use_start[a]; c < X.adm_use_start[a + 1]; c++)  // cache.DeleteWorkload
      atomicAdd((unsigned long long *)&X.cq_usage[(size_t)cq * D.FR + X.adm_use_fr[c]], (unsigned long long)(-X.adm_use_qty[c]));
    const int w = X.adm_wl[a];
    X.wl_state[w] = KB_WS_QUEUED;
    X.wl_last_gen[w] = -1;
    for (int i = D.wl_ps_start[w] * R; i < D.wl_ps_start[w + 1] * R; i++) X.ps_last_tried[i] = -1;
    if (X.wl_has_qr) X.wl_has_qr[w] = 0;
    X.wl_admit_cycle[w] = -1;
    X.wl_evictions[w]++;  // a workload holds at most one row: one writer
    atomicMin(&X.cursor[X.wl_seg[w]], X.wl_pos[w]);
    X.root_mark[D.root_slot[cq]] = stamp;
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
  X.row_cells[a] = live ? X.adm_use_start[a + 1] - X.adm_use_start[a] : 0;
}
struct AdmTabs { int32_t *cq, *priority; i64 *ts, *qr_ts, *uid; uint8_t *evicted; int32_t *use_start, *use_fr; i64 *use_qty; int32_t *wl; i64 *finish; int32_t *lq; };
// live rows of [0, bound), in order, into the other half of the double buffer; thread bound writes the totals
__global__ void k_drain_compact(DrainDev X, AdmTabs O, int bound) {
  int a = blockIdx.x * blockDim.x + threadIdx.x;
  if (a > bound) return;
  if (a == bound) { O.use_start[X.row_new[a]] = X.cell_new[a]; X.counters[KB_DC_ROWS] = X.row_new[a]; X.counters[KB_DC_CELLS] = X.cell_new[a]; return; }
  if (!X.row_live[a]) return;
  const int n = X.row_new[a], c0 = X.cell_new[a], u0 = X.adm_use_start[a], nc = X.adm_use_start[a + 1] - u0;
  O.cq[n] = X.adm_cq[a]; O.priority[n] = X.adm_priority[a]; O.ts[n] = X.adm_ts[a]; O.qr_ts[n] = X.adm_qr_ts[a];
  O.uid[n] = X.adm_uid[a]; O.evicted[n] = X.adm_evicted[a]; O.wl[n] = X.adm_wl[a]; O.use_start[n] = c0;
  if (X.adm_finish) O.finish[n] = X.adm_finish[a];
  if (X.adm_lq) O.lq[n] = X.adm_lq[a];
  for (int c = 0; c < nc; c++) { O.use_fr[c0 + c] = X.adm_use_fr[u0 + c]; O.use_qty[c0 + c] = X.adm_use_qty[u0 + c]; }
}

// ---- event mode ---------------------------------------------------------------------------------------------------
__device__ __forceinline__ i64 ev_time(u64 key) { return (i64)(key ^ 0x8000000000000000ull); }
// first i in [lo, n) with arr_key[i] > t (the creations up to t are [.., i))
__device__ __forceinline__ int ev_upper_bound(const u64 *key, int lo, int n, i64 t) {
  const u64 k = (u64)t ^ 0x8000000000000000ull;
  int hi = n;
  while (lo < hi) { const int m = lo + (hi - lo) / 2; if (key[m] <= k) lo = m + 1; else hi = m; }
  return lo;
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
    X.clock[0] = now_ns; X.clock[1] = INT64_MAX;
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
  if (a < bound && a < n_rows && X.adm_dead[a] != X.cycle + 1) v = X.adm_finish[a];
  if (a == 0 && X.counters[KB_DC_ARR_HI] < X.n_arr) v = min(v, ev_time(X.arr_key[X.counters[KB_DC_ARR_HI]]));
  for (int o = 16; o > 0; o >>= 1) v = min(v, (i64)__shfl_xor_sync(0xffffffffu, (long long)v, o));
  if ((threadIdx.x & 31) == 0 && v < INT64_MAX) atomicMin((long long *)&X.clock[1], (long long)v);
}
// t_{c+1} and the end flag (one thread).  jump: no heads, the clock goes to E.  Otherwise a cycle that admitted or
// evicted steps, a quiet one waits for E; no E ends the drain.  Then the arrived prefix up to t_{c+1}.
__global__ void k_drain_ev_next(DrainDev X, i64 t_c, i64 step, int jump, const int32_t *n_new) {
  const i64 E = X.clock[1];
  const i64 stepped = t_c > INT64_MAX - step ? INT64_MAX : t_c + step;
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
}
// completions (thread per row): a live row with finish <= t_{c+1} gets the dead stamp, its cells leave its ClusterQueue's
// usage (cache.DeleteWorkload, integer atomics), its record becomes FINISHED and its root tree is marked.  Rows in
// [A + *n_new, bound) only pad the compaction's range.
__global__ void k_drain_finish(DevSnap D, DrainDev X, int bound, const int32_t *n_new) {
  const int a = blockIdx.x * blockDim.x + threadIdx.x;
  if (a >= bound || a >= X.A + (n_new ? *n_new : 0) || X.counters[KB_DC_FULL]) return;
  const int stamp = X.cycle + 1;
  if (X.counters[KB_DC_END] || X.adm_dead[a] == stamp || X.adm_finish[a] > X.clock[0]) return;
  X.adm_dead[a] = stamp;
  const int cq = X.adm_cq[a];
  for (int c = X.adm_use_start[a]; c < X.adm_use_start[a + 1]; c++)
    atomicAdd((unsigned long long *)&X.cq_usage[(size_t)cq * D.FR + X.adm_use_fr[c]], (unsigned long long)(-X.adm_use_qty[c]));
  const int w = X.adm_wl[a];
  if (w >= 0) { X.wl_state[w] = KB_WS_FINISHED; X.wl_admit_cycle[w] = -1; X.wl_finish_ns[w] = X.adm_finish[a]; }
  if (X.lq_last && X.adm_lq[a] >= 0 && X.cq_afs[cq]) {  // several rows of one LocalQueue can finish together
    i64 *adm = X.lq_adm + (size_t)X.adm_lq[a] * D.R;
    for (int c = X.adm_use_start[a]; c < X.adm_use_start[a + 1]; c++)
      atomicAdd((unsigned long long *)&adm[X.adm_use_fr[c] % D.R], (unsigned long long)(-X.adm_use_qty[c]));
  }
  X.root_mark[D.root_slot[cq]] = stamp;
  atomicAdd(&X.counters[KB_DC_FINISHED], 1);
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
// arrivals (grid-stride over the arrived prefix [lo, hi)): the workload joins its queue and the cursor moves back to it;
// in a BestEffortFIFO ClusterQueue a known hash in the NoFit set sets it aside (PushOrUpdate, cluster_queue.go:288-293)
__global__ void k_drain_arrive(DrainDev X) {
  const int lo = X.counters[KB_DC_ARR_LO], hi = X.counters[KB_DC_ARR_HI];
  if (blockIdx.x == 0 && threadIdx.x == 0) X.counters[KB_DC_ARRIVED] = hi - lo;
  for (int i = lo + blockIdx.x * blockDim.x + threadIdx.x; i < hi; i += gridDim.x * blockDim.x) {
    const int w = X.arr_order[i], s = X.wl_seg[w], p = X.wl_pos[w];
    if (X.class_nofit && X.wl_class[w] >= 0 && X.class_nofit[X.wl_class[w]]) {
      X.wl_state[w] = KB_WS_SET_ASIDE;
      atomicMin(&X.first_aside[s], p);
    } else {
      X.wl_state[w] = KB_WS_QUEUED;
      atomicMin(&X.cursor[s], p);
    }
  }
}
