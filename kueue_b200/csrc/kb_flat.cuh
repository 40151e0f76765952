// kb_flat.cuh — the scheduling cycle of one flat root cohort, start to finish in shared memory (k_cycle_flat).
//
// Same cycle as k_cycle_root's flat branch (kb_kernels.cuh: tree pass -> nominate -> iterator order -> threshold
// admit loop; scheduler.go:218-427 on a cohort whose ClusterQueues all hang directly off the root), rebuilt around
// one idea: the CTA first RELOCATES its root's slice of the snapshot into shared memory — quota tables, the static
// per-ClusterQueue policy / resource-group tables (one contiguous host-built block per tree, DevSnap::tree_blob) and
// the per-cycle head / podset records of its entries — renumbering every id (entry, workload, podset row,
// ClusterQueue, resource group) to be local to the root.  The flavor assigner, the iterator key and the request
// expansion are the SAME device functions every other kernel uses (assign_workload_coop, compute_entry_key,
// expand_entry): they run on a DevSnap whose table pointers all point into that relocated copy (tab_local == 2), so
// their chains of dependent loads (head -> workload -> podset rows -> resource group -> flavors -> quota cells) cost
// shared-memory latency instead of an L2 / HBM round trip per hop.  Global memory is touched in two bursts, each
// overlapped with compute: the staging at the start (every load independent, at most three dependent hops:
// tree_start -> node / head record -> rows; the tables read late land while phase 1 runs, the entries' records while
// the tree pass runs) and the publication of usage + decisions, which runs on the other warps behind the ordered loop.
//
// Used when k_cycle_root's conditions hold and, in addition, every tree is flat, FR <= 64 and the relocated copy fits
// shared memory (host: flat_layout).  Reference semantics are cited at the shared device functions.
#pragma once

struct FlatLay {  // byte offsets into the dynamic shared memory of k_cycle_flat (computed on the host, passed by value)
  uint32_t u, sub, lq, bl, av, pot, over, lend, blob, n_e, n_wl, n_ps0, n_psn, e_gid, e_cq, e_prio, e_ident, e_psn, e_at, blk_bar, e_ts, e_lg, e_qr,
      e_fast, e_mode, e_borrow, e_rank, m_sorted, d_sorted, r_gid, r_count, r_min, r_mask, r_group, r_ok, r_req, r_last, o_fl, o_md, o_tr, o_cnt, key, misc, snap, rec, total;
};
__host__ __device__ inline FlatLay flat_layout(int ncap, int FR, int R, int rcap, int bcap) {
  FlatLay L;
  size_t o = 0;
  auto take = [&](size_t bytes) { size_t at = o; o += (bytes + 15) & ~(size_t)15; return (uint32_t)(at < 0xffffffffu ? at : 0xffffffffu); };
  const size_t T = (size_t)ncap * FR;
  L.u = take(T * 8); L.sub = take(T * 8); L.lq = take(T * 8); L.bl = take(T * 8); L.av = take(T * 8); L.pot = take(T * 8);
  L.over = take((size_t)ncap * R * 8); L.lend = take((size_t)ncap * R * 8);
  L.blob = take((size_t)bcap);
  L.n_e = take((size_t)ncap * 4); L.n_wl = take((size_t)ncap * 4); L.n_ps0 = take((size_t)ncap * 4); L.n_psn = take((size_t)ncap * 4);
  L.e_gid = take((size_t)ncap * 4); L.e_cq = take((size_t)ncap * 4); L.e_prio = take((size_t)ncap * 4); L.e_ident = take((size_t)ncap * 4);
  L.e_psn = take((size_t)(ncap + 1) * 4); L.e_at = take((size_t)ncap * 4); L.blk_bar = take(((size_t)ncap / 32 + 2) * 8);
  L.e_ts = take((size_t)ncap * 8); L.e_lg = take((size_t)ncap * 8); L.e_qr = take((size_t)ncap);
  L.e_fast = take((size_t)ncap);
  L.e_mode = take((size_t)ncap * 4); L.e_borrow = take((size_t)ncap * 4); L.e_rank = take((size_t)ncap * 4);
  L.m_sorted = take((size_t)ncap * 4); L.d_sorted = take(((size_t)ncap / 32 + 2) * 4);
  L.r_gid = take((size_t)rcap * 4); L.r_count = take((size_t)rcap * 4); L.r_min = take((size_t)rcap * 4); L.r_mask = take((size_t)rcap * 4);
  L.r_group = take((size_t)rcap * 4); L.r_ok = take((size_t)rcap * 8); L.r_req = take((size_t)rcap * R * 8); L.r_last = take((size_t)rcap * R);
  L.o_fl = take((size_t)rcap * R); L.o_md = take((size_t)rcap * R); L.o_tr = take((size_t)rcap * R); L.o_cnt = take((size_t)rcap * 4);
  L.key = take((size_t)ncap * 32);
  L.misc = take(64 + 256);
  L.snap = take(sizeof(DevSnap));
  L.rec = take((size_t)ncap * 16);
  L.total = (uint32_t)(o < 0xffffffffu ? o : 0xffffffffu);
  return L;
}

// Header of one tree's static block (DevSnap::tree_blob): counts + byte offsets (from the block start, 16 B aligned)
// of its arrays, all in the tree's local numbering (node handle = position in tree_nodes, resource groups and flavor
// lists renumbered in node order).
struct TreeBlobHdr {
  int32_t nn, nrg, nfl, bytes;
  int32_t gid, par, hgt, rgs;           // int32 [nn] global node id, local parent (-1 root), height, [nn+1] first local resource group
  int32_t gen, wgt;                     // i64 [nn] cq_generation, f64 [nn] fair_weight
  int32_t within, reclaim, borrow_w, wcb, wcp, pref;  // u8 [nn] each
  int32_t rgmask, rgfl, fl;             // u32 [nrg], int32 [nrg+1] first flavor slot, int32 [nfl] flavors
  int32_t pad;
};
static_assert(sizeof(TreeBlobHdr) == 80, "TreeBlobHdr layout");

// Head records: per tree node (tree-local order) {entry, workload, first podset row, podset count | KB_REC_GENERAL |
// stamp << 16} of the ClusterQueue's head.  A record is valid only when its stamp is the current one
// (DevSnap::rec_stamp), so the table is never cleared between cycles (the host clears it when it is (re)allocated or
// the 16-bit stamp wraps).  KB_REC_GENERAL marks a head that k_cycle_flat nominates with the general walk: several
// podsets (or none), or one that partial admission could reduce.
#define KB_REC_GENERAL 0x8000
__device__ __forceinline__ void cq_rec_write(const DevSnap &D, int4 *rec, int e) {
  const int wl = D.heads[e];
  const int cq = D.wl_cq[wl];
  const int slot = D.root_slot[cq] - D.nLone;
  if (slot < 0) return;
  const int ps0 = D.wl_ps_start[wl], np = D.wl_ps_start[wl + 1] - ps0;
  const bool general = np != 1 || ((D.flags & KB_F_PARTIAL_ADMISSION) && D.ps_min_count[ps0] >= 0 && D.ps_count[ps0] > D.ps_min_count[ps0]);
  rec[D.tree_start[slot] + D.local_idx[cq]] = make_int4(e, wl, ps0, np | (general ? KB_REC_GENERAL : 0) | (int)(D.rec_stamp << 16));
}
// usage rows into tree-local order (cohort rows zero): cell i of [tree nodes][FR]
__device__ __forceinline__ void tl_usage_write(const DevSnap &D, int i) {
  const int nd = D.tree_nodes[i / D.FR];
  D.tl_usage[i] = nd < D.Q ? D.cq_usage[(size_t)nd * D.FR + i % D.FR] : 0;
}
__global__ void k_cq_rec(DevSnap D, int4 *rec, int tl_cells) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < D.H) cq_rec_write(D, rec, i);
  if (i < tl_cells) tl_usage_write(D, i);
}
// static quota tables into tree-local row order (once per static upload), holding the quotas k_cycle_flat derives from
// them: SubtreeQuota (a ClusterQueue's is its nominal quota, resource_node.go:160-166) and localQuota (:66-71) per cell.
// A flat root's SubtreeQuota and localQuota depend on its ClusterQueues' rows and are written by k_tl_root.  Cohort
// rows of hierarchical trees are left at nominal / local_quota(nominal) and never read: k_cycle_flat needs every tree flat.
__global__ void k_tl_static(DevSnap D, i64 *subtree, i64 *blimit, i64 *lquota, int tl_cells) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= tl_cells) return;
  const size_t g = (size_t)D.tree_nodes[i / D.FR] * D.FR + i % D.FR;
  subtree[i] = D.nominal[g]; blimit[i] = D.blimit[g]; lquota[i] = local_quota(D.nominal[g], D.llimit[g]);
}
// the root row of a flat tree: SubtreeQuota = nominal + sum of (SubtreeQuota - localQuota) over the ClusterQueues
// (accumulateFromChild resource_node.go:210-217), then its localQuota.  One thread per (tree, column), after k_tl_static.
__global__ void k_tl_root(DevSnap D, i64 *subtree, i64 *lquota) {
  const int k = blockIdx.x * blockDim.x + threadIdx.x;
  if (k >= D.nTrees * D.FR) return;
  const int t = k / D.FR, fr = k % D.FR;
  if (!D.tree_flat[t]) return;
  const size_t r0 = (size_t)D.tree_start[t] * D.FR + fr;
  const int nn = D.tree_start[t + 1] - D.tree_start[t];
  i64 sub = subtree[r0];
  for (int h = 1; h < nn; h++) sub += subtree[r0 + (size_t)h * D.FR] - lquota[r0 + (size_t)h * D.FR];
  subtree[r0] = sub;
  lquota[r0] = local_quota(sub, D.llimit[(size_t)D.tree_nodes[D.tree_start[t]] * D.FR + fr]);
}
// Everything the cycle needs prepared on the device, in one launch: head records, result rows of workloads that are
// not heads (-1 / 0), cleared cycle header.
__global__ void k_flat_prep(DevSnap D, int4 *rec, int fill_words, int P, int tl_cells) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < D.H) cq_rec_write(D, rec, i);
  if (i < tl_cells) tl_usage_write(D, i);
  if (i < fill_words) ((uint32_t *)D.ps_flavor)[i] = 0xffffffffu;  // flavor, res_mode, tried are adjacent (out_layout)
  if (i < P) D.ps_count_out[i] = 0;
  if (i < 32) D.status[i] = 0;
}

__device__ __forceinline__ void cp_async16(void *smem_dst, const void *gsrc) {
  unsigned d = (unsigned)__cvta_generic_to_shared(smem_dst);
  asm volatile("cp.async.cg.shared.global [%0], [%1], 16;" ::"r"(d), "l"(gsrc) : "memory");
}
// 4- and 8-byte copies (naturally aligned on both sides)
template <int B>
__device__ __forceinline__ void cp_async_small(void *smem_dst, const void *gsrc) {
  static_assert(B == 4 || B == 8, "cp.async.ca copies 4, 8 or 16 bytes");
  unsigned d = (unsigned)__cvta_generic_to_shared(smem_dst);
  asm volatile("cp.async.ca.shared.global [%0], [%1], %2;" ::"r"(d), "l"(gsrc), "n"(B) : "memory");
}
__device__ __forceinline__ void cp_async_commit() { asm volatile("cp.async.commit_group;" ::: "memory"); }
__device__ __forceinline__ void cp_async_wait_prior1() { asm volatile("cp.async.wait_group 1;" ::: "memory"); }
// 1-D bulk copies (the TMA engine, no tensor map) completing on an mbarrier
__device__ __forceinline__ void mbar_init(unsigned long long *bar, unsigned count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;\n\tfence.mbarrier_init.release.cluster;" ::"r"((unsigned)__cvta_generic_to_shared(bar)), "r"(count) : "memory");
}
__device__ __forceinline__ void mbar_expect_tx(unsigned long long *bar, unsigned bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"((unsigned)__cvta_generic_to_shared(bar)), "r"(bytes) : "memory");
}
__device__ __forceinline__ void bulk_g2s(void *smem_dst, const void *gsrc, unsigned bytes, unsigned long long *bar) {
  asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];"
               ::"r"((unsigned)__cvta_generic_to_shared(smem_dst)), "l"(gsrc), "r"(bytes), "r"((unsigned)__cvta_generic_to_shared(bar)) : "memory");
}
__device__ __forceinline__ bool mbar_try_wait(unsigned long long *bar, unsigned parity) {
  unsigned ok;
  asm volatile("{\n\t.reg .pred p;\n\tmbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\tselp.b32 %0, 1, 0, p;\n\t}"
               : "=r"(ok) : "r"((unsigned)__cvta_generic_to_shared(bar)), "r"(parity) : "memory");
  return ok != 0;
}
// waits (suspended in try_wait, acquire at CTA scope) until the barrier's phase of the given parity has completed
__device__ __forceinline__ void mbar_wait(unsigned long long *bar, unsigned parity) {
  unsigned spins = 0;
  while (!mbar_try_wait(bar, parity)) if (++spins > (1u << 24)) __trap();  // a lost copy or signal must not hang the device
}
__device__ __forceinline__ void mbar_arrive(unsigned long long *bar) {  // release at CTA scope
  asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"((unsigned)__cvta_generic_to_shared(bar)) : "memory");
}
__device__ __forceinline__ void cp_async_wait_all() { asm volatile("cp.async.commit_group;\ncp.async.wait_group 0;" ::: "memory"); }

// ordered admit loop over the entries in iterator order (scheduler.go:269-401) on one threshold per (position, column):
//   Fit      : fits <=> usage_root[c] <= lim[pos][c] for every column   (INT64_MAX: no condition, INT64_MIN: never)
//              admitted: usage_root[c] += max(0, SubtreeQuota_root[c] - lim)
//   Preempt  : (no targets possible) reserves unconditionally (:303-318); lim holds SubtreeQuota_root - reserved amount,
//              so the amount added has the same form as for Fit
// One warp; lane = column (and column + 32 when kTwo).  Per entry the dependent chain is compare -> vote -> add; the
// thresholds of the next four positions are in flight while the current four are decided.  Results: one bit per
// position (the vote) in ok_bits; the decision follows from the bit and the entry's mode.  Block b of 32 positions is
// signalled on blk_bar[b] as soon as its word is written, so the decisions can be published behind the loop.
template <bool kTwo>
__device__ inline void flat_ordered_loop(int n, int FR, int lane, const i64 *s_lim, const int *m_sorted, uint32_t *ok_bits,
                                         unsigned long long *blk_bar, i64 *s_u, const i64 *s_sub) {
  const int fr0 = lane, fr1 = lane + 32;
  const bool c0 = fr0 < FR, c1 = kTwo && fr1 < FR;
  i64 urt0 = c0 ? s_u[fr0] : 0, urt1 = c1 ? s_u[fr1] : 0;
  const i64 srt0 = c0 ? s_sub[fr0] : 0, srt1 = c1 ? s_sub[fr1] : 0;
  const i64 *col0 = s_lim + (c0 ? fr0 : 0), *col1 = s_lim + (c1 ? fr1 : 0);
  auto fetch = [&](i64 (&v0)[4], i64 (&v1)[4], int p0) {  // clamped: positions >= n are masked out by their mode bits
#pragma unroll
    for (int k = 0; k < 4; k++) {
      const size_t row = (size_t)min(p0 + k, n - 1) * FR;
      v0[k] = col0[row];
      if (kTwo) v1[k] = col1[row];
    }
  };
  i64 a0[4], a1[4], b0[4], b1[4];
  fetch(a0, a1, 0);
  for (int blk = 0; blk < n; blk += 32) {
    const int m = blk + lane < n ? m_sorted[blk + lane] : KB_MODE_NOFIT;
    const unsigned fitm = __ballot_sync(0xffffffffu, m == KB_MODE_FIT), anym = fitm | __ballot_sync(0xffffffffu, m == KB_MODE_PREEMPT);
    unsigned okb = 0;
    auto decide = [&](const i64 (&v0)[4], const i64 (&v1)[4], int p) {
#pragma unroll
      for (int k = 0; k < 4; k++) {
        const bool fit = (fitm >> (p + k)) & 1, any = (anym >> (p + k)) & 1;
        const i64 t0 = (fit && c0) ? v0[k] : INT64_MAX;
        const i64 d0r = (i64)((u64)srt0 - (u64)v0[k]);
        const i64 d0 = (any && c0 && d0r > 0) ? d0r : 0;
        i64 t1 = INT64_MAX, d1 = 0;
        if (kTwo) { t1 = (fit && c1) ? v1[k] : INT64_MAX; const i64 d1r = (i64)((u64)srt1 - (u64)v1[k]); d1 = (any && c1 && d1r > 0) ? d1r : 0; }
        const bool ok = __all_sync(0xffffffffu, urt0 <= t0 && (!kTwo || urt1 <= t1));  // the chain: compare -> vote -> add
        urt0 += ok ? d0 : 0;
        if (kTwo) urt1 += ok ? d1 : 0;
        okb |= (ok ? 1u : 0u) << (p + k);
      }
    };
    for (int p = 0; p < 32 && blk + p < n; p += 8) {
      fetch(b0, b1, blk + p + 4);
      decide(a0, a1, p);
      fetch(a0, a1, blk + p + 8);
      decide(b0, b1, p + 4);
    }
    if (lane == 0) { ok_bits[blk >> 5] = okb; mbar_arrive(blk_bar + (blk >> 5)); }
  }
  if (c0) s_u[fr0] = urt0;
  if (c1) s_u[fr1] = urt1;
}
__device__ __forceinline__ int flat_decision(int mode, const uint32_t *ok_bits, int pos) {
  if (mode == KB_MODE_FIT) return (ok_bits[pos >> 5] >> (pos & 31)) & 1 ? KB_DEC_ASSUMED : KB_DEC_SKIPPED_NO_FIT;
  return mode == KB_MODE_PREEMPT ? KB_DEC_PREEMPT_NO_TARGETS : KB_DEC_NOFIT;
}

#ifndef KB_FLAT_THREADS
#define KB_FLAT_THREADS 1024
#endif
#ifndef KB_FLAT_NG
#define KB_FLAT_NG 4  // lanes per entry in the nominate walks
#endif
// Entries that do not take the group walk of phase 5 (flat_nominate_group) go through the shared device functions on the relocated snapshot.
// They are out of line, so that their register needs do not constrain the rest of the kernel.
__device__ __noinline__ int flat_nominate_general(const DevSnap &L, int i, int *borrowing, unsigned gmask, int gbase, int glane) {
  bool need_search = false;  // stays false: no ClusterQueue of a relocated view has preemption candidates
  return get_assignments_coop<KB_FLAT_NG>(L, &need_search, i, borrowing, gmask, gbase, glane);
}
__device__ __noinline__ void flat_key_general(const DevSnap &L, int i, u64 *k) { compute_entry_key(L, i, k); }
__device__ __noinline__ void flat_expand_general(const DevSnap &L, int i, i64 *qrow, int FR) {
  for (int c = 0; c < FR; c++) qrow[c] = -1;
  expand_entry(L, i, qrow);
}
// Phase 5 of k_cycle_flat for an entry with one podset that cannot be reduced (the usual case): the group walk of
// findFlavorForPodSets on the shared tables.  One group of NG lanes per entry (as in get_assignments_coop), lane =
// flavor slot of the resource group being assigned, rounds of NG flavors; the lane evaluates fitsResourceQuota
// (flavorassigner.go:1017-1047, what cell_eval computes) for each resource of its flavor, reading the shared tables
// directly instead of through the relocated DevSnap.  On a flat tree every ClusterQueue hangs off the root, so
// find_height gives 0 or the root's height and mayReclaim is "fits within nominal"; no ClusterQueue has preemption
// candidates (candidates_possible), so SimulatePreemption is NoCandidates.  The flavors of a round are then taken in
// order by flavor_take, the rule get_assignments_coop uses.  The group also writes the podset's assignment row, the
// entry's mode / borrowing and its iterator key.  A group of one podset assigns like the podset alone.
// available / potentialAvailable (resource_node.go:104-133) of a ClusterQueue cell of a flat tree: sub, u, lq, bl of
// the cell, srt / urt the root's SubtreeQuota and usage in the same column
__device__ __forceinline__ void flat_cell_available(i64 sub, i64 u, i64 lq, i64 bl, i64 srt, i64 urt, i64 &av, i64 &pot) {
  i64 pa = srt - urt;
  pot = lq + srt;
  if (bl != KB_NO_LIMIT) { pa = imin((sub - lq) - imax(0, u - lq) + bl, pa); pot = imin(sub + bl, pot); }
  av = imax(0, lq - u) + pa;
}
// The lanes compute available / potentialAvailable of the cells they evaluate and the over-usage of the entry's own
// row themselves (the root's lendable is in s_lend from the tree pass), so the walk needs no sweep over the tree.
// With qrow set, the group also writes the entry's dense request row (Assignment.Usage.Quota, absent = -1).
template <int NG>
__device__ __forceinline__ void flat_nominate_group(const FlatLay &Y, int i, int R, int FR, unsigned flags, int pods, bool has_qr_table,
                                                    unsigned gmask, int gbase, int glane, i64 *qrow) {
  extern __shared__ __align__(16) unsigned char smem_raw[];  // the kernel's
  const i64 *s_u = (const i64 *)(smem_raw + Y.u), *s_sub = (const i64 *)(smem_raw + Y.sub), *s_lq = (const i64 *)(smem_raw + Y.lq),
            *s_bl = (const i64 *)(smem_raw + Y.bl);
  const unsigned char *s_blob = smem_raw + Y.blob;
  const TreeBlobHdr *BH = (const TreeBlobHdr *)s_blob;
  const int32_t *b_rgs = (const int32_t *)(s_blob + BH->rgs), *b_rgfl = (const int32_t *)(s_blob + BH->rgfl), *b_fl = (const int32_t *)(s_blob + BH->fl);
  const uint32_t *b_rgmask = (const uint32_t *)(s_blob + BH->rgmask);
  const i64 *r_req = (const i64 *)(smem_raw + Y.r_req);
  int8_t *o_fl = (int8_t *)(smem_raw + Y.o_fl), *o_md = (int8_t *)(smem_raw + Y.o_md), *o_tr = (int8_t *)(smem_raw + Y.o_tr);
  const bool fair = (flags & KB_F_FAIR_SHARING) != 0, fung = (flags & KB_F_FLAVOR_FUNGIBILITY) != 0;

  const int hq = ((const int *)(smem_raw + Y.e_cq))[i], l = ((const int *)(smem_raw + Y.e_psn))[i];
  const u64 ok = ((const u64 *)(smem_raw + Y.r_ok))[l];
  const int cnt = ((const int *)(smem_raw + Y.r_count))[l];
  const i64 lg = ((const i64 *)(smem_raw + Y.e_lg))[i];
  const bool use_last = fung && lg >= 0 && !(((const i64 *)(s_blob + BH->gen))[hq] > lg);
  const int pref = s_blob[BH->pref + hq], wcb = s_blob[BH->wcb + hq], wcp = s_blob[BH->wcp + hq];
  const bool can_pwb = s_blob[BH->borrow_w + hq] != KB_POLICY_NEVER || (fair && s_blob[BH->reclaim + hq] != KB_POLICY_NEVER);  // :1049-1052
  const int P = ((const int32_t *)(s_blob + BH->par))[hq];
  const int hp = ((const int32_t *)(s_blob + BH->hgt))[P];  // borrow height of a cell above nominal
  const int rg0 = b_rgs[hq], rg1 = b_rgs[hq + 1];
  bool covers = false;  // pods resource flavorassigner.go:585-587
  if (pods >= 0) for (int g = rg0; g < rg1; g++) if ((b_rgmask[g] >> pods) & 1) covers = true;
  const uint32_t mask = ((const uint32_t *)(smem_raw + Y.r_mask))[l] | (covers ? 1u << pods : 0u);
  auto request = [&](int r) { return covers && r == pods ? (i64)cnt : r_req[(size_t)l * R + r]; };  // full count: ps_request unscaled
  // resource r of the row is written by lane r % NG only, so the row needs no synchronisation within the group
  for (int r = glane; r < R; r += NG) { o_fl[(size_t)l * R + r] = -1; o_md[(size_t)l * R + r] = -1; o_tr[(size_t)l * R + r] = -1; }
  uint32_t assigned = 0, ps_pmask = 0;
  int ps_borrow = 0;
  bool has_reasons = false, failed = false;
  for (int r0 = 0; r0 < R; r0++) {  // resource groups in the order of their first requested resource
    if (!((mask >> r0) & 1) || ((assigned >> r0) & 1)) continue;
    int g = -1;
    for (int k = rg0; k < rg1 && g < 0; k++) if ((b_rgmask[k] >> r0) & 1) g = k;
    if (g < 0) {
      if (request(r0) == 0) continue;
      has_reasons = failed = true;
      break;
    }
    const uint32_t rgm = b_rgmask[g] & mask;
    const int fl0 = b_rgfl[g], nfl = b_rgfl[g + 1] - fl0;
    int best_f = -1, best_pm = PM_NOFIT, best_rb = INT32_MAX, best_maxb = 0, attempted = -1;
    uint32_t best_pmask = 0;
    bool any_reason = false, done = false;
    for (int base = use_last ? ((const int8_t *)(smem_raw + Y.r_last))[(size_t)l * R + r0] + 1 : 0; base < nfl && !done; base += NG) {
      // ---- one flavor per lane: representative mode over its resources, as in assign_workload_coop ----
      const int idx = base + glane;
      u64 res = 0;  // [0..2] rpm [3..9] rb [10..16] maxb [17] any_reason [19] eligible [20..27] flavor [32..63] pmask
      if (idx < nfl) {
        const int f = b_fl[fl0 + idx];
        if ((ok >> f) & 1) {  // ps_flavor_ok: checkFlavorForPodSets
          int rpm = PM_FIT, rb = 0, maxb = 0; uint32_t pmask = 0; bool reason = false;
          for (int r = 0; r < R; r++) {
            if (!((rgm >> r) & 1)) continue;
            const int fr = f * R + r, c = hq * FR + fr;
            const i64 val = request(r), sub = s_sub[c], u = s_u[c];
            i64 av, pot;
            flat_cell_available(sub, u, s_lq[c], s_bl[c], s_sub[fr], s_u[fr], av, pot);
            int pm = PM_NOFIT, b = 0;
            if (val <= pot) {  // cell_eval: find_height on a flat tree is the root's height above nominal, mayReclaim below
              const bool above = u + val > sub;  // nominal == SubtreeQuota for a ClusterQueue
              b = above ? hp : 0;
              pm = fits_mode(val, av, sub, !above, [&] { return can_pwb; });
              if (pm == PM_NEED) pm = PM_NOCAND;  // no candidates: what SimulatePreemption returns
            }
            if (pm != PM_FIT) reason = true;
            if (gm_preferred(rpm, rb, pm, b, pref)) { rpm = pm; rb = b; }
            if (rpm == PM_NOFIT) break;
            if (fa_mode(pm) == KB_MODE_PREEMPT) pmask |= 1u << r;
            if (b > maxb) maxb = b;
          }
          res = (u64)rpm | ((u64)(rb & 127) << 3) | ((u64)(maxb & 127) << 10) | ((u64)reason << 17) | (1ull << 19) | ((u64)f << 20) |
                ((u64)pmask << 32);
        }
      }
      // ---- ordered walk over the flavors of this round ----
      for (int j = 0; j < NG && base + j < nfl; j++) {
        const u64 rj = __shfl_sync(gmask, res, gbase + j);
        attempted = base + j;
        if (!((rj >> 19) & 1)) { any_reason = true; continue; }
        const int rpm = (int)(rj & 7), rb = (int)((rj >> 3) & 127);
        if ((rj >> 17) & 1) any_reason = true;
        if (flavor_take(fung, wcb, wcp, pref, rpm, rb, best_pm, best_rb, &done)) {
          best_f = (int)((rj >> 20) & 255); best_pm = rpm; best_rb = rb; best_maxb = (int)((rj >> 10) & 127); best_pmask = (uint32_t)(rj >> 32);
        }
        if (done) break;
      }
    }
    if (best_f < 0) { has_reasons = failed = true; break; }
    const int tried = fung ? (attempted == nfl - 1 ? -1 : attempted) : 0;
    for (int r = glane; r < R; r += NG)
      if ((rgm >> r) & 1) { o_fl[(size_t)l * R + r] = (int8_t)best_f; o_md[(size_t)l * R + r] = (best_pmask >> r) & 1 ? KB_MODE_PREEMPT : KB_MODE_FIT; o_tr[(size_t)l * R + r] = (int8_t)tried; }
    assigned |= rgm;
    ps_pmask |= best_pmask & rgm;
    if (best_maxb > ps_borrow) ps_borrow = best_maxb;
    if (best_pm != PM_FIT && any_reason) has_reasons = true;
  }
  int mode = KB_MODE_FIT, borrowing = 0;
  if (failed) {
    mode = KB_MODE_NOFIT;
    for (int r = glane; r < R; r += NG) { o_fl[(size_t)l * R + r] = -1; o_md[(size_t)l * R + r] = -1; o_tr[(size_t)l * R + r] = -1; }
  } else {
    borrowing = ps_borrow;
    if (has_reasons) mode = (assigned & mask) == 0 ? KB_MODE_NOFIT : ((ps_pmask & mask) ? KB_MODE_PREEMPT : KB_MODE_FIT);
  }
  // iterator key: max over the resources of the DominantResourceShare terms of entry_share_ratio
  double best = 0.0;
  if (fair) {
    const i64 *s_lend = (const i64 *)(smem_raw + Y.lend);
    for (int r = glane; r < R; r += NG) {
      i64 bo = 0;  // over-usage of the row in resource r, summed over the flavors
      for (int c = hq * FR + r; c < (hq + 1) * FR; c += R) bo += imax(0, s_u[c] - s_sub[c]);
      const int f = o_fl[(size_t)l * R + r];
      if (f >= 0) {
        const int c = hq * FR + f * R + r;
        const i64 q = request(r), base = s_u[c] - s_sub[c];
        bo += imax(0, base + (q > 0 ? q : 0)) - imax(0, base);
      }
      const i64 lend = s_lend[P * R + r];
      const double ratio = (bo > 0 && lend > 0) ? (double)bo * 1000.0 / (double)lend : 0.0;
      if (ratio > best) best = ratio;
    }
    for (int o = NG >> 1; o > 0; o >>= 1) { const double x = __shfl_xor_sync(gmask, best, o); if (x > best) best = x; }
  }
  if (glane == 0) {
    ((int *)(smem_raw + Y.o_cnt))[l] = cnt;
    ((int *)(smem_raw + Y.e_mode))[i] = mode; ((int *)(smem_raw + Y.e_borrow))[i] = borrowing;
    (smem_raw + Y.e_fast)[i] = covers ? 3 : 1;
    entry_key_pack(flags, fair, best, fair ? ((const double *)(s_blob + BH->wgt))[hq] : 0.0, ((const int *)(smem_raw + Y.e_prio))[i],
                   ((const i64 *)(smem_raw + Y.e_ts))[i], has_qr_table && (smem_raw + Y.e_qr)[i], borrowing,
                   fair ? (unsigned)((const int32_t *)(s_blob + BH->gid))[hq] : (unsigned)((const int *)(smem_raw + Y.e_gid))[i],
                   (u64 *)(smem_raw + Y.key) + (size_t)i * 4);
  }
  if (qrow) {  // one podset: the row is its request on the assigned flavors
    __syncwarp(gmask);  // the assignment row was written by all lanes of the group
    for (int fr = glane; fr < FR; fr += NG) {
      const int f = fr / R, r = fr - f * R;
      qrow[fr] = o_fl[(size_t)l * R + r] == f ? request(r) : -1;
    }
  }
}

__global__ void __launch_bounds__(KB_FLAT_THREADS) k_cycle_flat(const __grid_constant__ DevSnap D, const __grid_constant__ FlatLay Y) {
  extern __shared__ __align__(16) unsigned char smem_raw[];
  const int FR = D.FR, R = D.R;
  const int t = blockIdx.x, tid = threadIdx.x, nthreads = blockDim.x;
  const int lane = tid & 31, warp = tid >> 5;
  const int fr_sh = 31 - __clz(FR); const bool fr_p2 = (1 << fr_sh) == FR;
  auto row_of = [&](int i) { return fr_p2 ? i >> fr_sh : i / FR; };
  auto col_of = [&](int i) { return fr_p2 ? i & (FR - 1) : i % FR; };
  long long tk0 = clock64();
  // phase probe (tools/phase_probe.py): SM cycles of thread 0 of CTA 0 since the previous point
#define KB_FPHASE(k) do { if (blockIdx.x == 0 && threadIdx.x == 0) { long long now_ = clock64(); D.sstat[k] = (u64)(now_ - tk0); tk0 = now_; } } while (0)
  i64 *s_u = (i64 *)(smem_raw + Y.u), *s_sub = (i64 *)(smem_raw + Y.sub), *s_lq = (i64 *)(smem_raw + Y.lq), *s_bl = (i64 *)(smem_raw + Y.bl);
  i64 *s_av = (i64 *)(smem_raw + Y.av), *s_pot = (i64 *)(smem_raw + Y.pot), *s_over = (i64 *)(smem_raw + Y.over), *s_lend = (i64 *)(smem_raw + Y.lend);
  unsigned char *s_blob = smem_raw + Y.blob;
  int *n_e = (int *)(smem_raw + Y.n_e), *n_wl = (int *)(smem_raw + Y.n_wl), *n_ps0 = (int *)(smem_raw + Y.n_ps0), *n_psn = (int *)(smem_raw + Y.n_psn);
  int *e_gid = (int *)(smem_raw + Y.e_gid), *e_cq = (int *)(smem_raw + Y.e_cq), *e_prio = (int *)(smem_raw + Y.e_prio), *e_ident = (int *)(smem_raw + Y.e_ident);
  int *e_psn = (int *)(smem_raw + Y.e_psn), *e_at = (int *)(smem_raw + Y.e_at);  // e_at: the entry at each iterator position
  unsigned long long *blk_bar = (unsigned long long *)(smem_raw + Y.blk_bar);    // one per 32 positions (flat_ordered_loop)
  i64 *e_ts = (i64 *)(smem_raw + Y.e_ts), *e_lg = (i64 *)(smem_raw + Y.e_lg); uint8_t *e_qr = smem_raw + Y.e_qr;
  uint8_t *e_fast = smem_raw + Y.e_fast;  // bit 0: nominated by the group walk, bit 1: its ClusterQueue covers the pods resource
  int *e_mode = (int *)(smem_raw + Y.e_mode), *e_borrow = (int *)(smem_raw + Y.e_borrow), *e_rank = (int *)(smem_raw + Y.e_rank);
  int *m_sorted = (int *)(smem_raw + Y.m_sorted); uint32_t *ok_bits = (uint32_t *)(smem_raw + Y.d_sorted);
  int *r_gid = (int *)(smem_raw + Y.r_gid), *r_count = (int *)(smem_raw + Y.r_count), *r_min = (int *)(smem_raw + Y.r_min);
  uint32_t *r_mask = (uint32_t *)(smem_raw + Y.r_mask); int *r_group = (int *)(smem_raw + Y.r_group); u64 *r_ok = (u64 *)(smem_raw + Y.r_ok);
  i64 *r_req = (i64 *)(smem_raw + Y.r_req); int8_t *r_last = (int8_t *)(smem_raw + Y.r_last);
  int8_t *o_fl = (int8_t *)(smem_raw + Y.o_fl), *o_md = (int8_t *)(smem_raw + Y.o_md), *o_tr = (int8_t *)(smem_raw + Y.o_tr); int *o_cnt = (int *)(smem_raw + Y.o_cnt);
  u64 *s_key = (u64 *)(smem_raw + Y.key);
  int *s_misc = (int *)(smem_raw + Y.misc);  // [0] n entries, [1] total rows

  // ---- 0. staging.  Everything this CTA will read from global memory is requested here, all loads independent.
  const int ts0 = D.tree_start[t];
  const int nn = D.tree_start[t + 1] - ts0;
  const int tb = nn * FR;
  const size_t r0 = (size_t)ts0 * FR;  // first cell of the tree in the tree-local tables (DevSnap::tl_*)
  int4 *s_rec = (int4 *)(smem_raw + Y.rec);
  __shared__ __align__(8) unsigned long long s_mbar[2];
  // Two stages, both requested here.  Stage A is what the entry compaction and the tree pass of phase 1 read: head
  // records, usage, localQuota.  Stage B is read from the end of phase 1 on: SubtreeQuota, borrowing limits and the
  // static tree block; it lands while phase 1 runs.  A root's rows are contiguous in the tree-local tables -> one bulk
  // copy per table, issued by one thread, completion counted in bytes on the stage's mbarrier.  Rows of odd width are
  // not 16 B aligned: per-thread cp.async, one commit group per stage.
  // SubtreeQuota and localQuota arrive final (k_tl_static / k_tl_root): the tree pass below only sums usage.
  if ((FR & 1) == 0) {
    if (tid == 0) { mbar_init(&s_mbar[0], 1); mbar_init(&s_mbar[1], 1); }
    __syncthreads();
    if (tid == 0) {
      const int b0 = D.tree_blob_off[t], bn = D.tree_blob_off[t + 1] - b0;  // static block of the tree (multiple of 16 B)
      const unsigned tbytes = (unsigned)tb * 8u;
      mbar_expect_tx(&s_mbar[0], 2u * tbytes + (unsigned)nn * 16u);
      bulk_g2s(s_rec, D.cq_rec + ts0, (unsigned)nn * 16u, &s_mbar[0]);
      bulk_g2s(s_u, D.tl_usage + r0, tbytes, &s_mbar[0]);      // ClusterQueue usage, zero rows for cohorts
      bulk_g2s(s_lq, D.tl_lquota + r0, tbytes, &s_mbar[0]);
      mbar_expect_tx(&s_mbar[1], 2u * tbytes + (unsigned)bn);
      bulk_g2s(s_sub, D.tl_subtree + r0, tbytes, &s_mbar[1]);
      bulk_g2s(s_bl, D.tl_blimit + r0, tbytes, &s_mbar[1]);
      bulk_g2s(s_blob, D.tree_blob + b0, (unsigned)bn, &s_mbar[1]);
    }
    if (tid == nthreads - 1) *(DevSnap *)(smem_raw + Y.snap) = D;  // bulk of the relocated view (patched below), under the load latency
    mbar_wait(&s_mbar[0], 0);
  } else {
    for (int h = tid; h < nn; h += nthreads) cp_async16(s_rec + h, D.cq_rec + ts0 + h);
    for (int i = tid; i < tb; i += nthreads) { cp_async_small<8>(s_u + i, D.tl_usage + r0 + i); cp_async_small<8>(s_lq + i, D.tl_lquota + r0 + i); }
    cp_async_commit();
    {
      const int b0 = D.tree_blob_off[t], bn = D.tree_blob_off[t + 1] - b0;  // static block of the tree (multiple of 16 B)
      for (int c = tid * 16; c < bn; c += nthreads * 16) cp_async16(s_blob + c, D.tree_blob + b0 + c);
    }
    for (int i = tid; i < tb; i += nthreads) { cp_async_small<8>(s_sub + i, D.tl_subtree + r0 + i); cp_async_small<8>(s_bl + i, D.tl_blimit + r0 + i); }
    cp_async_commit();
    if (tid == nthreads - 1) *(DevSnap *)(smem_raw + Y.snap) = D;
    cp_async_wait_prior1();  // stage A
    __syncthreads();
  }
  bool general_mine = false;  // a head of the general walk (see phase 2)
  for (int h = tid; h < nn; h += nthreads) {  // the head of every ClusterQueue of the tree (record written by k_flat_prep / k_cq_rec)
    const int4 rc = s_rec[h];
    const bool live = ((unsigned)rc.w >> 16) == D.rec_stamp;  // written for this cycle
    n_e[h] = live ? rc.x : -1; n_wl[h] = rc.y; n_ps0[h] = rc.z; n_psn[h] = live ? (rc.w & (KB_REC_GENERAL - 1)) : 0;
    if (live) {  // the entry's per-cycle records are copied in phase 1: request their lines now
      auto touch = [](const void *p) { asm volatile("prefetch.global.L2 [%0];" ::"l"(p)); };
      const int wl = rc.y, row = rc.z;
      touch(D.wl_priority + wl); touch(D.wl_ts + wl); touch(D.wl_last_gen + wl);
      if (D.wl_has_qr) touch(D.wl_has_qr + wl);
      if ((rc.w & (KB_REC_GENERAL - 1)) > 0) {
        touch(D.ps_count + row); touch(D.ps_min_count + row); touch(D.ps_req_mask + row); touch(D.ps_flavor_ok + row);
        touch(D.ps_req + (size_t)row * R); touch(D.ps_last_tried + (size_t)row * R);
        if (D.ps_group) touch(D.ps_group + row);
      }
      if (rc.w & KB_REC_GENERAL) general_mine = true;
    }
  }
  // The general walk reads available / potentialAvailable and the fair-sharing sums of every cell: the sweep of
  // phase 2 runs only for a root with a head of the general walk.
  const bool sweep = __syncthreads_or(general_mine);
  KB_FPHASE(0);
  const bool fair = (D.flags & KB_F_FAIR_SHARING) != 0;  // every tree is flat here: all entries take the fair flat key

  // ---- 1. entries of the root in ClusterQueue (= local handle) order + local podset-row numbering, and the
  // bottom-up pass of the flat tree for everyone: accumulateFromChild resource_node.go:210-217, children -> root
  // one warp per 32 nodes: ballot + warp scan, then the warps' totals are scanned (chunks of 32 warps, carried).
  // The thread that places an entry copies its per-cycle records (one hop: the workload / row ids are in the head
  // record) with cp.async; they land while the tree pass runs and are waited for at the end of the phase.
  {
    // ps_last_tried rows by words when they are word aligned on both sides, byte by byte otherwise
    const bool lt_words = (R & 3) == 0 && ((uintptr_t)D.ps_last_tried & 3) == 0;
    const int nw = nthreads >> 5;
    int *w_cnt = s_misc + 4, *w_rows = s_misc + 4 + 32;  // [32] each (misc is 64 + 256 B)
    int cnt_base = 0, rows_base = 0;
    for (int c0 = 0; c0 < nn; c0 += nthreads) {
      const int h = c0 + tid;
      const int e = h < nn ? n_e[h] : -1;
      const int pn = e >= 0 ? n_psn[h] : 0;
      const unsigned m = __ballot_sync(0xffffffffu, e >= 0);
      int incl = pn;  // inclusive scan of the row counts over the lanes
      for (int o = 1; o < 32; o <<= 1) { int v = __shfl_up_sync(0xffffffffu, incl, o); if (lane >= o) incl += v; }
      if (lane == 31) { w_cnt[warp] = __popc(m); w_rows[warp] = incl; }
      __syncthreads();
      int pc = 0, pr = 0, tc = 0, tr = 0;  // totals of the warps before mine / of all warps of this chunk
      {
        const int wc = lane < nw ? w_cnt[lane] : 0, wr = lane < nw ? w_rows[lane] : 0;
        int ic = wc, ir = wr;
        for (int o = 1; o < 32; o <<= 1) { int a = __shfl_up_sync(0xffffffffu, ic, o), b = __shfl_up_sync(0xffffffffu, ir, o); if (lane >= o) { ic += a; ir += b; } }
        pc = __shfl_sync(0xffffffffu, ic - wc, warp & 31); pr = __shfl_sync(0xffffffffu, ir - wr, warp & 31);
        tc = __shfl_sync(0xffffffffu, ic, 31); tr = __shfl_sync(0xffffffffu, ir, 31);
      }
      if (e >= 0) {
        const int i = cnt_base + pc + __popc(m & ((1u << lane) - 1)), l0 = rows_base + pr + incl - pn;
        const int wl = n_wl[h], ps0 = n_ps0[h];
        e_gid[i] = e; e_cq[i] = h; e_ident[i] = i; e_psn[i] = l0;
        e_fast[i] = (s_rec[h].w & KB_REC_GENERAL) ? 0 : 1;
        n_e[h] = i;  // from here on: the local entry of the ClusterQueue (publish)
        cp_async_small<4>(e_prio + i, D.wl_priority + wl); cp_async_small<8>(e_ts + i, D.wl_ts + wl); cp_async_small<8>(e_lg + i, D.wl_last_gen + wl);
        if (D.wl_has_qr) e_qr[i] = D.wl_has_qr[wl];
        for (int k = 0; k < pn; k++) {  // every podset row of the entry, for either walk
          const int row = ps0 + k, l = l0 + k;
          r_gid[l] = row;
          cp_async_small<4>(r_count + l, D.ps_count + row); cp_async_small<4>(r_min + l, D.ps_min_count + row);
          cp_async_small<4>(r_mask + l, D.ps_req_mask + row); cp_async_small<8>(r_ok + l, D.ps_flavor_ok + row);
          if (D.ps_group) cp_async_small<4>(r_group + l, D.ps_group + row); else r_group[l] = -1;
          for (int r = 0; r < R; r++) cp_async_small<8>(r_req + (size_t)l * R + r, D.ps_req + (size_t)row * R + r);
          if (lt_words) for (int r = 0; r < R; r += 4) cp_async_small<4>(r_last + (size_t)l * R + r, D.ps_last_tried + (size_t)row * R + r);
          else for (int r = 0; r < R; r++) r_last[(size_t)l * R + r] = D.ps_last_tried[(size_t)row * R + r];
        }
      }
      cnt_base += tc; rows_base += tr;
      if (c0 + nthreads < nn) __syncthreads();  // w_cnt / w_rows are rewritten by the next chunk
    }
    if (tid == 0) { e_psn[cnt_base] = rows_base; s_misc[0] = cnt_base; s_misc[1] = rows_base; }
  }
  if (nthreads % FR == 0) {  // a thread stays in one column: private partial sums over its rows
    const int fr = tid % FR, g = tid / FR, G = nthreads / FR;
    i64 dus = 0;
    for (int h = 1 + g; h < nn; h += G) { const int c = h * FR + fr; dus += imax(0, s_u[c] - s_lq[c]); }
    const int pitch = FR + 1;  // padded: the column-wise read below is conflict free
    if ((size_t)tb >= (size_t)G * pitch) {
      // partials -> scratch (avail is not written yet), one warp per column sums them by shuffles
      i64 *p_u = s_av;
      p_u[g * pitch + fr] = dus;
      __syncthreads();
      for (int c = warp; c < FR; c += nthreads >> 5) {
        i64 b = 0;
        for (int k = lane; k < G; k += 32) b += p_u[k * pitch + c];
        for (int o = 16; o > 0; o >>= 1) b += __shfl_xor_sync(0xffffffffu, b, o);
        if (lane == 0) s_u[c] += b;
      }
    } else if (dus) {  // small tree: few rows per column, little contention
      atomicAdd((u64 *)&s_u[fr], (u64)dus);
    }
  } else {
    for (int c = FR + tid; c < tb; c += nthreads) {
      const i64 spill = imax(0, s_u[c] - s_lq[c]);
      if (spill) atomicAdd((u64 *)&s_u[col_of(c)], (u64)spill);
    }
  }
  // stage B and this thread's record copies have landed (a CTA never exits with a copy in flight into its shared memory)
  if ((FR & 1) == 0) {
    mbar_wait(&s_mbar[1], 0);
    cp_async_wait_all();
  } else {
    cp_async_wait_all();
    __syncthreads();  // stage B was copied by every thread
  }
  const TreeBlobHdr *BH = (const TreeBlobHdr *)s_blob;
  const int32_t *b_gid = (const int32_t *)(s_blob + BH->gid), *b_par = (const int32_t *)(s_blob + BH->par), *b_hgt = (const int32_t *)(s_blob + BH->hgt);
  const uint8_t *b_reclaim = s_blob + BH->reclaim;
  // the relocated snapshot: every table the shared device functions read, in local numbering.  It lives in shared
  // memory itself (one thread fills it in): ~50 patched pointers would otherwise sit in every thread's stack.
  if (tid == nthreads - 1) {
  DevSnap &L = *(DevSnap *)(smem_raw + Y.snap);
  L.tab_local = 2; L.local_flat = 1; L.ent_gid = e_gid; L.node_gid = b_gid;
  L.parent = b_par; L.height = b_hgt; L.lq = s_lq;
  L.nominal = s_sub;  // only ever read for ClusterQueues: SubtreeQuota == Nominal there (resource_node.go:160-166)
  L.subtree = s_sub; L.usage = s_u; L.avail = s_av; L.potential = s_pot; L.blimit = s_bl; L.fs_over = s_over; L.fs_lend = s_lend;
  L.fair_weight = (const double *)(s_blob + BH->wgt); L.cq_generation = (const i64 *)(s_blob + BH->gen);
  L.cq_within_cq = s_blob + BH->within; L.cq_reclaim_within = b_reclaim; L.cq_borrow_within = s_blob + BH->borrow_w;
  L.cq_when_can_borrow = s_blob + BH->wcb; L.cq_when_can_preempt = s_blob + BH->wcp; L.cq_preference = s_blob + BH->pref;
  L.cq_rg_start = (const int32_t *)(s_blob + BH->rgs); L.rg_res_mask = (const uint32_t *)(s_blob + BH->rgmask);
  L.rg_flavor_start = (const int32_t *)(s_blob + BH->rgfl); L.rg_flavors = (const int32_t *)(s_blob + BH->fl);
  L.heads = e_ident; L.wl_cq = e_cq; L.wl_priority = e_prio; L.wl_ts = e_ts; L.wl_last_gen = e_lg; L.wl_ps_start = e_psn;
  L.wl_has_qr = D.wl_has_qr ? e_qr : nullptr;
  L.ps_req = r_req; L.ps_req_mask = r_mask; L.ps_count = r_count; L.ps_min_count = r_min; L.ps_flavor_ok = r_ok; L.ps_last_tried = r_last;
  L.ps_group = D.ps_group ? r_group : nullptr;
  L.ps_flavor = o_fl; L.ps_res_mode = o_md; L.ps_tried = o_tr; L.ps_count_out = o_cnt;
  L.borrow = e_borrow;
  }
  // the root's lendable per resource (k_fair_prep): potentialAvailable of the root == its SubtreeQuota, static
  if (fair)
    for (int r = tid; r < R; r += nthreads) {
      i64 lend = 0;
      for (int c = r; c < FR; c += R) lend += s_sub[c];
      s_lend[r] = lend;
    }
  __syncthreads();
  KB_FPHASE(1);
  const int n = s_misc[0], nrows = s_misc[1];
  if (n == 0) {
    for (int i = tid; i < tb; i += nthreads) D.usage[(size_t)b_gid[row_of(i)] * FR + col_of(i)] = s_u[i];
    return;
  }
  const DevSnap &L = *(const DevSnap *)(smem_raw + Y.snap);
  // ---- 2. for the general walk only: available / potentialAvailable (resource_node.go:104-133) of every cell in one
  // sweep, with the fair-sharing inputs (k_fair_prep: over-usage per (ClusterQueue, resource), lendable per (node,
  // resource)) summed by shuffles when a row is one aligned segment of a warp, in a pass of their own otherwise
  if (sweep) {
    const bool fair_rows = fair && FR <= 32 && fr_p2 && (R & (R - 1)) == 0;
    const int tb_sweep = fair_rows ? (tb + 31) & ~31 : tb;
    for (int i = tid; i < tb_sweep; i += nthreads) {
      i64 pot = 0, over = 0;
      if (i < tb) {
        const int fr = col_of(i);
        const i64 sub = s_sub[i], u = s_u[i];
        if (i < FR) { s_av[i] = sub - u; pot = sub; }
        else { i64 av; flat_cell_available(sub, u, s_lq[i], s_bl[i], s_sub[fr], s_u[fr], av, pot); s_av[i] = av; }
        s_pot[i] = pot;
        over = imax(0, u - sub);
      }
      if (fair_rows) {
        i64 lend = pot;
        for (int o = R; o < FR; o <<= 1) { lend += __shfl_xor_sync(0xffffffffu, lend, o); over += __shfl_xor_sync(0xffffffffu, over, o); }
        if (i < tb && col_of(i) < R) { const int h = row_of(i); s_lend[h * R + col_of(i)] = lend; s_over[h * R + col_of(i)] = over; }
      }
    }
    __syncthreads();
    if (fair && !fair_rows) {
      const int Fn = D.F;
      for (int i = tid; i < nn * R; i += nthreads) {
        const int h = i / R, r = i % R;
        i64 over = 0, lend = 0;
        for (int f = 0; f < Fn; f++) {
          const int c = h * FR + f * R + r;
          lend += s_pot[c];
          const i64 o = s_u[c] - s_sub[c];
          if (o > 0) over += o;
        }
        s_lend[i] = lend; s_over[i] = over;
      }
      __syncthreads();
    }
  }
  // ---- 3. one pass per entry, KB_FLAT_NG lanes each, on the records staged in phase 1: nominate (getInitialAssignments,
  // scheduler.go:584-625), iterator key and dense request row (Assignment.Usage.Quota, absent = -1), with no barrier in
  // between.  Entries with one podset that cannot be reduced take the group walk on
  // the shared tables (flat_nominate_group); every other entry (several podsets, or partial admission with a reducible
  // podset) takes get_assignments_coop on the relocated snapshot L.  A round evaluates KB_FLAT_NG flavors of a resource
  // group at once; the walk usually stops in its first round, so fewer lanes per entry mean fewer warps competing for
  // the SM's issue slots at the same chain length.
  i64 *s_q = s_av;    // [n][FR]: written here when there is no sweep, after this pass otherwise (avail is live until then)
  i64 *s_lim = s_pot; // [n][FR] thresholds in iterator order
  int walked = 0;
  {
    const int glane = lane % KB_FLAT_NG, gbase = lane - glane;
    const unsigned gmask = (KB_FLAT_NG == 32 ? 0xffffffffu : ((1u << KB_FLAT_NG) - 1u)) << gbase;
    const int groups = nthreads / KB_FLAT_NG;
    bool fast_mine = false;  // lane k of a group reports the entry of its round k: every entry < nthreads once
    for (int i0 = 0, k = 0; i0 < n; i0 += groups, k++) {
      const int i = i0 + tid / KB_FLAT_NG;
      if (i >= n) continue;  // whole lane groups take the branches together
      const bool fast = e_fast[i] & 1;
      if (fast) {
        flat_nominate_group<KB_FLAT_NG>(Y, i, R, FR, D.flags, D.pods_res, D.wl_has_qr != nullptr, gmask, gbase, glane,
                                        sweep ? nullptr : s_q + (size_t)i * FR);
      } else {
        int borrowing;
        const int mode = flat_nominate_general(L, i, &borrowing, gmask, gbase, glane);
        if (glane == 0) { e_mode[i] = mode; e_borrow[i] = borrowing; }
        __syncwarp(gmask);  // the assignment rows were written by all lanes of the group
        if (glane == 0) flat_key_general(L, i, s_key + (size_t)i * 4);
      }
      if (glane == k) fast_mine = fast;
    }
    walked = __syncthreads_count(fast_mine);
  }
  if (blockIdx.x == 0 && tid == 0) { D.sstat[8] = (u64)walked; D.sstat[9] = (u64)min(n, nthreads); }  // CTA 0: group walk / entries, of the first nthreads
  if (sweep) {  // request rows, now that avail is dead
    const bool r_p2 = (R & (R - 1)) == 0;
    const int r_sh = 31 - __clz(R);
    for (int c = tid; c < n * FR; c += nthreads) {  // the group walk's entries, cell-parallel (one podset: the row is its request)
      const int i = row_of(c);
      const int fb = e_fast[i];
      if (!(fb & 1)) continue;
      const int fr = col_of(c), f = r_p2 ? fr >> r_sh : fr / R, r = fr - f * R;
      const int l = e_psn[i];
      i64 q = -1;
      if (o_fl[(size_t)l * R + r] == f) q = (fb & 2) && r == D.pods_res ? (i64)o_cnt[l] : r_req[(size_t)l * R + r];
      s_q[c] = q;
    }
    for (int i = tid; i < n; i += nthreads)
      if (!(e_fast[i] & 1)) flat_expand_general(L, i, s_q + (size_t)i * FR, FR);
    __syncthreads();
  }
  KB_FPHASE(2);
  // ---- 4. position in the iterator order: S lanes share the comparisons of one entry, then write its thresholds
  // (see flat_ordered_loop) at that position
  {
    int S = 32;
    while (S > 1 && n * S > nthreads) S >>= 1;
    const int per = nthreads / S, sub = tid % S;
    for (int base = 0; base < n; base += per) {
      const int i = base + tid / S;
      const bool act = i < n;
      int cnt = 0;
      if (act) {
        const u64 *mine = s_key + (size_t)i * 4;
        for (int j = sub; j < n; j += S) cnt += key4_less(s_key + (size_t)j * 4, mine) ? 1 : 0;
      }
      for (int o = S >> 1; o > 0; o >>= 1) cnt += __shfl_xor_sync(0xffffffffu, cnt, o);
      if (!act) continue;
      const int mode = e_mode[i], hq = e_cq[i];
      if (sub == 0) { e_rank[i] = cnt; m_sorted[cnt] = mode; e_at[cnt] = i; }
      for (int fr = sub; fr < FR; fr += S) {
        const i64 q = s_q[(size_t)i * FR + fr];
        const int r = hq * FR + fr;
        const i64 u = s_u[r], l = s_lq[r], bl = s_bl[r], sb = s_sub[r];
        const i64 A = imax(0, l - u);
        i64 v = INT64_MAX;  // Fit: threshold on the root usage; Preempt: SubtreeQuota_root - amount added to the root
        if (mode == KB_MODE_FIT) {
          if (q > 0) {
            const i64 x = q - A;
            const bool cap_ok = bl == KB_NO_LIMIT || (sb - l) - imax(0, u - l) + bl >= x;
            v = cap_ok ? s_sub[fr] - x : INT64_MIN;
          }
        } else if (mode == KB_MODE_PREEMPT) {
          i64 amt = 0;
          if (q >= 0 && b_reclaim[hq] != KB_POLICY_ANY) {  // quotaResourcesToReserve scheduler.go:530-548
            const i64 rsv = e_borrow[i] > 0 ? (bl == KB_NO_LIMIT ? q : imin(q, sb + bl - u)) : imax(0, imin(q, sb - u));
            amt = rsv > A ? rsv - A : 0;
          }
          v = s_sub[fr] - amt;
        }
        s_lim[(size_t)cnt * FR + fr] = v;
      }
    }
  }
  for (int b = tid; b < (n + 31) >> 5; b += nthreads) mbar_init(blk_bar + b, 1);  // arrived on by warp 0 (flat_ordered_loop)
  __syncthreads();
  KB_FPHASE(3);
  // ---- 5. the ordered loop on warp 0, and 6. publication behind it on the other warps: usage table with the
  // ClusterQueue rows of the admitted / reserving entries (cq.AddUsage) applied on the way out, decisions, flavor
  // assignment rows.  Only a ClusterQueue row of an entry and its decision wait for the loop, each for the block of 32
  // positions that holds the entry; the root row is the loop's own result.
  auto final_usage = [&](int h, int c) {  // cell c of row h
    const int i = n_e[h];
    i64 u = s_u[c];
    if (i >= 0) {
      const int dec = flat_decision(e_mode[i], ok_bits, e_rank[i]);
      const i64 q = s_q[(size_t)i * FR + (c - h * FR)];
      if (dec == KB_DEC_ASSUMED) { if (q > 0) u += q; }
      else if (dec == KB_DEC_PREEMPT_NO_TARGETS && q >= 0 && b_reclaim[h] != KB_POLICY_ANY) {
        const i64 bl = s_bl[c], sb = s_sub[c];
        u = u + (e_borrow[i] > 0 ? (bl == KB_NO_LIMIT ? q : imin(q, sb + bl - u)) : imax(0, imin(q, sb - u)));
      }
    }
    return u;
  };
  const int upr = (FR & 1) == 0 ? FR >> 1 : FR;  // stores per usage row: pairs of cells (16 B), single cells for odd FR
  auto publish_usage = [&](int h, int k) {       // store k of row h
    const int fr = (FR & 1) == 0 ? k << 1 : k, c = h * FR + fr;
    i64 *dst = D.usage + (size_t)b_gid[h] * FR + fr;
    if ((FR & 1) == 0) *(longlong2 *)dst = make_longlong2(final_usage(h, c), final_usage(h, c + 1));
    else *dst = final_usage(h, c);
  };
  const int nw = nthreads >> 5;
  if (warp == 0) {
    if (FR > 32) flat_ordered_loop<true>(n, FR, lane, s_lim, m_sorted, ok_bits, blk_bar, s_u, s_sub);
    else flat_ordered_loop<false>(n, FR, lane, s_lim, m_sorted, ok_bits, blk_bar, s_u, s_sub);
    KB_FPHASE(4);
    for (int c = lane; c < FR; c += 32) D.usage[(size_t)b_gid[0] * FR + c] = s_u[c];  // the root row (h = 0, no entry)
  } else if ((warp & 3) != 0) {  // off warp 0's scheduler (warp % 4): its compare -> vote -> add chain keeps the issue slots
    const int pw = warp - 1 - (warp >> 2), npw = nw - 1 - ((nw - 1) >> 2);  // publisher warp index / count
    const int pt = pw * 32 + lane, NP = npw * 32;
    // ---- 6a. what no decision changes
    for (int i = pt; i < n; i += NP) {
      const int e = e_gid[i];
      D.mode[e] = (uint8_t)e_mode[i]; D.borrow[e] = e_borrow[i]; D.rank[e] = e_rank[i];
      D.tgt_cnt[e] = 0; D.tgt_off[e] = 0;
    }
    if ((R & 3) == 0) {  // rows of R bytes are word aligned in both copies
      const int wpr = R >> 2;
      for (int c = pt; c < nrows * wpr; c += NP) {
        const int l = c / wpr, w = c % wpr;
        const size_t dst = (size_t)r_gid[l] * wpr + w, src = (size_t)l * wpr + w;
        ((uint32_t *)D.ps_flavor)[dst] = ((const uint32_t *)o_fl)[src];
        ((uint32_t *)D.ps_res_mode)[dst] = ((const uint32_t *)o_md)[src];
        ((uint32_t *)D.ps_tried)[dst] = ((const uint32_t *)o_tr)[src];
        if (w == 0) D.ps_count_out[r_gid[l]] = o_cnt[l];
      }
    } else {
      for (int l = pt; l < nrows; l += NP) {
        const int row = r_gid[l];
        D.ps_count_out[row] = o_cnt[l];
        for (int r = 0; r < R; r++) {
          D.ps_flavor[(size_t)row * R + r] = o_fl[(size_t)l * R + r];
          D.ps_res_mode[(size_t)row * R + r] = o_md[(size_t)l * R + r];
          D.ps_tried[(size_t)row * R + r] = o_tr[(size_t)l * R + r];
        }
      }
    }
    for (int k = upr + pt; k < nn * upr; k += NP) {  // ClusterQueue rows without an entry
      const int h = k / upr;
      if (n_e[h] < 0) publish_usage(h, k - h * upr);
    }
    // ---- 6b. per block of 32 positions, once the loop has passed it: decisions and ClusterQueue rows of its entries.
    // The publisher warps form min(warps, blocks) groups; group g takes blocks g, g + groups, ...
    const int nblk = (n + 31) >> 5, ng = min(npw, nblk), g = pw % ng;
    const int gi = (pw / ng) * 32 + lane, GT = ((npw - 1 - g) / ng + 1) * 32;
    for (int b = g; b < nblk; b += ng) {
      mbar_wait(blk_bar + b, 0);
      const int p0 = b << 5, np = min(32, n - p0);
      for (int k = gi; k < np; k += GT) { const int i = e_at[p0 + k]; D.decision[e_gid[i]] = (uint8_t)flat_decision(e_mode[i], ok_bits, p0 + k); }
      for (int k = gi; k < np * upr; k += GT) { const int p = k / upr, i = e_at[p0 + p]; publish_usage(e_cq[i], k - p * upr); }
    }
  }
  __syncthreads();
  KB_FPHASE(5);
#undef KB_FPHASE
}
