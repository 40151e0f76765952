// kb_api.cu — C-ABI of libkueue_b200 (include/kueue_b200.h): handle, snapshot upload
// (host -> HBM, plus the static topology tables the kernels need), cycle launch,
// result download.  One handle = one CUDA device + one stream; calls are blocking and
// not re-entrant per handle (SURVEY.md §8b threading row).
#include <algorithm>
#include <cstdio>
#include <cstring>
#include <string>
#include <chrono>
#include <vector>
#include <map>
#include <mutex>

#include "kb_kernels.cuh"

#define KB_VERSION 100

namespace {

inline size_t pad256(size_t b) { b = (b + 255) & ~(size_t)255; return b ? b : 256; }

// Grow-only device arena, 256 B aligned sub-allocations.  An arena without a base is a sizing pass: take() only
// counts bytes (returns nullptr), so one layout function run on it and then on the real arena describes a buffer once.
struct Arena {
  char *base = nullptr;
  size_t cap = 0, used = 0;
  void reset() { used = 0; }
  void release() {
    if (base) cudaFree(base);
    base = nullptr; cap = used = 0;
  }
  bool reserve(size_t bytes) {
    if (bytes <= cap) return true;
    release();
    size_t want = bytes + bytes / 4 + (1 << 20);
    if (cudaMalloc(&base, want) != cudaSuccess) return false;
    cap = want;
    return true;
  }
  template <typename T> T *take(size_t n) {
    T *p = base ? (T *)(base + used) : nullptr;
    used += pad256(n * sizeof(T));
    return p;
  }
  // layout(Arena &) takes every sub-allocation of a buffer: run once to size, once to carve this arena from the start
  template <typename F> bool carve(F &&layout) {
    Arena sizing;
    layout(sizing);
    if (!reserve(sizing.used)) return false;
    reset();
    layout(*this);
    return true;
  }
};

// Launch configuration of the preemption-target searches, and the scratch sizes the per-cycle arena takes for them
// (plan_search).  The classical-search fields keep their values through uploads that have no classical search.
struct SearchPlan {
  // fair-sharing search: single-warp CTAs on a private copy of the whole tree
  int search_grid = 1; bool search_smem = true; size_t search_smem_bytes = 0;
  // warp-cooperative classical search (k_search_cells / k_nominate_walk)
  int sa_wpb = 1, sa_grid = 1, sa_col_elems = 0, sa_codes = 0; size_t sa_smem = 0;
  int sb_wpb = 1, sb_grid = 1, sb_col_elems = 0; size_t sb_smem = 0;
  int sa_list_cap = 32, sb_list_cap = 32;
  bool sg_on = false; int sg_wpb = 1, sg_grid = 1, sg_ncap = 1; size_t sg_smem = 0;  // grouped form of k_search_cells
  // scratch: memo rows, per-warp columns and lists, fair-search state for G CTAs of acap admitted rows and ncap nodes
  size_t memo_items = 0, ws_warps = 1, ws_col_stride = 0, ws_list_total = 32, G = 1, acap = 1, ncap = 1;
};

}  // namespace

struct kb_handle {
  int device = 0;
  int sm_count = 0;
  cudaStream_t stream = nullptr;
  cudaEvent_t ev0 = nullptr, ev1 = nullptr, ev2 = nullptr, ev3 = nullptr, ev4 = nullptr, ev5 = nullptr;
  Arena arena;   // per-cycle scratch, outputs
  Arena iarena;  // per-cycle input tables (copied before the host-side checks finish)
  char *d_out_block = nullptr;  // result tables of the cycle in the canonical layout
  int32_t *d_tgt_start = nullptr, *d_tgt_adm = nullptr; uint8_t *d_tgt_reason = nullptr;  // preemption targets, CSR by entry
  bool tgt_csr = false;
  Arena sarena;  // static tables (quotas, policies, topology): kept while kb_snapshot.static_generation is unchanged
  int64_t static_gen = 0;
  int s_dims[6] = {-1, -1, -1, -1, -1, -1};
  DevSnap D{};
  bool uploaded = false;
  bool profile = false;
  cudaEvent_t kev[KB_N_KERNELS + 1] = {};
  int kev_id[KB_N_KERNELS + 1] = {};
  int kev_n = 0;
  std::string err;
  kb_stats stats{};
  uint32_t *host_words = nullptr;  // pinned scratch words; [32..63] = copy of the cycle header, [64..] kb_run_drain's
  const uint32_t *hdr_host = nullptr;  // where the last cycle's header landed (host_words or the caller's result block)
  int last_launches = 0;
  int64_t last_d2h_bytes = 0;
  // tree_eval scratch
  i64 *d_drs_rounded = nullptr; int32_t *d_drs_res = nullptr; uint8_t *d_drs_borrowing = nullptr;
  // host-side derived topology
  std::vector<int32_t> root_slot, depth, height, tree_start, tree_nodes, tree_level, lone, cq_adm_start, cq_adm, local_idx, child_start, child_list, adm_sorted, root_adm_start, adm_rank, root_cq_start;
  std::vector<uint8_t> tree_flat;
  // host copies of the static tables build_dynamic consults every cycle (the caller's static pointers are not read
  // again while static_generation is unchanged)
  std::vector<int32_t> s_parent; std::vector<uint8_t> s_within_cq, s_reclaim_within;
  std::vector<uint32_t> seen; uint32_t seen_stamp = 0;  // one-head-per-ClusterQueue check without clearing a table per cycle
  bool s_any_lone_within = false, s_preempt_policy = false;  // static: some cohort-less CQ has WithinClusterQueue != Never / some CQ has a preemption policy
  std::vector<int32_t> sn_node, slot_base, nd_tin, nd_tout, cq_path, cq_plen; int path_stride = 1;
  int max_root_adm = 1;
  int max_frl_len = 1;      // longest (root, flavor-resource) candidate bucket of this cycle
  int max_head_podsets = 1; // most podsets of one entry (bounds the columns a GetTargets search tracks)
  SearchPlan plan;
  // kb_run_drain: capacity reserved beyond the snapshot's admitted tables, heads chosen on the device
  size_t drain_extra_adm = 0, drain_extra_au = 0; bool drain_mode = false; bool preempt_possible = true;
  bool drain_events = false;  // kb_run_drain in event mode: rows admitted during the drain are preemption candidates
  size_t out_tgt_capacity = 0;  // kb_run_cycle: the caller's target buffer, a lower bound of the device target pool
  Arena drain_arena; cudaEvent_t ev_d = nullptr;  // kb_run_drain's queue tables, double buffer and scratch
  Arena tas_arena;  // kb_tas_find's inputs, lists and outputs
  bool fused_on = false; size_t fused_smem = 0; bool one_head_per_cq = false; int32_t *d_cq_entry = nullptr;
  // k_cycle_flat (kb_flat.cuh): static per-tree blocks in local numbering, head records per tree node
  std::vector<unsigned char> tree_blob; std::vector<int32_t> tree_blob_off; int max_blob_bytes = 16;
  // incremental usage (kb_snapshot.usage_delta_*): the ClusterQueue usage table kept between calls
  i64 *d_usage_res = nullptr; size_t usage_res_cells = 0; bool usage_res_valid = false; int64_t usage_res_gen = 0;
  std::vector<uint32_t> delta_seen; uint32_t delta_stamp = 0;
  bool flat_on = false, flat_attr_set = false, hdr_clean = false; size_t flat_static_smem = 0; unsigned rec_stamp = 0; const void *rec_seen = nullptr; size_t rec_seen_n = 0; size_t flat_smem = 0; int flat_rcap = 1; int4 *d_cq_rec = nullptr;
  // device ranking of the admitted workloads (kb_rank.cuh)
  u64 *rk_keys[2] = {nullptr, nullptr}; int32_t *rk_vals[2] = {nullptr, nullptr}; void *rk_temp = nullptr; size_t rk_temp_bytes = 0;
  int max_tree_nodes = 1;
  int max_root_entries_hint = 0;
};

static thread_local std::string g_err;

static int32_t fail(kb_handle *h, int32_t code, const std::string &msg) {
  if (h) h->err = msg; else g_err = msg;
  return code;
}
#define CUDA_TRY(h, expr)                                                                           \
  do {                                                                                              \
    cudaError_t _e = (expr);                                                                        \
    if (_e != cudaSuccess) return fail(h, KB_ERR_CUDA, std::string(#expr) + ": " + cudaGetErrorString(_e)); \
  } while (0)

extern "C" {

int32_t kb_version(void) { return KB_VERSION; }

const char *kb_last_error(const kb_handle *h) { return h ? h->err.c_str() : g_err.c_str(); }

// blocks handed out by kb_alloc_pinned: a span upload only ever reads inside ONE of them
static std::mutex g_pin_mu;
static std::map<uintptr_t, size_t> g_pinned;
static bool inside_one_pinned_block(uintptr_t lo, uintptr_t hi) {
  std::lock_guard<std::mutex> lk(g_pin_mu);
  auto it = g_pinned.upper_bound(lo);
  if (it == g_pinned.begin()) return false;
  --it;
  return lo >= it->first && hi <= it->first + it->second;
}

// Canonical layout of the eight per-entry / per-podset output tables: the device block of every cycle and the host
// block of kb_alloc_cycle_out use the same offsets, so those results come back with ONE device-to-host DMA.
// The block ends with the 128-byte cycle header (status word, counters), so that it too needs no copy of its own.
struct OutLayout { size_t off[8]; size_t hdr; size_t prefix; };
static OutLayout out_layout(size_t H, size_t P, size_t R) {
  const size_t sz[8] = {H, H, 4 * H, 4 * H, P * R, P * R, P * R, 4 * P};  // decision mode borrow rank flavor res_mode tried count
  OutLayout L; size_t o = 0;
  for (int i = 0; i < 8; i++) { L.off[i] = o; o += pad256(sz[i]); }
  L.hdr = o; o += 256;
  L.prefix = o;
  return L;
}
struct OutBlock { size_t H, P, R; };
static std::map<uintptr_t, OutBlock> g_out_blocks;  // base of a kb_alloc_cycle_out block -> its dimensions

int32_t kb_alloc_cycle_out(int32_t n_heads, int32_t n_podset, int32_t n_resource, int32_t tgt_capacity, int64_t n_node_cells, kb_cycle_out *out) {
  if (!out || n_heads < 0 || n_podset < 0 || n_resource < 0 || tgt_capacity < 0 || n_node_cells < 0) return KB_ERR_INVALID;
  const size_t H = (size_t)n_heads, P = (size_t)n_podset, R = (size_t)n_resource, cap = (size_t)tgt_capacity;
  OutLayout L = out_layout(H, P, R);
  size_t o_ts = L.prefix, o_ta = o_ts + pad256(4 * (H + 1)), o_tr = o_ta + pad256(4 * cap), o_nu = o_tr + pad256(cap);
  size_t total = o_nu + pad256(8 * (size_t)n_node_cells);
  void *base = nullptr;
  int32_t rc = kb_alloc_pinned(&base, total);
  if (rc != KB_OK) return rc;
  memset(base, 0, total);
  char *b = (char *)base;
  out->decision = (uint8_t *)(b + L.off[0]); out->mode = (uint8_t *)(b + L.off[1]);
  out->borrow = (int32_t *)(b + L.off[2]); out->commit_rank = (int32_t *)(b + L.off[3]);
  out->ps_flavor = (int8_t *)(b + L.off[4]); out->ps_res_mode = (int8_t *)(b + L.off[5]); out->ps_tried_idx = (int8_t *)(b + L.off[6]);
  out->ps_count = (int32_t *)(b + L.off[7]);
  out->tgt_start = (int32_t *)(b + o_ts); out->tgt_adm = (int32_t *)(b + o_ta); out->tgt_reason = (uint8_t *)(b + o_tr);
  out->tgt_capacity = tgt_capacity; out->n_targets = 0;
  out->node_usage = n_node_cells ? (int64_t *)(b + o_nu) : nullptr;
  std::lock_guard<std::mutex> lk(g_pin_mu);
  g_out_blocks[(uintptr_t)base] = OutBlock{H, P, R};
  return KB_OK;
}

int32_t kb_alloc_pinned(void **ptr, uint64_t bytes) {
  if (!ptr) return KB_ERR_INVALID;
  cudaError_t e = cudaHostAlloc(ptr, bytes ? bytes : 1, cudaHostAllocDefault);
  if (e != cudaSuccess) { g_err = cudaGetErrorString(e); return KB_ERR_CUDA; }
  std::lock_guard<std::mutex> lk(g_pin_mu);
  g_pinned[(uintptr_t)*ptr] = bytes ? bytes : 1;
  return KB_OK;
}
int32_t kb_free_pinned(void *ptr) {
  if (!ptr) return KB_OK;
  { std::lock_guard<std::mutex> lk(g_pin_mu); g_pinned.erase((uintptr_t)ptr); g_out_blocks.erase((uintptr_t)ptr); }
  return cudaFreeHost(ptr) == cudaSuccess ? KB_OK : KB_ERR_CUDA;
}

int32_t kb_create(const kb_config *cfg, kb_handle **out) {
  if (!out) return KB_ERR_INVALID;
  *out = nullptr;
  int ndev = 0;
  if (cudaGetDeviceCount(&ndev) != cudaSuccess || ndev == 0) return fail(nullptr, KB_ERR_NO_DEVICE, "no CUDA device");
  int dev = cfg ? cfg->device : 0;
  if (dev < 0 || dev >= ndev) return fail(nullptr, KB_ERR_INVALID, "bad device ordinal");
  kb_handle *h = new kb_handle();
  h->device = dev;
  if (cudaSetDevice(dev) != cudaSuccess) { delete h; return fail(nullptr, KB_ERR_CUDA, "cudaSetDevice failed"); }
  cudaDeviceGetAttribute(&h->sm_count, cudaDevAttrMultiProcessorCount, dev);
  if (cudaStreamCreateWithFlags(&h->stream, cudaStreamNonBlocking) != cudaSuccess) { delete h; return fail(nullptr, KB_ERR_CUDA, "stream"); }
  cudaEventCreate(&h->ev0); cudaEventCreate(&h->ev1); cudaEventCreate(&h->ev2); cudaEventCreate(&h->ev3); cudaEventCreate(&h->ev4); cudaEventCreate(&h->ev5);
  for (int i = 0; i <= KB_N_KERNELS; i++) cudaEventCreate(&h->kev[i]);
  cudaHostAlloc((void **)&h->host_words, 512, cudaHostAllocDefault);
  h->stats.sm_count = h->sm_count;
  *out = h;
  return KB_OK;
}

void kb_destroy(kb_handle *h) {
  if (!h) return;
  cudaSetDevice(h->device);
  for (Arena *a : {&h->arena, &h->sarena, &h->iarena, &h->drain_arena, &h->tas_arena}) a->release();
  if (h->d_usage_res) cudaFree(h->d_usage_res);
  if (h->ev_d) cudaEventDestroy(h->ev_d);
  if (h->host_words) cudaFreeHost(h->host_words);
  if (h->stream) cudaStreamDestroy(h->stream);
  if (h->ev0) cudaEventDestroy(h->ev0);
  if (h->ev1) cudaEventDestroy(h->ev1);
  if (h->ev2) cudaEventDestroy(h->ev2);
  if (h->ev3) cudaEventDestroy(h->ev3);
  if (h->ev4) cudaEventDestroy(h->ev4);
  if (h->ev5) cudaEventDestroy(h->ev5);
  for (int i = 0; i <= KB_N_KERNELS; i++) if (h->kev[i]) cudaEventDestroy(h->kev[i]);
  delete h;
}

}  // extern "C"

// ---------------------------------------------------------------------------
// validation + static topology
// ---------------------------------------------------------------------------
// static part: validation of the node tables + everything derived from the cohort forest alone
static int32_t build_static(kb_handle *h, const kb_snapshot *s) {
  int Q = s->n_cq, C = s->n_cohort, N = Q + C;
  if (Q < 0 || C < 0 || s->n_flavor < 1 || s->n_flavor > KB_MAX_FLAVORS || s->n_resource < 1 ||
      s->n_resource > KB_MAX_RESOURCES || s->n_wl < 0 || s->n_podset < 0 || s->n_adm < 0 || s->n_heads < 0)
    return fail(h, KB_ERR_INVALID, "bad dimensions");
  if (s->n_flavor > 127) return fail(h, KB_ERR_INVALID, "flavor index must fit int8");
  if (s->n_rg < 0 || s->pods_resource < -1 || s->pods_resource >= s->n_resource) return fail(h, KB_ERR_INVALID, "bad n_rg / pods_resource");
  // resource-group CSR tables (resource.go:31-38): monotone, in range, flavor indexes < F
  if (Q > 0) {
    if (s->cq_rg_start[0] != 0 || s->cq_rg_start[Q] != s->n_rg) return fail(h, KB_ERR_INVALID, "cq_rg_start must run from 0 to n_rg");
    for (int q = 0; q < Q; q++) if (s->cq_rg_start[q + 1] < s->cq_rg_start[q]) return fail(h, KB_ERR_INVALID, "cq_rg_start not monotone");
  }
  if (s->n_rg > 0) {
    if (s->rg_flavor_start[0] != 0) return fail(h, KB_ERR_INVALID, "rg_flavor_start[0] != 0");
    for (int g = 0; g < s->n_rg; g++) if (s->rg_flavor_start[g + 1] < s->rg_flavor_start[g]) return fail(h, KB_ERR_INVALID, "rg_flavor_start not monotone");
    for (int k = 0; k < s->rg_flavor_start[s->n_rg]; k++)
      if (s->rg_flavors[k] < 0 || s->rg_flavors[k] >= s->n_flavor) return fail(h, KB_ERR_INVALID, "rg_flavors out of range");
  }
  for (int n = 0; n < N; n++) {
    int p = s->parent[n];
    if (p != -1 && (p < Q || p >= N)) return fail(h, KB_ERR_INVALID, "parent must be a cohort node or -1");
  }
  h->depth.assign(N, -1);
  h->root_slot.assign(N, -1);
  std::vector<int32_t> root(N, -1);
  for (int n = 0; n < N; n++) {  // depth + root with cycle detection (hierarchy/cycle.go:31-44)
    int steps = 0, t = n;
    while (s->parent[t] >= 0) {
      t = s->parent[t];
      if (++steps > KB_MAX_DEPTH) return fail(h, KB_ERR_INVALID, "cohort tree deeper than KB_MAX_DEPTH or cyclic");
    }
    h->depth[n] = steps;
    root[n] = t;
  }
  // roots: every parentless node; slots in ascending node order
  int nroots = 0;
  std::vector<int32_t> slot_of_root(N, -1);
  for (int n = 0; n < N; n++) if (s->parent[n] < 0) slot_of_root[n] = nroots++;
  for (int n = 0; n < N; n++) h->root_slot[n] = slot_of_root[root[n]];
  // children counts -> height (getNodeHeight hierarchical_preemption.go:202-208)
  std::vector<int32_t> nchild(N, 0);
  for (int n = 0; n < N; n++) if (s->parent[n] >= 0) nchild[s->parent[n]]++;
  h->height.assign(N, 0);
  for (int n = Q; n < N; n++) h->height[n] = std::min(nchild[n], 1);
  {  // process cohorts by depth descending so children are final before parents
    std::vector<int32_t> order;
    for (int n = Q; n < N; n++) order.push_back(n);
    std::stable_sort(order.begin(), order.end(), [&](int a, int b) { return h->depth[a] > h->depth[b]; });
    for (int n : order) {
      int p = s->parent[n];
      if (p >= 0) h->height[p] = std::max(h->height[p], h->height[n] + 1);
    }
  }
  // cohort-rooted trees: nodes grouped by root, ordered by depth ascending
  std::vector<int32_t> tree_of_root(N, -1);
  int ntrees = 0;
  for (int n = Q; n < N; n++) if (s->parent[n] < 0) tree_of_root[n] = ntrees++;
  std::vector<int32_t> cnt(ntrees + 1, 0);
  h->lone.clear();
  for (int n = 0; n < N; n++) {
    int t = tree_of_root[root[n]];
    if (t >= 0) cnt[t + 1]++;
    else h->lone.push_back(n);  // parentless CQ
  }
  for (int t = 0; t < ntrees; t++) cnt[t + 1] += cnt[t];
  h->tree_start.assign(cnt.begin(), cnt.end());
  h->tree_nodes.assign(cnt[ntrees], 0);
  h->tree_level.assign((size_t)ntrees * KB_LEVELS, 0);
  {
    // counting sort by (tree, depth)
    std::vector<int32_t> lvlcnt((size_t)ntrees * KB_LEVELS, 0);
    for (int n = 0; n < N; n++) { int t = tree_of_root[root[n]]; if (t >= 0) lvlcnt[(size_t)t * KB_LEVELS + h->depth[n] + 1]++; }
    for (int t = 0; t < ntrees; t++)
      for (int l = 0; l + 1 < KB_LEVELS; l++) lvlcnt[(size_t)t * KB_LEVELS + l + 1] += lvlcnt[(size_t)t * KB_LEVELS + l];
    h->tree_level = lvlcnt;
    std::vector<int32_t> cur = lvlcnt;
    for (int n = 0; n < N; n++) {
      int t = tree_of_root[root[n]];
      if (t < 0) continue;
      int pos = cur[(size_t)t * KB_LEVELS + h->depth[n]]++;
      h->tree_nodes[h->tree_start[t] + pos] = n;
    }
  }
  // children CSR (cohort children first: their node ids are >= Q, so sort descending by class)
  h->child_start.assign(N + 1, 0);
  for (int n = 0; n < N; n++) if (s->parent[n] >= 0) h->child_start[s->parent[n] + 1]++;
  for (int n = 0; n < N; n++) h->child_start[n + 1] += h->child_start[n];
  h->child_list.assign(std::max(1, h->child_start[N]), 0);
  {
    std::vector<int32_t> cur(h->child_start.begin(), h->child_start.end() - 1);
    for (int n = Q; n < N; n++) if (s->parent[n] >= 0) h->child_list[cur[s->parent[n]]++] = n;  // cohorts ascending
    for (int n = 0; n < Q; n++) if (s->parent[n] >= 0) h->child_list[cur[s->parent[n]]++] = n;  // then CQs ascending
  }
  h->tree_flat.assign(std::max(1, ntrees), 1);
  for (int n = 0; n < Q; n++) { int t = tree_of_root[root[n]]; if (t >= 0 && h->depth[n] != 1) h->tree_flat[t] = 0; }
  h->local_idx.assign(N, 0);
  h->max_tree_nodes = 1;
  for (int t = 0; t < ntrees; t++) {
    int nn = h->tree_start[t + 1] - h->tree_start[t];
    h->max_tree_nodes = std::max(h->max_tree_nodes, nn);
    for (int i = 0; i < nn; i++) h->local_idx[h->tree_nodes[h->tree_start[t] + i]] = i;
  }
  h->root_cq_start.assign(nroots + 1, 0);
  for (int q = 0; q < Q; q++) h->root_cq_start[h->root_slot[q] + 1]++;
  for (int r = 0; r < nroots; r++) h->root_cq_start[r + 1] += h->root_cq_start[r];
  h->D.nTrees = ntrees;
  h->D.nLone = (int)h->lone.size();
  h->D.nRoots = nroots;
  {  // static ClusterQueue -> root paths (global-table admit loop)
    int maxd = 0;
    for (int q = 0; q < Q; q++) maxd = std::max(maxd, h->depth[q]);
    h->path_stride = maxd + 1;
    h->cq_path.assign((size_t)std::max(1, Q) * h->path_stride, -1); h->cq_plen.assign(std::max(1, Q), 1);
    for (int q = 0; q < Q; q++) { int k = 0; for (int t = q; t >= 0; t = s->parent[t]) h->cq_path[(size_t)q * h->path_stride + k++] = t; h->cq_plen[q] = k; }
  }
  h->s_parent.assign(s->parent, s->parent + N);
  h->s_within_cq.assign(s->cq_within_cq, s->cq_within_cq + Q);
  h->s_reclaim_within.assign(s->cq_reclaim_within, s->cq_reclaim_within + Q);
  h->s_any_lone_within = false; h->s_preempt_policy = false;
  for (int q = 0; q < Q; q++) {
    if (s->parent[q] < 0 && s->cq_within_cq[q] != KB_POLICY_NEVER) h->s_any_lone_within = true;
    if (s->cq_within_cq[q] != KB_POLICY_NEVER || (s->parent[q] >= 0 && s->cq_reclaim_within[q] != KB_POLICY_NEVER)) h->s_preempt_policy = true;
  }
  {  // slot-node numbering (cohort-less ClusterQueues, then the trees) and Euler-tour intervals inside every tree
    int nl = (int)h->lone.size();
    h->sn_node.assign(std::max(1, N), 0); h->nd_tin.assign(std::max(1, N), 0); h->nd_tout.assign(std::max(1, N), 1);
    h->slot_base.assign(nroots + 1, 0);
    for (int i = 0; i < nl; i++) { h->sn_node[i] = h->lone[i]; h->slot_base[i] = i; }
    for (int t = 0; t < ntrees; t++) h->slot_base[nl + t] = nl + h->tree_start[t];
    h->slot_base[nroots] = N;
    for (size_t i = 0; i < h->tree_nodes.size(); i++) h->sn_node[nl + i] = h->tree_nodes[i];
    std::vector<int32_t> stack, it;
    for (int t = 0; t < ntrees; t++) {
      int base = nl + h->tree_start[t];
      int rootn = h->tree_nodes[h->tree_start[t]];
      int clock = 0;
      stack.assign(1, rootn); it.assign(1, h->child_start[rootn]);
      h->nd_tin[base + h->local_idx[rootn]] = clock++;
      while (!stack.empty()) {
        int n = stack.back();
        if (it.back() < h->child_start[n + 1]) {
          int c = h->child_list[it.back()++];
          h->nd_tin[base + h->local_idx[c]] = clock++;
          stack.push_back(c); it.push_back(h->child_start[c]);
        } else {
          h->nd_tout[base + h->local_idx[n]] = clock;
          stack.pop_back(); it.pop_back();
        }
      }
    }
  }
  {  // static per-tree blocks in local numbering (TreeBlobHdr, kb_flat.cuh)
    h->tree_blob.clear(); h->tree_blob_off.assign(ntrees + 1, 0); h->max_blob_bytes = 16;
    for (int t = 0; t < ntrees; t++) {
      const int nn = h->tree_start[t + 1] - h->tree_start[t];
      const int32_t *nodes = h->tree_nodes.data() + h->tree_start[t];
      int nrg = 0, nfl = 0;
      for (int i = 0; i < nn; i++) if (nodes[i] < Q) for (int g = s->cq_rg_start[nodes[i]]; g < s->cq_rg_start[nodes[i] + 1]; g++) { nrg++; nfl += s->rg_flavor_start[g + 1] - s->rg_flavor_start[g]; }
      TreeBlobHdr H{};
      size_t o = sizeof(TreeBlobHdr);
      auto take = [&](size_t bytes) { o = (o + 15) & ~(size_t)15; size_t at = o; o += bytes; return (int32_t)at; };
      H.nn = nn; H.nrg = nrg; H.nfl = nfl;
      H.gid = take((size_t)nn * 4); H.par = take((size_t)nn * 4); H.hgt = take((size_t)nn * 4); H.rgs = take((size_t)(nn + 1) * 4);
      H.gen = take((size_t)nn * 8); H.wgt = take((size_t)nn * 8);
      H.within = take(nn); H.reclaim = take(nn); H.borrow_w = take(nn); H.wcb = take(nn); H.wcp = take(nn); H.pref = take(nn);
      H.rgmask = take((size_t)nrg * 4); H.rgfl = take((size_t)(nrg + 1) * 4); H.fl = take((size_t)nfl * 4);
      o = (o + 15) & ~(size_t)15;
      H.bytes = (int32_t)o;
      size_t base = h->tree_blob.size();
      if (base + o >= (size_t)INT32_MAX) return fail(h, KB_ERR_INVALID, "static tree tables exceed 2 GiB");
      h->tree_blob.resize(base + o, 0);
      unsigned char *b = h->tree_blob.data() + base;
      memcpy(b, &H, sizeof(H));
      int32_t *gid = (int32_t *)(b + H.gid), *par = (int32_t *)(b + H.par), *hgt = (int32_t *)(b + H.hgt), *rgs = (int32_t *)(b + H.rgs);
      i64 *gen = (i64 *)(b + H.gen); double *wgt = (double *)(b + H.wgt);
      uint32_t *rgmask = (uint32_t *)(b + H.rgmask); int32_t *rgfl = (int32_t *)(b + H.rgfl), *fl = (int32_t *)(b + H.fl);
      int lg = 0, lf = 0;
      for (int i = 0; i < nn; i++) {
        const int nd = nodes[i];
        gid[i] = nd; par[i] = s->parent[nd] < 0 ? -1 : h->local_idx[s->parent[nd]]; hgt[i] = h->height[nd]; rgs[i] = lg;
        wgt[i] = s->fair_weight[nd];
        if (nd >= Q) continue;
        gen[i] = s->cq_generation[nd];
        b[H.within + i] = s->cq_within_cq[nd]; b[H.reclaim + i] = s->cq_reclaim_within[nd]; b[H.borrow_w + i] = s->cq_borrow_within[nd];
        b[H.wcb + i] = s->cq_when_can_borrow[nd]; b[H.wcp + i] = s->cq_when_can_preempt[nd]; b[H.pref + i] = s->cq_preference[nd];
        for (int g = s->cq_rg_start[nd]; g < s->cq_rg_start[nd + 1]; g++) {
          rgmask[lg] = s->rg_res_mask[g]; rgfl[lg] = lf;
          for (int k = s->rg_flavor_start[g]; k < s->rg_flavor_start[g + 1]; k++) fl[lf++] = s->rg_flavors[k];
          lg++;
        }
      }
      rgs[nn] = lg; rgfl[lg] = lf;
      h->tree_blob_off[t + 1] = (int32_t)(base + o);
      h->max_blob_bytes = std::max(h->max_blob_bytes, (int)o);
    }
    if (h->tree_blob.empty()) h->tree_blob.resize(16, 0);
  }
  return KB_OK;
}

// per-cycle part: admitted workloads (grouping, candidate pre-order) and bounds checks of the entry tables
static int32_t build_dynamic(kb_handle *h, const kb_snapshot *s) {
  int Q = s->n_cq;
  int nroots = h->D.nRoots;
  if (s->n_wl < 0 || s->n_podset < 0 || s->n_adm < 0 || s->n_heads < 0) return fail(h, KB_ERR_INVALID, "bad dimensions");
  // admitted workloads grouped by CQ (ClusterQueueSnapshot.Workloads)
  h->cq_adm_start.assign(Q + 1, 0);
  for (int a = 0; a < s->n_adm; a++) {
    int c = s->adm_cq[a];
    if (c < 0 || c >= Q) return fail(h, KB_ERR_INVALID, "adm_cq out of range");
    h->cq_adm_start[c + 1]++;
  }
  for (int q = 0; q < Q; q++) h->cq_adm_start[q + 1] += h->cq_adm_start[q];
  // admitted workloads per root: only the counts are needed on the host (scratch sizing); the ranking by the
  // preemptor-independent part of CandidatesOrdering runs on the device every cycle (kb_rank.cuh)
  h->root_adm_start.assign(nroots + 1, 0);
  for (int a = 0; a < s->n_adm; a++) h->root_adm_start[h->root_slot[s->adm_cq[a]] + 1]++;
  h->max_root_adm = 1;
  for (int r = 0; r < nroots; r++) { h->max_root_adm = std::max(h->max_root_adm, h->root_adm_start[r + 1]); h->root_adm_start[r + 1] += h->root_adm_start[r]; }
  h->max_root_adm += (int)h->drain_extra_adm;  // a drain may admit everything into one root
  if (h->max_root_adm >= (1 << 28)) return fail(h, KB_ERR_INVALID, "more than 2^28 admitted workloads under one root");
  {  // longest (root, flavor-resource) bucket: sizes the per-warp candidate-code scratch of the single-cell searches
    int FRn = s->n_flavor * s->n_resource;
    std::vector<int32_t> cnt((size_t)nroots * FRn + 1, 0);
    for (int a = 0; a < s->n_adm; a++) {
      if (s->adm_use_start[a + 1] < s->adm_use_start[a]) return fail(h, KB_ERR_INVALID, "adm_use_start not monotone");
      size_t b = (size_t)h->root_slot[s->adm_cq[a]] * FRn;
      for (int k = s->adm_use_start[a]; k < s->adm_use_start[a + 1]; k++) {
        int fr = s->adm_use_fr[k];
        if (fr < 0 || fr >= FRn) return fail(h, KB_ERR_INVALID, "adm_use_fr out of range");
        cnt[b + fr]++;
      }
    }
    h->max_frl_len = 1;
    for (int32_t c : cnt) h->max_frl_len = std::max(h->max_frl_len, c);
    h->max_frl_len += (int)h->drain_extra_adm;
    h->max_head_podsets = 1;
    if (h->drain_mode) for (int w = 0; w < s->n_wl; w++) h->max_head_podsets = std::max(h->max_head_podsets, s->wl_ps_start[w + 1] - s->wl_ps_start[w]);
  }
  // light bounds checks on the hot tables
  for (int w = 0; w < s->n_wl; w++) {
    if (s->wl_cq[w] < 0 || s->wl_cq[w] >= Q) return fail(h, KB_ERR_INVALID, "wl_cq out of range");
    if (s->wl_ps_start[w + 1] < s->wl_ps_start[w]) return fail(h, KB_ERR_INVALID, "wl_ps_start not monotone");
    if (s->wl_ps_start[w + 1] - s->wl_ps_start[w] > KB_MAX_WL_PODSETS) return fail(h, KB_ERR_INVALID, "a workload with more than KB_MAX_WL_PODSETS podsets");
  }
  if (s->n_wl && (s->wl_ps_start[0] != 0 || s->wl_ps_start[s->n_wl] != s->n_podset)) return fail(h, KB_ERR_INVALID, "wl_ps_start must run from 0 to n_podset");
  // heads: range, most podsets of one entry, one head per ClusterQueue? (fairSharingIterator keeps one entry per CQ,
  // fair_sharing_iterator.go:52-54) — one pass
  h->one_head_per_cq = true;
  if (!h->drain_mode) {
    h->seen_stamp++;
    if ((int)h->seen.size() < Q || h->seen_stamp == 0) { h->seen.assign((size_t)std::max(1, Q), 0); h->seen_stamp = 1; }
    const uint32_t stamp = h->seen_stamp;
    int maxps = 1; bool dup = false;
    for (int i = 0; i < s->n_heads; i++) {
      const int w = s->heads[i];
      if (w < 0 || w >= s->n_wl) return fail(h, KB_ERR_INVALID, "heads out of range");
      maxps = std::max(maxps, s->wl_ps_start[w + 1] - s->wl_ps_start[w]);
      const int c = s->wl_cq[w];
      if (h->seen[c] == stamp) dup = true;
      h->seen[c] = stamp;
    }
    h->max_head_podsets = std::max(h->max_head_podsets, maxps);
    if (dup) {
      if (s->flags & KB_F_FAIR_SHARING) return fail(h, KB_ERR_INVALID, "fair sharing: more than one head for a ClusterQueue");
      h->one_head_per_cq = false;
    }
  }
  if (s->n_adm_use < 0 || (s->n_adm && (s->adm_use_start[0] != 0 || s->adm_use_start[s->n_adm] != s->n_adm_use)))
    return fail(h, KB_ERR_INVALID, "adm_use_start must run from 0 to n_adm_use");
  {  // ps_last_tried >= -1 (int8): eight at a time — a byte below -1 has its top bit set and is not 0xff
    const size_t nb = (size_t)s->n_podset * s->n_resource;
    const int8_t *lt = s->ps_last_tried;
    size_t i = 0;
    bool bad = false;
    for (; i + 8 <= nb; i += 8) {
      uint64_t v; memcpy(&v, lt + i, 8);
      const uint64_t top = v & 0x8080808080808080ull;         // bytes that are negative
      if (top) { for (int k = 0; k < 8; k++) if (lt[i + k] < -1) bad = true; }
    }
    for (; i < nb; i++) if (lt[i] < -1) bad = true;
    if (bad) return fail(h, KB_ERR_INVALID, "ps_last_tried below -1");
  }
  if (s->ps_group)  // the podsets of one PodSetGroup are adjacent rows of their workload
    for (int w = 0; w < s->n_wl; w++)
      for (int a = s->wl_ps_start[w]; a < s->wl_ps_start[w + 1]; a++) {
        int g = s->ps_group[a];
        if (g < 0 || (a > s->wl_ps_start[w] && s->ps_group[a - 1] == g)) continue;
        int b = a + 1;
        while (b < s->wl_ps_start[w + 1] && s->ps_group[b] == g) b++;
        for (int c = b; c < s->wl_ps_start[w + 1]; c++)
          if (s->ps_group[c] == g) return fail(h, KB_ERR_INVALID, "ps_group: podsets of one group must be adjacent");
      }
  // warp-per-root admit for cohort-less CQs: only when none of them can ever get preemption targets
  {
    bool any = false;
    if (h->s_any_lone_within) {
      for (int q = 0; q < Q && !any; q++)
        if (h->s_parent[q] < 0 && h->s_within_cq[q] != KB_POLICY_NEVER && h->cq_adm_start[q + 1] > h->cq_adm_start[q]) any = true;
      if (h->drain_mode) any = true;  // admitted workloads appear during the drain
    }
    h->D.lone_fast = !any && s->n_flavor * s->n_resource <= 64;
    // can any ClusterQueue ever have preemption candidates?  (candidates_possible, kb_kernels.cuh)
    h->preempt_possible = h->s_preempt_policy;
  }
  if (s->wl_lq) {  // AdmissionFairSharing tables (include/kueue_b200.h)
    const int L = s->n_lq;
    if (L < 0 || !s->lq_cq || !s->cq_afs || !s->lq_weight || !s->lq_consumed || !s->lq_consumed_scale || !s->afs_res_weight || !s->afs_milli_mul)
      return fail(h, KB_ERR_INVALID, "afs: wl_lq given without the LocalQueue tables");
    for (int l = 0; l < L; l++) {
      if (s->lq_cq[l] < 0 || s->lq_cq[l] >= Q) return fail(h, KB_ERR_INVALID, "afs: lq_cq out of range");
      if (l && s->lq_cq[l] < s->lq_cq[l - 1]) return fail(h, KB_ERR_INVALID, "afs: LocalQueues must be numbered ClusterQueue-major");
    }
    for (int w = 0; w < s->n_wl; w++) {
      const int l = s->wl_lq[w];
      if (l < 0 || l >= L) return fail(h, KB_ERR_INVALID, "afs: wl_lq out of range");
      if (s->lq_cq[l] != s->wl_cq[w]) return fail(h, KB_ERR_INVALID, "afs: the LocalQueue of a workload feeds another ClusterQueue");
    }
    for (int r = 0; r < s->n_resource; r++)
      if (s->afs_milli_mul[r] < 1) return fail(h, KB_ERR_INVALID, "afs: afs_milli_mul must be positive");
    for (size_t i = 0; i < (size_t)L * s->n_resource; i++)
      if (s->lq_consumed_scale[i] < -AFS_MAX_SCALE || s->lq_consumed_scale[i] > AFS_MAX_SCALE)
        return fail(h, KB_ERR_UNSUPPORTED, "afs: consumed quantity scale outside [-22, 22]");
    bool any_afs = false;
    for (int q = 0; q < Q; q++) any_afs |= s->cq_afs[q] != 0;
    if (any_afs && h->preempt_possible)
      return fail(h, KB_ERR_UNSUPPORTED, "afs: preemption candidate ordering with AdmissionFairSharing is not supported (not a transitive order across ClusterQueues)");
  }
  return KB_OK;
}

// next stamp of the head records (kb_flat.cuh); the table is cleared when it moved, grew or the 16-bit stamp wrapped
static int32_t flat_rec_stamp(kb_handle *h) {
  const size_t n = h->tree_nodes.size() + 1;
  if (h->rec_seen != (const void *)h->d_cq_rec || h->rec_seen_n != n || h->rec_stamp >= 0xffffu) {
    CUDA_TRY(h, cudaMemsetAsync(h->d_cq_rec, 0, sizeof(int4) * n, h->stream));
    h->rec_seen = h->d_cq_rec; h->rec_seen_n = n; h->rec_stamp = 0;
  }
  h->D.rec_stamp = ++h->rec_stamp;
  return KB_OK;
}

// rows of the resident usage table replaced by the caller's deltas (kb_snapshot.usage_delta_*)
__global__ void k_usage_patch(i64 *usage, const int32_t *cq, const i64 *rows, int n, int FR) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n * FR) return;
  usage[(size_t)cq[i / FR] * FR + i % FR] = rows[i];
}

// host -> device on the handle's stream; an empty table copies nothing
static cudaError_t h2d(kb_handle *h, const void *dst, const void *src, size_t bytes) {
  return bytes ? cudaMemcpyAsync(const_cast<void *>(dst), src, bytes, cudaMemcpyHostToDevice, h->stream) : cudaSuccess;
}

// One table of an upload: host source, bytes to copy, the DevSnap pointer that receives its device address, and the
// device bytes it needs (more than it copies for the admitted tables kb_run_drain grows on the device).
struct HostTab { const void *src; size_t bytes; const void **dst; size_t cap; };
#define UPC(field, src, n, capn) tabs.push_back(HostTab{(const void *)(src), (size_t)(n) * sizeof(*D.field), (const void **)&D.field, (size_t)(capn) * sizeof(*D.field)})
#define UP(field, src, n) UPC(field, src, n, n)

// Static tables (quotas, policies, topology), and the tree-local quota tables k_tl_static / k_tl_root derive from them
static int32_t upload_static(kb_handle *h, const kb_snapshot *s, int n_rg_fl, int64_t *bytes) {
  int32_t rc = build_static(h, s);
  if (rc != KB_OK) return rc;
  DevSnap &D = h->D;
  const int Q = s->n_cq, N = Q + s->n_cohort, FR = s->n_flavor * s->n_resource;
  const size_t NF = (size_t)N * FR;
  std::vector<HostTab> tabs;
  UP(parent, s->parent, N); UP(fair_weight, s->fair_weight, N);
  UP(nominal, (const i64 *)s->nominal, NF); UP(blimit, (const i64 *)s->borrow_limit, NF); UP(llimit, (const i64 *)s->lend_limit, NF);
  UP(cq_within_cq, s->cq_within_cq, Q); UP(cq_reclaim_within, s->cq_reclaim_within, Q); UP(cq_borrow_within, s->cq_borrow_within, Q);
  UP(cq_has_bwc_threshold, s->cq_has_bwc_threshold, Q); UP(cq_bwc_threshold, s->cq_bwc_threshold, Q);
  UP(cq_when_can_borrow, s->cq_when_can_borrow, Q); UP(cq_when_can_preempt, s->cq_when_can_preempt, Q);
  UP(cq_preference, s->cq_preference, Q); UP(cq_strategy, s->cq_strategy, Q); UP(cq_generation, (const i64 *)s->cq_generation, Q);
  UP(cq_rg_start, s->cq_rg_start, Q + 1); UP(rg_res_mask, s->rg_res_mask, s->n_rg); UP(rg_flavor_start, s->rg_flavor_start, s->n_rg + 1);
  UP(rg_flavors, s->rg_flavors, n_rg_fl);
  UP(root_slot, h->root_slot.data(), N); UP(depth, h->depth.data(), N); UP(height, h->height.data(), N);
  UP(tree_start, h->tree_start.data(), D.nTrees + 1); UP(tree_nodes, h->tree_nodes.data(), h->tree_nodes.size());
  UP(tree_level, h->tree_level.data(), h->tree_level.size()); UP(lone_cqs, h->lone.data(), h->lone.size());
  UP(local_idx, h->local_idx.data(), N);
  UP(tree_flat, h->tree_flat.data(), h->tree_flat.size());
  UP(child_start, h->child_start.data(), N + 1); UP(child_list, h->child_list.data(), h->child_list.size());
  UP(root_cq_start, h->root_cq_start.data(), h->root_cq_start.size());
  UP(sn_node, h->sn_node.data(), h->sn_node.size()); UP(slot_base, h->slot_base.data(), h->slot_base.size());
  UP(nd_tin, h->nd_tin.data(), h->nd_tin.size()); UP(nd_tout, h->nd_tout.data(), h->nd_tout.size());
  UP(cq_path, h->cq_path.data(), h->cq_path.size()); UP(cq_plen, h->cq_plen.data(), h->cq_plen.size());
  UP(tree_blob, h->tree_blob.data(), h->tree_blob.size()); UP(tree_blob_off, h->tree_blob_off.data(), h->tree_blob_off.size());
  const size_t tl_cells = h->tree_nodes.size() * (size_t)FR;
  const bool tree_local = tl_cells && tl_cells < (size_t)INT32_MAX;
  i64 *tl[3] = {nullptr, nullptr, nullptr};  // subtree quota, borrowing limit, local quota
  auto layout = [&](Arena &a) {
    for (const HostTab &t : tabs) *t.dst = a.take<char>(t.bytes);
    if (tree_local) for (i64 *&t : tl) t = a.take<i64>(tl_cells);
  };
  if (!h->sarena.carve(layout)) return fail(h, KB_ERR_CUDA, "cudaMalloc failed");
  for (const HostTab &t : tabs) { CUDA_TRY(h, h2d(h, *t.dst, t.src, t.bytes)); *bytes += (int64_t)t.bytes; }
  D.tl_subtree = D.tl_blimit = D.tl_lquota = nullptr; D.tl_usage = nullptr;
  if (tree_local) {
    D.FR = FR; D.Q = Q;
    k_tl_static<<<(unsigned)((tl_cells + 255) / 256), 256, 0, h->stream>>>(D, tl[0], tl[1], tl[2], (int)tl_cells);
    k_tl_root<<<(unsigned)(((size_t)D.nTrees * FR + 255) / 256), 256, 0, h->stream>>>(D, tl[0], tl[2]);
    D.tl_subtree = tl[0]; D.tl_blimit = tl[1]; D.tl_lquota = tl[2];
  }
  D.path_stride = h->path_stride;
  return KB_OK;
}

// Per-cycle input tables, enqueued before build_dynamic: the DMA runs while the host validates the tables and sizes
// the scratch arena.  The caller's tables (dynamic part of kb_snapshot) usually sit close together in one pinned
// block (kb_alloc_pinned carved by the shim): when their host span is not much larger than their total size the
// whole span goes to the device with ONE DMA and the device tables alias into it at the same offsets; otherwise every
// table is copied on its own.
static int32_t upload_inputs(kb_handle *h, const kb_snapshot *s, bool reuse, int64_t *bytes) {
  DevSnap &D = h->D;
  const int Q = s->n_cq, R = s->n_resource, FR = s->n_flavor * R;
  // A / AU are CAPACITIES (kb_run_drain grows the admitted tables on the device); A_in / AU_in what the caller passed
  const size_t A_in = (size_t)s->n_adm, AU_in = (size_t)s->n_adm_use, A = A_in + h->drain_extra_adm, AUc = AU_in + h->drain_extra_au;
  const size_t P = (size_t)s->n_podset, W = (size_t)s->n_wl, H = (size_t)s->n_heads;
  std::vector<HostTab> tabs;
  // ClusterQueue usage: the full table with the other per-cycle tables | into the resident buffer (KB_F_USAGE_RESIDENT)
  // | the resident buffer patched with the caller's rows (usage_delta_*)
  const bool delta = s->usage_delta_cq != nullptr;
  const bool keep_usage = (s->flags & KB_F_USAGE_RESIDENT) != 0 && !h->drain_mode;
  const int32_t *d_delta_cq = nullptr; const i64 *d_delta_rows = nullptr;
  if (delta) {
    if (h->drain_mode) return fail(h, KB_ERR_INVALID, "usage deltas are not available for kb_run_drain");
    if (!reuse || !h->usage_res_valid || h->usage_res_gen != s->static_generation || h->usage_res_cells != (size_t)Q * FR)
      return fail(h, KB_ERR_INVALID, "usage_delta_*: no resident usage table of this static_generation (pass cq_usage with KB_F_USAGE_RESIDENT first)");
    if (s->n_usage_delta < 0 || (s->n_usage_delta > 0 && !s->usage_delta_rows)) return fail(h, KB_ERR_INVALID, "usage_delta_*: bad count / null rows");
    h->delta_stamp++;
    if ((int)h->delta_seen.size() < Q || h->delta_stamp == 0) { h->delta_seen.assign((size_t)std::max(1, Q), 0); h->delta_stamp = 1; }
    for (int i = 0; i < s->n_usage_delta; i++) {
      const int c = s->usage_delta_cq[i];
      if (c < 0 || c >= Q) return fail(h, KB_ERR_INVALID, "usage_delta_cq out of range");
      if (h->delta_seen[c] == h->delta_stamp) return fail(h, KB_ERR_INVALID, "usage_delta_cq lists a ClusterQueue twice");
      h->delta_seen[c] = h->delta_stamp;
    }
    tabs.push_back(HostTab{(const void *)s->usage_delta_cq, (size_t)s->n_usage_delta * 4, (const void **)&d_delta_cq, (size_t)s->n_usage_delta * 4});
    tabs.push_back(HostTab{(const void *)s->usage_delta_rows, (size_t)s->n_usage_delta * FR * 8, (const void **)&d_delta_rows, (size_t)s->n_usage_delta * FR * 8});
  } else if (keep_usage) {
    if (h->usage_res_cells != (size_t)Q * FR || !h->d_usage_res) {
      if (h->d_usage_res) cudaFree(h->d_usage_res);
      h->d_usage_res = nullptr; h->usage_res_cells = 0;
      if (cudaMalloc((void **)&h->d_usage_res, std::max<size_t>(8, (size_t)Q * FR * 8)) != cudaSuccess) return fail(h, KB_ERR_CUDA, "cudaMalloc failed");
      h->usage_res_cells = (size_t)Q * FR;
    }
  } else {
    UP(cq_usage, (const i64 *)s->cq_usage, (size_t)Q * FR);
  }
  if (!delta) h->usage_res_valid = false;  // a full table supersedes whatever was resident
  UP(wl_cq, s->wl_cq, W); UP(wl_priority, s->wl_priority, W); UP(wl_ts, (const i64 *)s->wl_ts, W); UP(wl_uid, (const i64 *)s->wl_uid, W);
  UP(wl_last_gen, (const i64 *)s->wl_last_gen, W); UP(wl_ps_start, s->wl_ps_start, W + 1);
  UP(ps_req, (const i64 *)s->ps_req, P * R); UP(ps_req_mask, s->ps_req_mask, P); UP(ps_count, s->ps_count, P);
  UP(ps_min_count, s->ps_min_count, P); UP(ps_flavor_ok, (const u64 *)s->ps_flavor_ok, P); UP(ps_last_tried, s->ps_last_tried, P * R);
  UPC(adm_cq, s->adm_cq, A_in, A); UPC(adm_priority, s->adm_priority, A_in, A); UPC(adm_ts, (const i64 *)s->adm_ts, A_in, A);
  UPC(adm_qr_ts, (const i64 *)s->adm_qr_ts, A_in, A); UPC(adm_uid, (const i64 *)s->adm_uid, A_in, A); UPC(adm_evicted, s->adm_evicted, A_in, A);
  UPC(adm_use_start, s->adm_use_start, A_in + 1, A + 1); UPC(adm_use_fr, s->adm_use_fr, AU_in, AUc); UPC(adm_use_qty, (const i64 *)s->adm_use_qty, AU_in, AUc);
  if (!h->drain_mode) UP(heads, s->heads, H);
  D.wl_has_qr = nullptr; D.wl_sched_hash = nullptr; D.ps_group = nullptr;
  if (s->ps_group) UP(ps_group, s->ps_group, P);
  if (s->wl_has_quota_reservation) UP(wl_has_qr, s->wl_has_quota_reservation, W);
  if (s->wl_sched_hash) UP(wl_sched_hash, (const i64 *)s->wl_sched_hash, W);
  uintptr_t lo = UINTPTR_MAX, hi = 0; size_t sum = 0;
  for (const HostTab &t : tabs) {
    if (!t.bytes) continue;
    if (!t.src) return fail(h, KB_ERR_INVALID, "null table with non-zero length");
    if (t.cap != t.bytes) continue;  // growable table: its own allocation
    lo = std::min(lo, (uintptr_t)t.src); hi = std::max(hi, (uintptr_t)t.src + t.bytes); sum += t.bytes;
  }
  const uintptr_t lo_al = lo & ~(uintptr_t)255;
  const bool span = sum > 0 && (hi - lo) <= sum + sum / 4 + (64u << 10) && inside_one_pinned_block(lo_al, hi);
  auto in_span = [&](const HostTab &t) { return span && t.bytes && t.cap == t.bytes; };
  char *dspan = nullptr;
  auto layout = [&](Arena &a) {
    if (span) dspan = a.take<char>(hi - lo_al);
    for (const HostTab &t : tabs) if (!in_span(t)) *t.dst = a.take<char>(std::max(t.bytes, t.cap));
  };
  if (!h->iarena.carve(layout)) return fail(h, KB_ERR_CUDA, "cudaMalloc failed");
  CUDA_TRY(h, cudaEventRecord(h->ev0, h->stream));
  if (span) {
    CUDA_TRY(h, cudaMemcpyAsync(dspan, (const void *)lo_al, hi - lo_al, cudaMemcpyHostToDevice, h->stream));
    *bytes += (int64_t)(hi - lo_al);
  }
  for (const HostTab &t : tabs) {
    if (in_span(t)) *t.dst = dspan + ((uintptr_t)t.src - lo_al);
    else { CUDA_TRY(h, h2d(h, *t.dst, t.src, t.bytes)); *bytes += (int64_t)t.bytes; }
  }
  if (delta) {
    D.cq_usage = h->d_usage_res;
    const int nd = s->n_usage_delta;
    if (nd > 0) k_usage_patch<<<(unsigned)(((size_t)nd * FR + 255) / 256), 256, 0, h->stream>>>(h->d_usage_res, d_delta_cq, d_delta_rows, nd, FR);
  } else if (keep_usage) {
    if ((size_t)Q * FR) {
      if (!s->cq_usage) return fail(h, KB_ERR_INVALID, "null table with non-zero length");
      CUDA_TRY(h, cudaMemcpyAsync(h->d_usage_res, s->cq_usage, (size_t)Q * FR * 8, cudaMemcpyHostToDevice, h->stream));
      *bytes += (int64_t)Q * FR * 8;
    }
    D.cq_usage = h->d_usage_res;
    h->usage_res_valid = s->static_generation != 0; h->usage_res_gen = s->static_generation;
  }
  CUDA_TRY(h, cudaEventRecord(h->ev1, h->stream));
  return KB_OK;
}
#undef UP
#undef UPC

// Launch configuration of the preemption-target searches of this upload (h->plan), and the scratch sizes they need.
static void plan_search(kb_handle *h, const kb_snapshot *s) {
  SearchPlan &p = h->plan;
  const int R = s->n_resource, FR = s->n_flavor * R;
  const size_t H = (size_t)s->n_heads, A = (size_t)s->n_adm + h->drain_extra_adm;
  const bool fair = (s->flags & KB_F_FAIR_SHARING) != 0;
  p.search_grid = 1; p.search_smem = true; p.search_smem_bytes = 0;
  p.ws_warps = 1; p.ws_col_stride = 0; p.ws_list_total = 32;
  p.memo_items = A ? std::min<size_t>(H, (64u << 20) / ((size_t)FR * sizeof(SimMemo))) : 0;
  if (fair && A) {  // fair-sharing preemption: single-warp CTAs on a private copy of the whole tree
    // private tree tables [nodes][FR] x 4, parent links, per-node search state (16 B: queue head, cached share, flags)
    size_t tb = (size_t)h->max_tree_nodes * FR * 32 + (size_t)h->max_tree_nodes * 4 + (size_t)h->max_tree_nodes * 16 + 128;
    p.search_smem = tb <= 190 * 1024;
    p.search_smem_bytes = p.search_smem ? tb : 0;
    // resident single-warp CTAs per SM as the occupancy calculator sees them (registers / shared memory)
    int per_sm = 1;
    if (p.search_smem) {
      cudaFuncSetAttribute(k_nominate_search_fair<true, true>, cudaFuncAttributeMaxDynamicSharedMemorySize, 200 * 1024);
      cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, k_nominate_search_fair<true, true>, 32, p.search_smem_bytes);
    } else {
      cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, k_nominate_search_fair<false, true>, 32, 0);
    }
    per_sm = std::max(1, std::min(per_sm, 16));
    // the oracle-cell pass has up to FR tasks per entry
    p.search_grid = (int)std::max<size_t>(1, std::min<size_t>((size_t)h->sm_count * per_sm, std::max<size_t>(1, H * (size_t)FR)));
  } else if (A) {
    // warp-cooperative classical search: shared memory per warp = context + private column(s) + candidate codes
    const size_t kSmemBudget = 200 * 1024;
    size_t ncap_s = (size_t)h->max_tree_nodes;
    // k_search_cells: one column, codes of the longest bucket
    size_t ctxA = (sizeof(WCtx<1>) + 15) & ~(size_t)15;
    size_t colA = ncap_s * 8 <= 48 * 1024 ? ncap_s : 0;
    size_t codesA = (size_t)h->max_frl_len <= 8192 ? (((size_t)h->max_frl_len + 31) & ~(size_t)31) : 0;
    size_t perA = ctxA + ((colA * 8 + 15) & ~(size_t)15) + ((codesA + 15) & ~(size_t)15);
    int wpbA = (int)std::max<size_t>(1, std::min<size_t>(16, kSmemBudget / perA));
    int bpsA = (int)std::max<size_t>(1, std::min<size_t>(32 / wpbA, (220 * 1024) / (perA * wpbA + 1024)));
    p.sa_wpb = wpbA; p.sa_col_elems = (int)colA; p.sa_codes = (int)codesA; p.sa_smem = perA * wpbA;
    p.sa_grid = std::max(1, std::min(h->sm_count * bpsA, (int)((H * (size_t)FR + 31) / 32)));
    // grouped form: one column's statics + base usage shared by the CTA, private column + codes per warp
    size_t shared_b = ((ncap_s * (sizeof(ColStat) + 8)) + 15) & ~(size_t)15;
    size_t perG = ctxA + ((ncap_s * 8 + 15) & ~(size_t)15) + ((codesA + 15) & ~(size_t)15);
    size_t budget = 220 * 1024;
    int wpbG = shared_b + perG <= budget ? (int)std::min<size_t>(16, (budget - shared_b) / perG) : 0;
    p.sg_on = wpbG >= 4;
    p.sg_wpb = std::max(1, wpbG); p.sg_ncap = (int)ncap_s; p.sg_smem = shared_b + perG * p.sg_wpb;
    p.sg_grid = h->sm_count;
    if (p.sg_on) { wpbA = std::max(wpbA, wpbG); p.sa_grid = std::max(p.sa_grid, p.sg_grid); }
    // k_nominate_walk: up to Kcap columns (cells of one workload's assignment)
    size_t kcap = std::min<size_t>(std::min<size_t>((size_t)FR, KB_MAX_CELLS), (size_t)h->max_head_podsets * R);
    size_t ctxB = (sizeof(WCtx<KB_MAX_CELLS>) + 15) & ~(size_t)15;
    // The walk is a chain of dependent loads per entry: occupancy (16 warps per SM at 128 registers) hides more
    // latency than shared-memory columns would save, so the private columns of its searches live in global scratch.
    size_t colB = 0;
    size_t perB = ctxB;
    int wpbB = 8;
    int bpsB = 2;
    p.sb_wpb = wpbB; p.sb_col_elems = (int)colB; p.sb_smem = perB * wpbB;
    p.sb_grid = std::max(1, std::min(h->sm_count * bpsB, (int)((H + wpbB - 1) / wpbB)));
    p.ws_warps = std::max((size_t)p.sa_grid * wpbA, (size_t)p.sb_grid * wpbB);
    // per-warp candidate-code / target scratch: a single-cell search sees one bucket, GetTargets at most the root's list
    p.sa_list_cap = (int)(((size_t)h->max_frl_len + 31) & ~(size_t)31);
    p.sb_list_cap = (int)(((size_t)h->max_root_adm + 31) & ~(size_t)31);
    p.ws_list_total = std::max((size_t)p.sa_grid * wpbA * p.sa_list_cap, (size_t)p.sb_grid * wpbB * p.sb_list_cap);
    if (colA == 0) p.ws_col_stride = ncap_s;
    if (kcap * ncap_s > colB) p.ws_col_stride = std::max(p.ws_col_stride, std::min<size_t>((size_t)FR, KB_MAX_CELLS) * ncap_s);
  }
  p.G = (fair && A) ? (size_t)p.search_grid : 1, p.acap = (fair && A) ? (size_t)h->max_root_adm : 1, p.ncap = (size_t)h->max_tree_nodes;
}

// Fused per-root cycle (k_cycle_root), and its k_cycle_flat form: see the kernels' headers for the conditions
static void choose_route(kb_handle *h, const kb_snapshot *s) {
  const DevSnap &D = h->D;
  const int R = s->n_resource, FR = s->n_flavor * R;
  bool all_flat = true;
  for (uint8_t f : h->tree_flat) if (!f) all_flat = false;
  size_t nnm = (size_t)h->max_tree_nodes, tbm = nnm * FR;
  h->fused_smem = 6 * tbm * 8 + 2 * nnm * R * 8 + 4 * nnm * 4 + 7 * KB_TILE * 4 + (KB_MAX_DEPTH + 2 + 4) * 4 + 32 + nnm * 32;
  h->fused_on = D.nLone == 0 && D.nTrees > 0 && h->one_head_per_cq && h->fused_smem <= 220 * 1024 &&
                ((s->n_adm == 0 && !h->drain_events) || !h->preempt_possible) && (!(s->flags & KB_F_FAIR_SHARING) || all_flat) &&
                getenv("KB_NO_FUSED") == nullptr;
  // k_cycle_flat: every tree flat, FR <= 64, the relocated copy of the largest root fits shared memory
  h->flat_rcap = (int)std::min<size_t>((size_t)1 << 20, nnm * (size_t)std::max(1, h->max_head_podsets));
  h->flat_smem = flat_layout((int)nnm, FR, R, h->flat_rcap, h->max_blob_bytes).total;
  if (h->flat_static_smem == 0) { cudaFuncAttributes fa{}; cudaFuncGetAttributes(&fa, k_cycle_flat); h->flat_static_smem = std::max<size_t>(16, fa.sharedSizeBytes); }
  h->flat_on = h->fused_on && all_flat && FR <= 64 && h->flat_smem + h->flat_static_smem <= 227 * 1024 && getenv("KB_FUSED_V1") == nullptr;
  h->flat_on = h->flat_on && h->max_head_podsets < KB_REC_GENERAL && D.tl_subtree != nullptr;  // head record; staged from the tree-local tables only
}

// Per-cycle scratch and result block, described once (Arena::carve), and the clears and launches that prepare them
static int32_t carve_scratch(kb_handle *h, const kb_snapshot *s) {
  DevSnap &D = h->D;
  const SearchPlan &p = h->plan;
  const int Q = s->n_cq, N = Q + s->n_cohort, R = s->n_resource, FR = s->n_flavor * R, nroots = D.nRoots;
  const size_t NF = (size_t)N * FR, P = (size_t)s->n_podset, H = (size_t)s->n_heads;
  const size_t A = (size_t)s->n_adm + h->drain_extra_adm, AUc = (size_t)s->n_adm_use + h->drain_extra_au;
  const bool fair = (s->flags & KB_F_FAIR_SHARING) != 0;
  h->rk_temp_bytes = 0;
  if (A) {
    size_t b1 = 0, b2 = 0;
    cub::DoubleBuffer<u64> dk(nullptr, nullptr); cub::DoubleBuffer<int32_t> dv(nullptr, nullptr);
    cub::DeviceRadixSort::SortPairs(nullptr, b1, dk, dv, (int)A, 0, 64, h->stream);
    cub::DeviceRadixSort::SortPairs(nullptr, b2, (const u64 *)nullptr, (u64 *)nullptr, (const int32_t *)nullptr, (int32_t *)nullptr, (int)A, 0, 32, h->stream);
    h->rk_temp_bytes = std::max(b1, b2) + 256;
  }
  // the entries' target lists may name the same admitted workload many times (one per entry that preempts it), so the
  // pool is at least as large as the caller's target buffer
  const size_t G = p.G, acap = p.acap, ncap = p.ncap, pool_cap = std::max(A * 4 + 1024, h->out_tgt_capacity);
  const size_t nbuckets = (size_t)nroots * FR, sNF = A ? NF : 1, sAU = A ? AUc : 1, tl_cells = h->tree_nodes.size() * (size_t)FR;
  const OutLayout L = out_layout(H, P, (size_t)R);
  auto layout = [&](Arena &a) {
    if (h->drain_mode) D.heads = a.take<int32_t>(H);
    D.cq_entry = h->d_cq_entry = a.take<int32_t>(Q);
    D.cq_rec = h->d_cq_rec = a.take<int4>(h->tree_nodes.size() + 1);
    D.tl_usage = D.tl_subtree ? a.take<i64>(tl_cells) : nullptr;
    D.over_list = a.take<int32_t>(Q); D.over_count = a.take<int32_t>(nroots);
    D.root_adm_start = a.take<int32_t>(nroots + 1); D.cq_adm_start = a.take<int32_t>(Q + 1);
    D.cq_adm = a.take<int32_t>(A); D.adm_rank = a.take<int32_t>(A);
    D.root_adm_count = a.take<int32_t>(nroots + 2); D.cq_adm_count = a.take<int32_t>(Q + 2);
    h->rk_keys[0] = a.take<u64>(A); h->rk_keys[1] = a.take<u64>(A);
    D.adm_sorted = h->rk_vals[0] = a.take<int32_t>(A); h->rk_vals[1] = a.take<int32_t>(A);
    h->rk_temp = a.take<char>(h->rk_temp_bytes);
    D.subtree = a.take<i64>(NF); D.usage = a.take<i64>(NF);
    D.avail = a.take<i64>(NF); D.potential = a.take<i64>(NF);
    D.root_count = a.take<int32_t>(nroots); D.root_offset = a.take<int32_t>(nroots + 1);
    D.root_cursor = a.take<int32_t>(nroots); D.root_entries = a.take<int32_t>(H);
    D.sorted = a.take<int32_t>(H); D.pos_slot = a.take<int32_t>(H); D.ekey = a.take<u64>(H * 4); D.skey = a.take<u64>(H * 4);
    D.fs_over = a.take<i64>((size_t)Q * R); D.fs_lend = a.take<i64>((size_t)N * R);
    h->d_out_block = a.take<char>(L.prefix);  // the result tables and the cycle header in the canonical layout (out_layout)
    D.ps_list = a.take<int32_t>(H);
    D.tgt_off = a.take<int32_t>(H); D.tgt_cnt = a.take<int32_t>(H);
    D.tgt_pool_adm = a.take<int32_t>(pool_cap); D.tgt_pool_reason = a.take<uint8_t>(pool_cap);
    h->d_tgt_start = a.take<int32_t>(H + 1); h->d_tgt_adm = a.take<int32_t>(pool_cap); h->d_tgt_reason = a.take<uint8_t>(pool_cap);
    D.preempted = a.take<uint8_t>(A);
    D.usage_shadow = a.take<i64>(A ? NF : 1);
    D.sc_cand = a.take<int32_t>(G * acap); D.sc_tgt = a.take<int32_t>(G * acap); D.sc_cq_lca = a.take<int32_t>(G * ncap);
    D.sc_aux1 = a.take<int32_t>(G * acap); D.sc_aux2 = a.take<int32_t>(G * acap);
    D.sc_variant = a.take<uint8_t>(G * acap); D.sc_tgt_reason = a.take<uint8_t>(G * acap);
    D.sc_cq_class = a.take<int8_t>(G * ncap); D.sc_on_path = a.take<int8_t>(G * ncap);
    D.sc_dirty = a.take<uint8_t>(G * ncap); D.sc_drs_ratio = a.take<double>(G * ncap); D.sc_drs_meta = a.take<int8_t>(G * ncap);
    D.sc_usage = (fair && A && !p.search_smem) ? a.take<i64>(G * ncap * FR) : nullptr;
    D.colU = a.take<i64>(sNF); D.colS = a.take<ColStat>(sNF); D.ovm = a.take<uint32_t>(sNF);
    D.frl_count = a.take<int32_t>(A ? nbuckets + 1 : 1); D.frl_start = a.take<int32_t>(A ? nbuckets + 2 : 1);
    D.frl = a.take<FrRec>(sAU); D.rrec = a.take<FrRec>(A);
    D.memo = a.take<SimMemo>(p.memo_items * FR);
    D.cell_cursor = a.take<int32_t>(1);
    D.cell_count = a.take<int32_t>(A ? nbuckets + 2 : 1); D.cell_start = a.take<int32_t>(A ? nbuckets + 2 : 1);
    D.cell_fill = a.take<int32_t>(A ? nbuckets + 2 : 1);
    D.cell_list = a.take<int32_t>(p.memo_items * FR); D.cell_bucket = a.take<int32_t>(p.memo_items * FR);
    D.ws_col = a.take<i64>(p.ws_warps * p.ws_col_stride);
    D.ws_codes = a.take<uint8_t>(p.ws_list_total); D.ws_tgt = a.take<int32_t>(p.ws_list_total);
    D.ws_tgt_reason = a.take<uint8_t>(p.ws_list_total);
    D.ws_tgtq = a.take<i64>(p.ws_warps * (size_t)p.sa_list_cap);
    if (fair) {
      D.q_scratch = a.take<i64>(H * FR); D.fs_state = a.take<unsigned char>(H * (48 + 16 * KB_MAX_DEPTH));
      D.fs_cq_entry = a.take<int32_t>(N); D.fs_winner = a.take<int32_t>(N);
    }
    h->d_drs_rounded = a.take<i64>(N); h->d_drs_res = a.take<int32_t>(N); h->d_drs_borrowing = a.take<uint8_t>(N);
  };
  if (!h->arena.carve(layout)) return fail(h, KB_ERR_CUDA, "cudaMalloc failed");
  char *ob = h->d_out_block;
  D.decision = (uint8_t *)(ob + L.off[0]); D.mode = (uint8_t *)(ob + L.off[1]);
  D.borrow = (int32_t *)(ob + L.off[2]); D.rank = (int32_t *)(ob + L.off[3]);
  D.ps_flavor = (int8_t *)(ob + L.off[4]); D.ps_res_mode = (int8_t *)(ob + L.off[5]); D.ps_tried = (int8_t *)(ob + L.off[6]);
  D.ps_count_out = (int32_t *)(ob + L.off[7]);
  // cycle header, cleared once per cycle: [0] status, [2..3] ps_n / ps_cursor, [4] target pool cursor, [8..23] search counters
  uint32_t *hdr = (uint32_t *)(ob + L.hdr);
  D.status = hdr; D.ps_n = (int32_t *)(hdr + 2); D.ps_cursor = D.ps_n + 1; D.tgt_pool_used = (int32_t *)(hdr + 4); D.sstat = (u64 *)(hdr + 8);
  D.tgt_pool_cap = (int)pool_cap; D.sc_adm_cap = (int)acap; D.sc_node_cap = (int)ncap;
  D.memo_items = (int)p.memo_items; D.ws_col_stride = p.ws_col_stride; D.ws_tgtq_cap = p.sa_list_cap;
  if (h->fused_on && !h->flat_on && !h->drain_mode) {
    CUDA_TRY(h, cudaMemsetAsync(h->d_cq_entry, 0xff, sizeof(int32_t) * (size_t)Q, h->stream));
    if (H) k_cq_entry<<<(unsigned)((H + 255) / 256), 256, 0, h->stream>>>(D, h->d_cq_entry);
  }
  if (!A) {  // candidates_possible() reads the (empty) group tables
    CUDA_TRY(h, cudaMemsetAsync(D.root_adm_start, 0, sizeof(int32_t) * (size_t)(nroots + 1), h->stream));
    CUDA_TRY(h, cudaMemsetAsync(D.cq_adm_start, 0, sizeof(int32_t) * (size_t)(Q + 1), h->stream));
  }
  h->hdr_clean = false;
  if (h->flat_on && !h->drain_mode) {  // head records + result-row fills + cleared header: one launch (k_flat_prep)
    int32_t rc = flat_rec_stamp(h);
    if (rc != KB_OK) return rc;
    const size_t fill_words = 3 * pad256(P * R) / 4;
    const size_t tlc = D.tl_usage ? tl_cells : 0;
    const size_t nthr = std::max(std::max(std::max(H, fill_words), std::max(P, (size_t)32)), tlc);
    k_flat_prep<<<(unsigned)((nthr + 255) / 256), 256, 0, h->stream>>>(D, h->d_cq_rec, (int)fill_words, (int)P, (int)tlc);
    h->hdr_clean = true;
  } else {
    // rows of workloads that are not heads stay at -1
    CUDA_TRY(h, cudaMemsetAsync(D.ps_flavor, 0xff, 3 * pad256(P * R), h->stream));  // flavor, res_mode, tried are adjacent (out_layout)
    CUDA_TRY(h, cudaMemsetAsync(D.ps_count_out, 0, P * 4, h->stream));
  }
  return KB_OK;
}

// The failure paths past the first copy synchronise the stream before they return: the copies read the caller's
// buffers, which the caller may release once the call returns.
static int32_t upload_impl(kb_handle *h, const kb_snapshot *s, bool sync) {
  if (!h || !s) return KB_ERR_INVALID;
  cudaSetDevice(h->device);
  h->uploaded = false;
  DevSnap &D = h->D;
  const int Q = s->n_cq, C = s->n_cohort, F = s->n_flavor, R = s->n_resource;
  const int n_rg_fl = (s->n_rg > 0 && s->rg_flavor_start) ? s->rg_flavor_start[s->n_rg] : 0;
  const int dims[6] = {Q, C, F, R, s->n_rg, n_rg_fl};
  const bool reuse = s->static_generation != 0 && s->static_generation == h->static_gen && memcmp(dims, h->s_dims, sizeof(dims)) == 0;
  auto refuse = [h](int32_t rc) { cudaStreamSynchronize(h->stream); return rc; };
  int64_t bytes = 0;
  if (!reuse) {
    h->static_gen = 0;
    const int32_t rc = upload_static(h, s, n_rg_fl, &bytes);
    if (rc != KB_OK) return refuse(rc);
    memcpy(h->s_dims, dims, sizeof(dims));
    h->static_gen = s->static_generation;
  }
  int32_t rc = upload_inputs(h, s, reuse, &bytes);
  if (rc == KB_OK) rc = build_dynamic(h, s);
  if (rc != KB_OK) return refuse(rc);
  D.tab_local = 0; D.gparent = D.parent; D.lq = nullptr; D.cq_entry = nullptr; D.ent_gid = nullptr; D.node_gid = nullptr; D.local_flat = 0; D.cq_rec = nullptr;
  D.Q = Q; D.C = C; D.N = Q + C; D.F = F; D.R = R; D.FR = F * R; D.W = s->n_wl; D.P = s->n_podset; D.A = s->n_adm;
  D.AU = s->n_adm_use; D.H = s->n_heads; D.NRG = s->n_rg; D.pods_res = s->pods_resource; D.flags = s->flags; D.now_ns = s->now_ns;
  plan_search(h, s);
  choose_route(h, s);
  rc = carve_scratch(h, s);
  if (rc != KB_OK) return refuse(rc);
  h->stats.h2d_bytes = bytes;
  h->uploaded = true;
  if (sync) {  // caller buffers may be released after return
    CUDA_TRY(h, cudaStreamSynchronize(h->stream));
    float ms = 0; cudaEventElapsedTime(&ms, h->ev0, h->ev1);
    h->stats.last_h2d_ms = ms;
  }
  return KB_OK;
}

extern "C" int32_t kb_upload(kb_handle *h, const kb_snapshot *s) { return upload_impl(h, s, true); }

// per-kernel timing: an event before each kernel (and one after the last) when profiling
static inline void kmark(kb_handle *h, int id) {
  if (!h->profile || h->kev_n > KB_N_KERNELS) return;
  h->kev_id[h->kev_n] = id;
  cudaEventRecord(h->kev[h->kev_n++], h->stream);
}
static int32_t launch_tree(kb_handle *h, int *launches) {
  DevSnap &D = h->D;
  if (D.nTrees) { kmark(h, KB_K_TREE); k_tree<<<D.nTrees, 1024, 0, h->stream>>>(D); (*launches)++; }
  if (D.nLone) { kmark(h, KB_K_LONE); int n = D.nLone * D.FR; k_lone<<<(n + 255) / 256, 256, 0, h->stream>>>(D); (*launches)++; }
  return KB_OK;
}

// admit kernel launches: lone-CQ roots (slots [0, nLone)) and cohort-tree roots
// (slots [nLone, nRoots)) separately so each class gets the shared memory it needs.
// k_admit's shared memory: quota tables of nn_tables nodes, a request tile of `tile` entries x FR, tile metadata, path
static size_t admit_smem(int nn_tables, int FR, int tile, int nn_stage = 0) {
  size_t tb = (size_t)nn_tables * FR * 32;
  size_t mid = (size_t)tile * FR * 8;
  // global-table mode: staging buffers of the commit pipeline (k_admit: cells, path table, target ids, scratch)
  size_t staging = nn_stage ? sizeof(TgCell) * 2 * KB_SUB * KB_ECAP + 4 * (size_t)nn_stage * KB_PF + 4 * 2 * KB_SUB * KB_TCAP +
                                  4 * KB_SUB * (KB_TCAP + 1) + 4 * KB_SUB * 32 + 2 * 2 * KB_SUB * 34 + (size_t)nn_stage + 2 * KB_SUB + 64
                            : 0;
  return tb + mid + 16 + (size_t)nn_tables * 4 + KB_TILE * 28 + (KB_MAX_DEPTH + 2) * 4 + 64 + staging;
}
// the longest request tile (<= KB_TILE entries) that fits `budget` next to the rest of k_admit's shared memory; 0 when
// not even one entry does.  KB_TILE entries of 1,024 cells take 1 MiB: wide snapshots commit in shorter tiles.
static int admit_tile(size_t budget, int nn_tables, int FR, int nn_stage = 0) {
  size_t fixed = admit_smem(nn_tables, FR, 0, nn_stage), row = (size_t)FR * 8;
  return fixed + row > budget ? 0 : (int)std::min<size_t>(KB_TILE, (budget - fixed) / row);
}
static int32_t launch_admit(kb_handle *h, int *launches) {
  DevSnap &D = h->D;
  const size_t kMaxSmem = 200 * 1024;
  if (D.nLone && D.lone_fast) {
    size_t sm = (size_t)KB_LONE_WARPS * 32 * D.FR * 8;
    CUDA_TRY(h, cudaFuncSetAttribute(k_admit_lone, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)kMaxSmem));
    k_admit_lone<<<(D.nLone + KB_LONE_WARPS - 1) / KB_LONE_WARPS, KB_LONE_WARPS * 32, sm, h->stream>>>(D); (*launches)++;
  }
  if (D.nLone) {
    int tile = admit_tile(kMaxSmem, 1, D.FR);
    if (!tile) return fail(h, KB_ERR_INVALID, "k_admit: one ClusterQueue's quota tables exceed shared memory");
    CUDA_TRY(h, cudaFuncSetAttribute(k_admit<true>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)kMaxSmem));
    k_admit<true><<<D.nLone, KB_ADMIT_THREADS, admit_smem(1, D.FR, tile), h->stream>>>(D, 0, tile, 0); (*launches)++;
  }
  bool fair_trees = D.nTrees && (D.flags & KB_F_FAIR_SHARING);
  bool any_deep = false;
  for (uint8_t f : h->tree_flat) if (!f) any_deep = true;
  if (fair_trees && any_deep) {  // tournament kernel for the non-flat trees (flat ones exit at once)
    // shared memory: [quota tables][path][per-entry tournament state]; entries per tree <= its ClusterQueues
    size_t tables = (size_t)h->max_tree_nodes * D.FR * 32 + (size_t)h->max_tree_nodes * 4 + 16;
    size_t misc = (KB_MAX_DEPTH + 2) * 4 + ((size_t)h->max_tree_nodes * 4 + 1) * 4 + 128 * 4 + 64;
    size_t state = (size_t)h->max_tree_nodes * (48 + 16 * KB_MAX_DEPTH);
    CUDA_TRY(h, cudaFuncSetAttribute(k_admit_fair<true>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)kMaxSmem));
    CUDA_TRY(h, cudaFuncSetAttribute(k_admit_fair<false>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)kMaxSmem));
    if (tables + misc <= kMaxSmem) {
      int in_smem = tables + misc + state <= kMaxSmem;
      k_admit_fair<true><<<D.nTrees, 128, tables + misc + (in_smem ? state : 0), h->stream>>>(D, D.nLone, in_smem); (*launches)++;
    } else {
      int in_smem = misc + state <= kMaxSmem;
      k_admit_fair<false><<<D.nTrees, 128, misc + (in_smem ? state : 0), h->stream>>>(D, D.nLone, in_smem); (*launches)++;
    }
  }
  if (D.nTrees) {  // classical order, and fair sharing in flat cohorts (static key order)
    // quota tables in shared memory when they fit next to a full tile, in global memory otherwise, with the staged
    // commit pipeline when its buffers fit next to a tile of at least one entry
    if (admit_smem(h->max_tree_nodes, D.FR, KB_TILE) <= kMaxSmem) {
      int tile = admit_tile(kMaxSmem, h->max_tree_nodes, D.FR);
      CUDA_TRY(h, cudaFuncSetAttribute(k_admit<true>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)kMaxSmem));
      k_admit<true><<<D.nTrees, KB_ADMIT_THREADS, admit_smem(h->max_tree_nodes, D.FR, tile), h->stream>>>(D, D.nLone, tile, 0); (*launches)++;
    } else {
      int tile = admit_tile(kMaxSmem, 0, D.FR, h->max_tree_nodes), staged = tile > 0;
      if (!staged) tile = admit_tile(kMaxSmem, 0, D.FR);
      if (!tile) return fail(h, KB_ERR_INVALID, "k_admit: no request tile fits shared memory");
      size_t sm = admit_smem(0, D.FR, tile, staged ? h->max_tree_nodes : 0);
      CUDA_TRY(h, cudaFuncSetAttribute(k_admit<false>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)kMaxSmem));
      k_admit<false><<<D.nTrees, KB_ADMIT_THREADS, sm, h->stream>>>(D, D.nLone, tile, staged); (*launches)++;
    }
  }
  return KB_OK;
}

static int32_t cycle_enqueue(kb_handle *h, bool hdr_copy = true) {
  if (!h || !h->uploaded) return fail(h, KB_ERR_INVALID, "kb_upload first");
  cudaSetDevice(h->device);
  DevSnap &D = h->D;
  int launches = 0;
  CUDA_TRY(h, cudaEventRecord(h->ev2, h->stream));
  // cycle header (status word, deferred-entry counters, target pool cursor, search counters): one contiguous block
  if (!h->hdr_clean) CUDA_TRY(h, cudaMemsetAsync(D.status, 0, 128, h->stream));  // (k_flat_prep cleared it with the upload)
  h->hdr_clean = false;
  if (!(h->fused_on && D.H)) CUDA_TRY(h, cudaMemsetAsync(D.root_count, 0, sizeof(int32_t) * (size_t)std::max(1, D.nRoots), h->stream));
  if (D.A) CUDA_TRY(h, cudaMemsetAsync(D.preempted, 0, (size_t)D.A, h->stream));
  h->kev_n = 0;
  int32_t rc_admit = KB_OK;
  if (D.A && !h->preempt_possible) { D.A = 0; D.AU = 0; }  // no ClusterQueue can ever preempt: the cycle never looks at the admitted tables
  if (D.A) {  // rank the admitted workloads (kb_rank.cuh): stable LSD passes UID -> reservation time -> (root | evicted | priority)
    kmark(h, KB_K_RANKADM);
    const int A = D.A, tb = 256, nb = (A + tb - 1) / tb;
    CUDA_TRY(h, cudaMemsetAsync(D.root_adm_count, 0, sizeof(int32_t) * (size_t)(D.nRoots + 2), h->stream));
    CUDA_TRY(h, cudaMemsetAsync(D.cq_adm_count, 0, sizeof(int32_t) * (size_t)(D.Q + 2), h->stream));
    cub::DoubleBuffer<u64> dk(h->rk_keys[0], h->rk_keys[1]);
    cub::DoubleBuffer<int32_t> dv(h->rk_vals[0], h->rk_vals[1]);
    size_t bytes = h->rk_temp_bytes;
    k_rank_keys_uid<<<nb, tb, 0, h->stream>>>(D, dk.Current(), dv.Current()); launches++;
    CUDA_TRY(h, cub::DeviceRadixSort::SortPairs(h->rk_temp, bytes, dk, dv, A, 0, 64, h->stream));
    k_rank_keys_qr<<<nb, tb, 0, h->stream>>>(D, dv.Current(), dk.Current()); launches++;
    CUDA_TRY(h, cub::DeviceRadixSort::SortPairs(h->rk_temp, bytes, dk, dv, A, 0, 64, h->stream));
    k_rank_keys_root<<<nb, tb, 0, h->stream>>>(D, dv.Current(), dk.Current()); launches++;
    int root_bits = 1; while ((1ll << root_bits) < (long long)D.nRoots) root_bits++;
    CUDA_TRY(h, cub::DeviceRadixSort::SortPairs(h->rk_temp, bytes, dk, dv, A, 0, 33 + root_bits, h->stream));
    D.adm_sorted = dv.Current();
    int32_t *other_vals = dv.Alternate();
    k_scan_i32<<<1, 1024, 0, h->stream>>>(D.root_adm_count, D.root_adm_start, D.nRoots); launches++;
    k_rank_positions<<<nb, tb, 0, h->stream>>>(D); launches++;
    // per-ClusterQueue lists in the same order: one more stable pass keyed by the ClusterQueue
    k_rank_keys_cq<<<nb, tb, 0, h->stream>>>(D, D.adm_sorted, dk.Current()); launches++;
    int cq_bits = 1; while ((1ll << cq_bits) < (long long)D.Q) cq_bits++;
    CUDA_TRY(h, cub::DeviceRadixSort::SortPairs(h->rk_temp, bytes, (const u64 *)dk.Current(), dk.Alternate(), (const int32_t *)D.adm_sorted, D.cq_adm, A, 0, cq_bits, h->stream));
    (void)other_vals;
    k_scan_i32<<<1, 1024, 0, h->stream>>>(D.cq_adm_count, D.cq_adm_start, D.Q); launches++;
    launches += 8;  // radix-sort passes (cub): histogram + onesweep kernels, counted coarsely
  }
  if (h->fused_on && D.H) {
    if (h->drain_mode) {
      if (h->flat_on) {
        int32_t rc2 = flat_rec_stamp(h);
        if (rc2 != KB_OK) return rc2;
        const size_t tlc = D.tl_usage ? h->tree_nodes.size() * (size_t)D.FR : 0;
        k_cq_rec<<<(unsigned)((std::max<size_t>((size_t)D.H, tlc) + 255) / 256), 256, 0, h->stream>>>(D, h->d_cq_rec, (int)tlc); launches++;
      } else {
        CUDA_TRY(h, cudaMemsetAsync(h->d_cq_entry, 0xff, sizeof(int32_t) * (size_t)D.Q, h->stream));
        k_cq_entry<<<(D.H + 255) / 256, 256, 0, h->stream>>>(D, h->d_cq_entry); launches++;
      }
    }
    kmark(h, KB_K_CYCLE_ROOT);
    if (h->flat_on) {
      if (!h->flat_attr_set) { CUDA_TRY(h, cudaFuncSetAttribute(k_cycle_flat, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)(227 * 1024 - h->flat_static_smem))); h->flat_attr_set = true; }
      k_cycle_flat<<<D.nTrees, KB_FLAT_THREADS, h->flat_smem, h->stream>>>(D, flat_layout(h->max_tree_nodes, D.FR, D.R, h->flat_rcap, h->max_blob_bytes)); launches++;
    } else {
      CUDA_TRY(h, cudaFuncSetAttribute(k_cycle_root, cudaFuncAttributeMaxDynamicSharedMemorySize, 224 * 1024));
      k_cycle_root<<<D.nTrees, KB_ROOT_THREADS, h->fused_smem, h->stream>>>(D); launches++;
    }
  } else {
  launch_tree(h, &launches);
  if (D.H) {
    // per-(node, resource) sums the DominantResourceShare reads (fair target search, fair admit loop); only needs the tree pass
    if (D.flags & KB_F_FAIR_SHARING) { kmark(h, KB_K_FAIR_PREP); k_fair_prep<<<(D.N * D.R + 255) / 256, 256, 0, h->stream>>>(D); launches++; }
    kmark(h, KB_K_NOMINATE);
    // few entries: latency-bound -> KB_NG lanes per entry; many entries: throughput-bound -> one thread per entry
    if ((size_t)D.H * KB_NG <= (size_t)h->sm_count * 2048) k_nominate_coop<<<(int)(((size_t)D.H * KB_NG + 127) / 128), 128, 0, h->stream>>>(D);
    else k_nominate<<<(D.H + 127) / 128, 128, 0, h->stream>>>(D);
    launches++;
    if (D.A) {  // target search for the entries k_nominate deferred
      const SearchPlan &p = h->plan;
      if (D.flags & KB_F_FAIR_SHARING) {
        kmark(h, KB_K_PREEMPT);
        CUDA_TRY(h, cudaMemsetAsync(D.over_count, 0, sizeof(int32_t) * (size_t)std::max(1, D.nRoots), h->stream));
        k_over<<<(D.Q + 255) / 256, 256, 0, h->stream>>>(D); launches++;
        CUDA_TRY(h, cudaMemsetAsync(D.cell_cursor, 0, 4, h->stream));
        if (p.search_smem) {
          CUDA_TRY(h, cudaFuncSetAttribute(k_nominate_search_fair<true, true>, cudaFuncAttributeMaxDynamicSharedMemorySize, 200 * 1024));
          CUDA_TRY(h, cudaFuncSetAttribute(k_nominate_search_fair<true, false>, cudaFuncAttributeMaxDynamicSharedMemorySize, 200 * 1024));
          if (D.memo_items) { k_nominate_search_fair<true, true><<<p.search_grid, 32, p.search_smem_bytes, h->stream>>>(D); launches++; }
          k_nominate_search_fair<true, false><<<p.search_grid, 32, p.search_smem_bytes, h->stream>>>(D);
        } else {
          if (D.memo_items) { k_nominate_search_fair<false, true><<<p.search_grid, 32, 0, h->stream>>>(D); launches++; }
          k_nominate_search_fair<false, false><<<p.search_grid, 32, 0, h->stream>>>(D);
        }
        launches++;
      } else {
        // per-cycle search tables: transposed columns + above-nominal masks, candidate buckets per (root, flavor-resource)
        kmark(h, KB_K_SEARCH_TABLES);
        size_t nf = (size_t)D.N * D.FR;
        int nb = D.nRoots * D.FR;
        k_columns<<<(unsigned)((nf + 255) / 256), 256, 0, h->stream>>>(D); launches++;
        CUDA_TRY(h, cudaMemsetAsync(D.frl_count, 0, sizeof(int32_t) * (size_t)(nb + 1), h->stream));
        CUDA_TRY(h, cudaMemsetAsync(D.cell_cursor, 0, 4, h->stream));
        if (D.AU) { k_frl_count<<<(D.AU + 255) / 256, 256, 0, h->stream>>>(D); launches++; }
        k_scan_i32<<<1, 1024, 0, h->stream>>>(D.frl_count, D.frl_start, nb); launches++;
        k_root_recs<<<(D.A + 255) / 256, 256, 0, h->stream>>>(D); launches++;
        if (D.AU) { k_frl_fill<<<(unsigned)(((size_t)nb * 32 + 127) / 128), 128, 0, h->stream>>>(D); launches++; }
        CUDA_TRY(h, cudaFuncSetAttribute(k_search_cells, cudaFuncAttributeMaxDynamicSharedMemorySize, 224 * 1024));
        CUDA_TRY(h, cudaFuncSetAttribute(k_nominate_walk, cudaFuncAttributeMaxDynamicSharedMemorySize, 224 * 1024));
        kmark(h, KB_K_SEARCH_CELLS);
        if (p.sg_on && D.memo_items) {
          long long ncell = (long long)D.memo_items * D.FR;
          CUDA_TRY(h, cudaMemsetAsync(D.cell_count, 0, sizeof(int32_t) * (size_t)(nb + 1), h->stream));
          CUDA_TRY(h, cudaMemsetAsync(D.cell_fill, 0, sizeof(int32_t) * (size_t)(nb + 1), h->stream));
          k_cells_mark<<<(unsigned)((ncell + 255) / 256), 256, 0, h->stream>>>(D); launches++;
          k_scan_i32<<<1, 1024, 0, h->stream>>>(D.cell_count, D.cell_start, nb); launches++;
          k_cells_scatter<<<(unsigned)((ncell + 255) / 256), 256, 0, h->stream>>>(D); launches++;
          CUDA_TRY(h, cudaFuncSetAttribute(k_search_cells_grouped, cudaFuncAttributeMaxDynamicSharedMemorySize, 224 * 1024));
          k_search_cells_grouped<<<p.sg_grid, p.sg_wpb * 32, p.sg_smem, h->stream>>>(D, p.sg_ncap, p.sa_codes, p.sa_list_cap); launches++;
        } else {
          k_search_cells<<<p.sa_grid, p.sa_wpb * 32, p.sa_smem, h->stream>>>(D, p.sa_col_elems, p.sa_codes, p.sa_list_cap); launches++;
        }
        kmark(h, KB_K_WALK);
        k_nominate_walk<<<p.sb_grid, p.sb_wpb * 32, p.sb_smem, h->stream>>>(D, p.sb_col_elems, p.sb_list_cap); launches++;
      }
    }
    kmark(h, KB_K_SCAN); k_scan_roots<<<1, 1024, 0, h->stream>>>(D); launches++;
    kmark(h, KB_K_SCATTER); k_scatter<<<(D.H + 255) / 256, 256, 0, h->stream>>>(D); launches++;
    kmark(h, KB_K_RANK); k_rank<<<(D.H + 255) / 256, 256, 0, h->stream>>>(D); launches++;
    kmark(h, KB_K_ADMIT);
    rc_admit = launch_admit(h, &launches);
  }
  }
  kmark(h, -1);
  CUDA_TRY(h, cudaEventRecord(h->ev3, h->stream));
  if (rc_admit != KB_OK) return rc_admit;
  CUDA_TRY(h, cudaGetLastError());
  h->last_launches = launches;
  // the cycle header (status word, counters, search / phase statistics: 128 contiguous bytes) comes back with one copy —
  // or, when the caller's result block has the canonical layout, inside the block's own copy (download_enqueue)
  h->hdr_host = &h->host_words[32];
  if (hdr_copy) CUDA_TRY(h, cudaMemcpyAsync(&h->host_words[32], D.status, 128, cudaMemcpyDeviceToHost, h->stream));
  return KB_OK;
}

// after the stream has been synchronized: timings + device status word
static int32_t cycle_finish(kb_handle *h) {
  float ms = 0; cudaEventElapsedTime(&ms, h->ev2, h->ev3);
  h->stats.last_cycle_gpu_ms = ms;
  h->stats.kernel_launches = h->last_launches;
  for (int i = 0; i < KB_N_KERNELS; i++) h->stats.kernel_ms[i] = 0.f;
  for (int i = 0; i + 1 < h->kev_n; i++) {
    float kms = 0; cudaEventElapsedTime(&kms, h->kev[i], h->kev[i + 1]);
    if (h->kev_id[i] >= 0) h->stats.kernel_ms[h->kev_id[i]] += kms;
  }
  memcpy(h->stats.search_stat, h->hdr_host + 8, 64);
  memcpy(h->stats.flat_group_walk, h->hdr_host + 24, 16);  // DevSnap::sstat[8..9]
  uint32_t st = h->hdr_host[0];
  if (st & KBS_UNSUPPORTED_PREEMPTION) return fail(h, KB_ERR_UNSUPPORTED, "unsupported preemption configuration");
  if (st & KBS_TARGET_OVERFLOW) return fail(h, KB_ERR_CAPACITY, "per-entry usage cell / target pool capacity exceeded");
  if (st & KBS_INTERNAL_LOOP) return fail(h, KB_ERR_CUDA, "internal: iteration guard tripped in the target search");
  return KB_OK;
}

extern "C" int32_t kb_cycle_resident(kb_handle *h) {
  int32_t rc = cycle_enqueue(h);
  if (rc != KB_OK) return rc;
  CUDA_TRY(h, cudaStreamSynchronize(h->stream));
  return cycle_finish(h);
}

// preemption targets of the cycle from the per-entry pool slices into CSR order (kb_cycle_out.tgt_start / tgt_adm / tgt_reason)
__global__ void k_tgt_compact(DevSnap D, const int32_t *start, int32_t *adm, uint8_t *reason) {
  int e = blockIdx.x * blockDim.x + threadIdx.x;
  if (e >= D.H) return;
  int n = D.tgt_cnt[e], o = D.tgt_off[e], s = start[e];
  for (int k = 0; k < n; k++) { adm[s + k] = D.tgt_pool_adm[o + k]; reason[s + k] = D.tgt_pool_reason[o + k]; }
}

// a kb_alloc_cycle_out block of this cycle's dimensions, pointers untouched: its tables have the device block's layout
static bool out_is_canonical_block(kb_handle *h, const kb_cycle_out *out) {
  const DevSnap &D = h->D;
  const size_t H = D.H;
  if (!out || !out->decision || !H) return false;
  OutLayout L = out_layout(H, (size_t)D.P, (size_t)D.R);
  const char *b = (const char *)out->decision;
  bool ok;
  {
    std::lock_guard<std::mutex> lk(g_pin_mu);
    auto it = g_out_blocks.find((uintptr_t)b);
    ok = it != g_out_blocks.end() && it->second.H == H && it->second.P == (size_t)D.P && it->second.R == (size_t)D.R;
  }
  return ok && (const char *)out->mode == b + L.off[1] && (const char *)out->borrow == b + L.off[2] && (const char *)out->commit_rank == b + L.off[3] &&
         (const char *)out->ps_flavor == b + L.off[4] && (const char *)out->ps_res_mode == b + L.off[5] && (const char *)out->ps_tried_idx == b + L.off[6] &&
         (const char *)out->ps_count == b + L.off[7];
}

static int32_t download_enqueue(kb_handle *h, kb_cycle_out *out) {
  if (!h || !h->uploaded || !out) return fail(h, KB_ERR_INVALID, "nothing to download");
  cudaSetDevice(h->device);
  DevSnap &D = h->D;
  size_t H = D.H, PR = (size_t)D.P * D.R;
  int64_t bytes = 0;
  CUDA_TRY(h, cudaEventRecord(h->ev4, h->stream));
#define DOWN(dst, src, n, T) if (out->dst && (n)) { CUDA_TRY(h, cudaMemcpyAsync(out->dst, D.src, (n) * sizeof(T), cudaMemcpyDeviceToHost, h->stream)); bytes += (n) * sizeof(T); }
  const bool one_dma = out_is_canonical_block(h, out);
  if (one_dma) {  // the eight result tables and the cycle header: one copy
    OutLayout L = out_layout(H, (size_t)D.P, (size_t)D.R);
    CUDA_TRY(h, cudaMemcpyAsync(out->decision, h->d_out_block, L.prefix, cudaMemcpyDeviceToHost, h->stream)); bytes += (int64_t)L.prefix;
    h->hdr_host = (const uint32_t *)((const char *)out->decision + L.hdr);
  }
  if (!one_dma) {
    DOWN(decision, decision, H, uint8_t); DOWN(mode, mode, H, uint8_t); DOWN(borrow, borrow, H, int32_t); DOWN(commit_rank, rank, H, int32_t);
    DOWN(ps_flavor, ps_flavor, PR, int8_t); DOWN(ps_res_mode, ps_res_mode, PR, int8_t); DOWN(ps_tried_idx, ps_tried, PR, int8_t);
    DOWN(ps_count, ps_count_out, (size_t)D.P, int32_t);
  }
  DOWN(node_usage, usage, (size_t)D.N * D.FR, i64);
#undef DOWN
  h->tgt_csr = false;
  if (out->tgt_start && D.A && H) {  // target lists -> CSR on the device: scan of the per-entry counts, one gather
    k_scan_i32<<<1, 1024, 0, h->stream>>>(D.tgt_cnt, h->d_tgt_start, (int)H);
    k_tgt_compact<<<(unsigned)((H + 127) / 128), 128, 0, h->stream>>>(D, h->d_tgt_start, h->d_tgt_adm, h->d_tgt_reason);
    CUDA_TRY(h, cudaMemcpyAsync(out->tgt_start, h->d_tgt_start, (H + 1) * 4, cudaMemcpyDeviceToHost, h->stream));
    bytes += (int64_t)(H + 1) * 4;
    h->tgt_csr = true;
  }
  CUDA_TRY(h, cudaEventRecord(h->ev5, h->stream));
  h->last_d2h_bytes = bytes;
  return KB_OK;
}

// after the stream has been synchronized (and cycle_finish filled host_words): preemption targets -> CSR
static int32_t download_finish(kb_handle *h, kb_cycle_out *out) {
  DevSnap &D = h->D;
  size_t H = D.H;
  int64_t bytes = h->last_d2h_bytes;
  out->n_targets = 0;
  if (out->tgt_start) {
    if (!h->tgt_csr) memset(out->tgt_start, 0, sizeof(int32_t) * (H + 1));
    else {
      int32_t nt = out->tgt_start[H];
      out->n_targets = nt;
      if (nt > out->tgt_capacity) return fail(h, KB_ERR_CAPACITY, "target buffer too small");
      if (nt > 0 && out->tgt_adm && out->tgt_reason) {
        CUDA_TRY(h, cudaMemcpyAsync(out->tgt_adm, h->d_tgt_adm, (size_t)nt * 4, cudaMemcpyDeviceToHost, h->stream));
        CUDA_TRY(h, cudaMemcpyAsync(out->tgt_reason, h->d_tgt_reason, (size_t)nt, cudaMemcpyDeviceToHost, h->stream));
        CUDA_TRY(h, cudaStreamSynchronize(h->stream));
        bytes += (int64_t)nt * 5;
      }
    }
  }
  float ms = 0; cudaEventElapsedTime(&ms, h->ev4, h->ev5);
  h->stats.last_d2h_ms = ms; h->stats.d2h_bytes = bytes;
  return KB_OK;
}

extern "C" int32_t kb_download(kb_handle *h, kb_cycle_out *out) {
  int32_t rc = download_enqueue(h, out);
  if (rc != KB_OK) return rc;
  // the target count of the last cycle is re-read here in case kb_cycle_resident ran several times
  CUDA_TRY(h, cudaStreamSynchronize(h->stream));
  return download_finish(h, out);
}

// One blocking call, one stream synchronisation: H2D copies, kernels and D2H copies are all enqueued first.
extern "C" int32_t kb_run_cycle(kb_handle *h, const kb_snapshot *s, kb_cycle_out *out) {
  static const bool trace = getenv("KB_TRACE") != nullptr;  // host-side phase times of the call on stderr
  auto now = [] { return std::chrono::duration<double, std::micro>(std::chrono::steady_clock::now().time_since_epoch()).count(); };
  double t0 = trace ? now() : 0, t1 = 0, t2 = 0, t3 = 0;
  if (h && out) h->out_tgt_capacity = (size_t)std::max(0, out->tgt_capacity);
  int32_t rc = upload_impl(h, s, false);
  if (h) h->out_tgt_capacity = 0;
  if (rc != KB_OK) return rc;
  if (trace) t1 = now();
  rc = cycle_enqueue(h, !out_is_canonical_block(h, out));
  if (rc != KB_OK) return rc;
  if (trace) t2 = now();
  rc = download_enqueue(h, out);
  if (rc != KB_OK) return rc;
  if (trace) t3 = now();
  CUDA_TRY(h, cudaStreamSynchronize(h->stream));
  if (trace) fprintf(stderr, "kb_run_cycle host us: upload %.1f enqueue %.1f download-enqueue %.1f wait %.1f\n", t1 - t0, t2 - t1, t3 - t2, now() - t3);
  { float ms = 0; cudaEventElapsedTime(&ms, h->ev0, h->ev1); h->stats.last_h2d_ms = ms; }
  rc = cycle_finish(h);
  if (rc != KB_OK) return rc;
  return download_finish(h, out);
}

// ---------------------------------------------------------------------------
// kb_run_drain: iterated cycles with the queue layer on the device (kb_drain.cuh)
// ---------------------------------------------------------------------------
// what a boundary of kb_run_drain reads back, in the pinned host words [64, 128)
struct DrainWords {
  uint32_t counters[KB_DC_RECLAIMS + 1];  // DrainDev::counters; [0] = heads of the next cycle
  uint32_t n_new, n_cells;              // this cycle's admissions and their usage cells (the admit scans' totals)
  uint32_t status;                      // the cycle's status word (KBS_AFS_OVERFLOW)
  i64 t_next;                           // event mode: t_{c+1}
};
static_assert(sizeof(DrainWords) <= 64 * 4, "host_words[64..127] hold the words of a drain boundary");

// The blocks a drain runs (include/kueue_b200.h), worked out once from the snapshot by drain_mode.  evict and compact
// also depend on whether any ClusterQueue can preempt, which upload_impl works out: drain_plan sets them.
struct DrainMode {
  bool replay;   // adm_wl: the admitted rows name their pending records (eviction replay)
  bool events;   // event mode: a clock replays arrivals, completions and the event blocks below
  bool lat;      // eviction latency
  bool decay;    // decay of AdmissionFairSharing consumed usage
  bool sticky;   // sticky workload
  bool checks;   // admission checks
  bool pr;       // WaitForPodsReady
  bool requeue;  // checks or pr: BACKOFF / DEACTIVATED, RequeueAt, queue-order timestamps, re-sorts
  bool mx;       // MaximumExecutionTimeSeconds
  bool quota;    // ClusterQueue / Cohort quota changes
  bool act;      // deactivation / reactivation edits
  bool blk;      // the edits, or their start state (wl_inactive) alone
  bool deact;    // requeue, mx or blk: records carry a deactivation reason
  bool rcl;      // reclaim steps
  bool afs;      // AdmissionFairSharing queues (wl_lq)
  bool evict;    // a preemption can evict a row
  bool compact;  // rows can die: the admitted tables are compacted after every boundary
  int n_qc, n_ac, n_rc;  // quota changes, active changes and reclaim steps the drain replays
};
static DrainMode drain_mode(const kb_snapshot *s) {
  DrainMode m{};
  m.replay = s->adm_wl != nullptr;
  m.quota = s->n_quota_change > 0 && s->qc_ns;
  m.act = s->n_active_change > 0 && s->ac_ns;
  m.blk = m.act || s->wl_inactive;
  m.rcl = s->wl_rc_start != nullptr;
  m.events = s->wl_create_ns || s->wl_run_ns || s->adm_finish_ns || s->wl_evict_ns || s->wl_check_ns || s->wl_pods_ready_ns ||
             s->wl_max_exec_s || m.quota || m.act || m.rcl;
  m.lat = s->wl_evict_ns != nullptr;
  m.decay = s->lq_last_update_ns != nullptr;
  m.sticky = s->cq_sticky != nullptr;
  m.checks = s->wl_check_ns != nullptr;
  m.pr = s->wl_pods_ready_ns != nullptr;
  m.requeue = m.checks || m.pr;
  m.mx = s->wl_max_exec_s != nullptr;
  m.deact = m.requeue || m.mx || m.blk;
  m.afs = s->wl_lq != nullptr;
  m.n_qc = m.quota ? s->n_quota_change : 0;
  m.n_ac = m.act ? s->n_active_change : 0;
  m.n_rc = m.rcl ? s->n_reclaim : 0;
  return m;
}

// ---- input checks of kb_run_drain (include/kueue_b200.h), one per block, run in this order by drain_validate: a
// snapshot that breaks two rules fails the first.  held[w]: an admitted row names record w (filled by check_replay).
using HeldRecords = std::vector<uint8_t>;
static int32_t check_replay(kb_handle *h, const kb_snapshot *s, const DrainMode &m, HeldRecords &held) {
  if (!m.replay) return KB_OK;
  if (!(s->flags & KB_F_PRIORITY_SORTING_WITHIN_COHORT))
    return fail(h, KB_ERR_UNSUPPORTED, "adm_wl: eviction replay needs KB_F_PRIORITY_SORTING_WITHIN_COHORT (a preempted workload's queue-order timestamp would be its eviction time)");
  for (int a = 0; a < s->n_adm; a++) {
    const int w = s->adm_wl[a];
    if (w < 0 || w >= s->n_wl) return fail(h, KB_ERR_INVALID, "adm_wl out of range");
    if (held[w]) return fail(h, KB_ERR_INVALID, "adm_wl names a pending record twice");
    held[w] = 1;
    if (s->adm_cq[a] < 0 || s->adm_cq[a] >= s->n_cq || s->wl_cq[w] != s->adm_cq[a]) return fail(h, KB_ERR_INVALID, "adm_wl: the record's ClusterQueue is not the admitted workload's");
  }
  return KB_OK;
}
static int32_t check_events(kb_handle *h, const kb_snapshot *s, const DrainMode &m, HeldRecords &) {
  if (!m.events) return KB_OK;
  if (s->adm_finish_ns)
    for (int a = 0; a < s->n_adm; a++)
      if (s->adm_finish_ns[a] <= s->now_ns) return fail(h, KB_ERR_INVALID, "adm_finish_ns: a row admitted before the drain finishes at or before now_ns");
  if (m.replay && s->wl_create_ns)
    for (int a = 0; a < s->n_adm; a++)
      if (s->wl_create_ns[s->adm_wl[a]] > s->now_ns) return fail(h, KB_ERR_INVALID, "adm_wl names a record created after now_ns");
  return KB_OK;
}
static int32_t check_latency(kb_handle *h, const kb_snapshot *s, const DrainMode &m, HeldRecords &) {
  if (!m.lat && !s->adm_evict_end_ns) return KB_OK;
  if (!m.replay) return fail(h, KB_ERR_INVALID, "eviction latency: wl_evict_ns / adm_evict_end_ns need adm_wl");
  if (!m.lat) return fail(h, KB_ERR_INVALID, "eviction latency: adm_evict_end_ns needs wl_evict_ns");
  for (int w = 0; w < s->n_wl; w++)
    if (s->wl_evict_ns[w] < 0) return fail(h, KB_ERR_INVALID, "eviction latency: wl_evict_ns < 0");
  if (s->adm_evict_end_ns && s->adm_evicted)
    for (int a = 0; a < s->n_adm; a++)
      if (s->adm_evicted[a] && s->adm_evict_end_ns[a] <= s->now_ns)
        return fail(h, KB_ERR_INVALID, "eviction latency: an eviction under way before the drain ends at or before now_ns");
  return KB_OK;
}
static int32_t check_decay(kb_handle *h, const kb_snapshot *s, const DrainMode &m, HeldRecords &) {
  if (!m.decay) return KB_OK;
  if (!s->wl_lq || !s->lq_cq || !m.events) return fail(h, KB_ERR_INVALID, "afs decay: lq_last_update_ns needs wl_lq and event mode");
  if (s->afs_half_life_ns < 0 || s->afs_sampling_ns <= 0) return fail(h, KB_ERR_INVALID, "afs decay: half-life < 0 or sampling interval <= 0");
  if (!(s->afs_alpha >= 0.0 && s->afs_alpha < 1.0) || (s->afs_half_life_ns == 0 && s->afs_alpha != 0.0))
    return fail(h, KB_ERR_INVALID, "afs decay: afs_alpha outside [0, 1), or non-zero with half-life 0");
  for (int l = 0; l < s->n_lq; l++)
    if (s->lq_last_update_ns[l] > s->now_ns) return fail(h, KB_ERR_INVALID, "afs decay: lq_last_update_ns after now_ns");
  if (s->n_adm > 0 && !s->adm_lq) return fail(h, KB_ERR_INVALID, "afs decay: adm_lq is NULL while n_adm > 0");
  for (int a = 0; a < s->n_adm; a++) {
    const int l = s->adm_lq[a];
    if (l < -1 || l >= s->n_lq) return fail(h, KB_ERR_INVALID, "afs decay: adm_lq out of range");
    if (l >= 0 && s->lq_cq[l] != s->adm_cq[a]) return fail(h, KB_ERR_INVALID, "afs decay: the LocalQueue of an admitted row feeds another ClusterQueue");
  }
  return KB_OK;
}
static int32_t check_sticky(kb_handle *h, const kb_snapshot *s, const DrainMode &m, HeldRecords &held) {
  if (!m.sticky) return KB_OK;
  for (int q = 0; q < s->n_cq; q++) {
    const int w = s->cq_sticky[q];
    if (w < -1 || w >= s->n_wl) return fail(h, KB_ERR_INVALID, "cq_sticky out of range");
    if (w < 0) continue;
    if (s->wl_cq[w] != q) return fail(h, KB_ERR_INVALID, "cq_sticky: the workload is not in the ClusterQueue's queue");
    if (held[w]) return fail(h, KB_ERR_INVALID, "cq_sticky names a record that holds quota (adm_wl): admission deleted it from its queue");
    if (s->wl_create_ns && s->wl_create_ns[w] > s->now_ns) return fail(h, KB_ERR_INVALID, "cq_sticky names a record created after now_ns");
    if (s->wl_lq && s->cq_afs && s->cq_afs[q])
      return fail(h, KB_ERR_UNSUPPORTED, "cq_sticky: a sticky workload on a ClusterQueue with AdmissionFairSharing");
  }
  return KB_OK;
}
// wl_requeue_at_ns of record w (admission checks, PodsReady): a record in backoff holds no quota and exists at now_ns
static int32_t check_requeue_at(kb_handle *h, const kb_snapshot *s, const HeldRecords &held, int w, const std::string &block) {
  if (!s->wl_requeue_at_ns || s->wl_requeue_at_ns[w] == INT64_MIN) return KB_OK;
  if (held[w]) return fail(h, KB_ERR_INVALID, block + ": wl_requeue_at_ns on a record that holds quota (adm_wl)");
  if (s->wl_create_ns && s->wl_create_ns[w] > s->now_ns) return fail(h, KB_ERR_INVALID, block + ": wl_requeue_at_ns on a record created after now_ns");
  return KB_OK;
}
static int32_t check_checks(kb_handle *h, const kb_snapshot *s, const DrainMode &m, HeldRecords &held) {
  if (!m.checks && !s->wl_check_fail && !s->wl_check_retries && !s->wl_check_evict_ns && !(s->wl_requeue_at_ns && !m.pr) && !s->adm_check_end_ns)
    return KB_OK;
  if (!m.checks) return fail(h, KB_ERR_INVALID, "admission checks: the tables need wl_check_ns");
  if (!m.replay) return fail(h, KB_ERR_INVALID, "admission checks: the tables need adm_wl");
  if (m.decay) return fail(h, KB_ERR_UNSUPPORTED, "admission checks with afs decay: a workload with checks never makes the Pending -> Admitted transition that updates consumed usage");
  if (s->check_backoff_base_s <= 0 || s->check_backoff_max_s < 0 || s->check_backoff_limit < 0)
    return fail(h, KB_ERR_INVALID, "admission checks: backoff base <= 0, max < 0 or limit < 0");
  i64 longest = 0;  // the longest WaitTime of attempts 1..limit (constant once capped: a base of >= 1 s gets there in < 64 doublings)
  for (int k = 1; k <= std::min(s->check_backoff_limit, 64); k++)
    longest = std::max(longest, kb_check_wait_ns(k, s->check_backoff_base_s, s->check_backoff_max_s));
  if (longest >= 10000ll * 1000000000ll)
    return fail(h, KB_ERR_UNSUPPORTED, "admission checks: a reachable backoff of 10,000 s or more is random in the reference (jitter)");
  for (int w = 0; w < s->n_wl; w++) {
    if (s->wl_check_ns[w] < 0 || (s->wl_check_fail && s->wl_check_fail[w] < 0) || (s->wl_check_retries && s->wl_check_retries[w] < 0))
      return fail(h, KB_ERR_INVALID, "admission checks: a negative delay, fail count or retry count");
    if (int32_t rc = check_requeue_at(h, s, held, w, "admission checks")) return rc;
  }
  if (s->adm_check_end_ns)
    for (int a = 0; a < s->n_adm; a++) {
      if (s->adm_check_end_ns[a] == INT64_MIN) continue;
      if (s->adm_check_end_ns[a] <= s->now_ns) return fail(h, KB_ERR_INVALID, "admission checks: adm_check_end_ns at or before now_ns");
      if (m.lat && s->adm_evict_end_ns && s->adm_evicted && s->adm_evicted[a])  // one end time per row
        return fail(h, KB_ERR_INVALID, "admission checks: a row with both an eviction under way (adm_evict_end_ns) and a check under way");
    }
  return KB_OK;
}
static int32_t check_pods_ready(kb_handle *h, const kb_snapshot *s, const DrainMode &m, HeldRecords &held) {
  if (!m.pr && !s->wl_pods_ready_fail && !s->wl_pods_ready_count && !s->wl_pods_ready_evict_ns && !s->adm_admitted_ns) return KB_OK;
  if (!m.pr) return fail(h, KB_ERR_INVALID, "pods ready: the tables need wl_pods_ready_ns");
  if (!m.replay) return fail(h, KB_ERR_INVALID, "pods ready: the tables need adm_wl");
  if (s->pods_ready_timeout_ns <= 0) return fail(h, KB_ERR_INVALID, "pods ready: timeout <= 0");
  if (s->pods_ready_backoff_base_s < 0 || s->pods_ready_backoff_max_s < 0 || s->pods_ready_backoff_limit < -1)
    return fail(h, KB_ERR_INVALID, "pods ready: backoff base < 0, max < 0 or limit < -1");
  if (s->pods_ready_requeue_creation != 0 && s->pods_ready_requeue_creation != 1)
    return fail(h, KB_ERR_INVALID, "pods ready: pods_ready_requeue_creation is neither 0 (Eviction) nor 1 (Creation)");
  for (int w = 0; w < s->n_wl; w++) {
    if (s->wl_pods_ready_ns[w] < 0 || (s->wl_pods_ready_fail && s->wl_pods_ready_fail[w] < 0) ||
        (s->wl_pods_ready_count && s->wl_pods_ready_count[w] < 0))
      return fail(h, KB_ERR_INVALID, "pods ready: a negative delay, fail count or requeue count");
    if (s->wl_pods_ready_evict_ns && s->wl_pods_ready_evict_ns[w] != INT64_MIN) {
      if (held[w]) return fail(h, KB_ERR_INVALID, "pods ready: wl_pods_ready_evict_ns on a record that holds quota (adm_wl)");
      if (s->wl_check_evict_ns && s->wl_check_evict_ns[w] != INT64_MIN)
        return fail(h, KB_ERR_INVALID, "pods ready: a record with both wl_pods_ready_evict_ns and wl_check_evict_ns (one Evicted condition)");
    }
    if (!m.checks)  // the admission checks check it otherwise
      if (int32_t rc = check_requeue_at(h, s, held, w, "pods ready")) return rc;
  }
  if (s->adm_admitted_ns)
    for (int a = 0; a < s->n_adm; a++) {
      if (s->adm_admitted_ns[a] == INT64_MIN) continue;
      if (s->adm_admitted_ns[a] > s->now_ns) return fail(h, KB_ERR_INVALID, "pods ready: adm_admitted_ns after now_ns");
      if (s->adm_check_end_ns && s->adm_check_end_ns[a] != INT64_MIN)
        return fail(h, KB_ERR_INVALID, "pods ready: adm_admitted_ns on a row whose checks run (adm_check_end_ns)");
      if (m.lat && s->adm_evict_end_ns && s->adm_evicted && s->adm_evicted[a])
        return fail(h, KB_ERR_INVALID, "pods ready: adm_admitted_ns on a row whose eviction is under way (adm_evict_end_ns)");
    }
  return KB_OK;
}
static int32_t check_max_exec(kb_handle *h, const kb_snapshot *s, const DrainMode &m, HeldRecords &) {
  if (!m.mx && !s->wl_exec_acc_s && !s->adm_exec_since_ns) return KB_OK;
  if (!m.mx) return fail(h, KB_ERR_INVALID, "max exec: the tables need wl_max_exec_s");
  if (!m.replay) return fail(h, KB_ERR_INVALID, "max exec: the tables need adm_wl");
  for (int w = 0; w < s->n_wl; w++) {
    if (s->wl_max_exec_s[w] < 0) return fail(h, KB_ERR_INVALID, "max exec: wl_max_exec_s < 0");
    if (s->wl_exec_acc_s && s->wl_exec_acc_s[w] < -1) return fail(h, KB_ERR_INVALID, "max exec: wl_exec_acc_s < -1");
  }
  if (s->n_adm > 0 && !s->adm_exec_since_ns) return fail(h, KB_ERR_INVALID, "max exec: adm_exec_since_ns is NULL while n_adm > 0");
  for (int a = 0; a < s->n_adm; a++) {
    const i64 A = s->adm_exec_since_ns[a];
    const bool chk = m.checks && s->adm_check_end_ns && s->adm_check_end_ns[a] != INT64_MIN;
    if (A == INT64_MIN && !chk) return fail(h, KB_ERR_INVALID, "max exec: adm_exec_since_ns missing on a row whose checks do not run");
    if (A != INT64_MIN && chk) return fail(h, KB_ERR_INVALID, "max exec: adm_exec_since_ns set on a row whose checks run (adm_check_end_ns)");
    if (A > s->now_ns) return fail(h, KB_ERR_INVALID, "max exec: adm_exec_since_ns after now_ns");
    if (m.pr && s->adm_admitted_ns && s->adm_admitted_ns[a] != INT64_MIN && s->adm_admitted_ns[a] != A)
      return fail(h, KB_ERR_INVALID, "max exec: adm_exec_since_ns differs from adm_admitted_ns");
  }
  return KB_OK;
}
static int32_t check_quota(kb_handle *h, const kb_snapshot *s, const DrainMode &m, HeldRecords &) {
  if (s->n_quota_change < 0) return fail(h, KB_ERR_INVALID, "quota changes: n_quota_change < 0");
  if (s->n_quota_change == 0) return KB_OK;
  if (!s->qc_ns || !s->qc_node || !s->qc_nominal || !s->qc_borrow_limit || !s->qc_lend_limit)
    return fail(h, KB_ERR_INVALID, "quota changes: a NULL table with n_quota_change > 0");
  const int Q = s->n_cq, R = s->n_resource, FR = s->n_flavor * R;
  std::vector<uint8_t> covered((size_t)Q * FR, 0);  // the cells a ClusterQueue's resource groups cover
  for (int q = 0; q < Q; q++)
    for (int g = s->cq_rg_start[q]; g < s->cq_rg_start[q + 1]; g++)
      for (int k = s->rg_flavor_start[g]; k < s->rg_flavor_start[g + 1]; k++)
        for (int r = 0; r < R; r++)
          if (s->rg_res_mask[g] & (1u << r)) covered[(size_t)q * FR + (size_t)s->rg_flavors[k] * R + r] = 1;
  for (int i = 0; i < m.n_qc; i++) {
    if (s->qc_ns[i] <= s->now_ns) return fail(h, KB_ERR_INVALID, "quota changes: qc_ns at or before now_ns");
    if (i > 0 && s->qc_ns[i] < s->qc_ns[i - 1]) return fail(h, KB_ERR_INVALID, "quota changes: qc_ns decreasing");
    const int n = s->qc_node[i];
    if (n < 0 || n >= Q + s->n_cohort) return fail(h, KB_ERR_INVALID, "quota changes: qc_node out of range");
    for (int c = 0; c < FR; c++) {
      const size_t k = (size_t)i * FR + c;
      if (s->qc_nominal[k] < 0 || s->qc_nominal[k] == KB_NO_LIMIT) return fail(h, KB_ERR_INVALID, "quota changes: a negative nominal or KB_NO_LIMIT in a nominal row");
      if (s->qc_borrow_limit[k] < 0 || s->qc_lend_limit[k] < 0) return fail(h, KB_ERR_INVALID, "quota changes: a negative limit");
      const size_t o = (size_t)n * FR + c;
      if (n < Q && !covered[o] && (s->qc_nominal[k] != s->nominal[o] || s->qc_borrow_limit[k] != s->borrow_limit[o] || s->qc_lend_limit[k] != s->lend_limit[o]))
        return fail(h, KB_ERR_INVALID, "quota changes: a ClusterQueue cell its resource groups do not cover");
    }
  }
  return KB_OK;
}
static int32_t check_active(kb_handle *h, const kb_snapshot *s, const DrainMode &m, HeldRecords &held) {
  if (s->n_active_change < 0) return fail(h, KB_ERR_INVALID, "active changes: n_active_change < 0");
  if (s->n_active_change > 0 && (!s->ac_ns || !s->ac_wl || !s->ac_active))
    return fail(h, KB_ERR_INVALID, "active changes: a NULL table with n_active_change > 0");
  if (!m.blk) return KB_OK;
  if (!m.replay) return fail(h, KB_ERR_INVALID, "active changes: the tables need adm_wl");
  for (int i = 0; i < m.n_ac; i++) {
    if (s->ac_ns[i] <= s->now_ns) return fail(h, KB_ERR_INVALID, "active changes: ac_ns at or before now_ns");
    if (i > 0 && s->ac_ns[i] < s->ac_ns[i - 1]) return fail(h, KB_ERR_INVALID, "active changes: ac_ns decreasing");
    const int w = s->ac_wl[i];
    if (w < 0 || w >= s->n_wl) return fail(h, KB_ERR_INVALID, "active changes: ac_wl out of range");
    if (s->ac_active[i] > 1) return fail(h, KB_ERR_INVALID, "active changes: ac_active neither 0 nor 1");
    if (s->wl_create_ns && s->ac_ns[i] <= s->wl_create_ns[w]) return fail(h, KB_ERR_INVALID, "active changes: an edit at or before its record's wl_create_ns");
  }
  if (s->wl_inactive)
    for (int w = 0; w < s->n_wl; w++) {
      if (s->wl_inactive[w] > KB_DR_USER) return fail(h, KB_ERR_INVALID, "active changes: wl_inactive above 4");
      if (!s->wl_inactive[w]) continue;
      if (held[w]) return fail(h, KB_ERR_INVALID, "active changes: an inactive start record that adm_wl names");
      if (s->wl_create_ns && s->wl_create_ns[w] > s->now_ns) return fail(h, KB_ERR_INVALID, "active changes: an inactive start record created after now_ns");
    }
  return KB_OK;
}
// restated by kueue_b200/drain.py check_reclaims
static int32_t check_reclaim(kb_handle *h, const kb_snapshot *s, const DrainMode &m, HeldRecords &) {
  if (!m.rcl && !s->rc_after_ns && !s->rc_ps && !s->rc_remaining && !s->rc_sched_hash && !s->ps_adm_flavor && !s->ps_adm_count && !s->ps_adm_usage &&
      !s->adm_run_start_ns)
    return KB_OK;
  const int W = s->n_wl, R = s->n_resource;
  if (!m.replay) return fail(h, KB_ERR_INVALID, "reclaim steps: the tables need adm_wl");
  if (!m.rcl || (s->n_reclaim > 0 && (!s->rc_after_ns || !s->rc_ps || !s->rc_remaining)))
    return fail(h, KB_ERR_INVALID, "reclaim steps: a NULL table (wl_rc_start, rc_after_ns, rc_ps, rc_remaining)");
  if (s->n_reclaim < 0 || s->wl_rc_start[0] != 0 || s->wl_rc_start[W] != s->n_reclaim)
    return fail(h, KB_ERR_INVALID, "reclaim steps: wl_rc_start is not a CSR of the steps");
  for (int w = 0; w < W; w++)
    if (s->wl_rc_start[w + 1] < s->wl_rc_start[w]) return fail(h, KB_ERR_INVALID, "reclaim steps: wl_rc_start is not a CSR of the steps");
  for (int w = 0; w < W; w++)
    for (int i = s->wl_rc_start[w]; i < s->wl_rc_start[w + 1]; i++)
      if (s->rc_ps[i] < s->wl_ps_start[w] || s->rc_ps[i] >= s->wl_ps_start[w + 1]) return fail(h, KB_ERR_INVALID, "reclaim steps: rc_ps outside its record");
  for (int w = 0; w < W; w++)
    for (int i = s->wl_rc_start[w]; i < s->wl_rc_start[w + 1]; i++)
      if (s->rc_after_ns[i] <= 0 || (i > s->wl_rc_start[w] && s->rc_after_ns[i] < s->rc_after_ns[i - 1]))
        return fail(h, KB_ERR_INVALID, "reclaim steps: rc_after_ns <= 0 or decreasing within a record");
  std::vector<int32_t> last((size_t)std::max(1, s->n_podset), INT32_MAX);
  for (int i = 0; i < m.n_rc; i++) {
    const int p = s->rc_ps[i];
    if (s->rc_remaining[i] < 0 || s->rc_remaining[i] > last[p]) return fail(h, KB_ERR_INVALID, "reclaim steps: rc_remaining negative or increasing within a podset");
    last[p] = s->rc_remaining[i];
  }
  for (int p = 0; p < s->n_podset; p++)
    if (last[p] != INT32_MAX && s->ps_count[p] > 0)
      for (int r = 0; r < R; r++)
        if (s->ps_req[(size_t)p * R + r] % s->ps_count[p] != 0) return fail(h, KB_ERR_INVALID, "reclaim steps: ps_req of a podset with steps not divisible by its ps_count");
  if (s->flags & KB_F_PARTIAL_ADMISSION)
    for (int w = 0; w < W; w++)
      if (s->wl_rc_start[w + 1] > s->wl_rc_start[w])
        for (int p = s->wl_ps_start[w]; p < s->wl_ps_start[w + 1]; p++)
          if (s->ps_min_count[p] >= 0) return fail(h, KB_ERR_UNSUPPORTED, "reclaim steps: steps on a record that can be partially admitted");
  if (s->adm_run_start_ns)
    for (int a = 0; a < s->n_adm; a++) {
      const i64 S = s->adm_run_start_ns[a];
      if (S != INT64_MIN && S > s->now_ns) return fail(h, KB_ERR_INVALID, "reclaim steps: adm_run_start_ns after now_ns");
    }
  if (s->adm_run_start_ns)
    for (int a = 0; a < s->n_adm; a++) {
      const bool idle = (s->adm_evicted && s->adm_evicted[a]) || (s->adm_check_end_ns && s->adm_check_end_ns[a] != INT64_MIN) ||
                        (s->adm_admitted_ns && s->adm_admitted_ns[a] != INT64_MIN);
      if (s->adm_run_start_ns[a] != INT64_MIN && idle) return fail(h, KB_ERR_INVALID, "reclaim steps: adm_run_start_ns on a row that is not running");
    }
  bool any_row = false;
  for (int a = 0; a < s->n_adm; a++) any_row |= s->wl_rc_start[s->adm_wl[a] + 1] > s->wl_rc_start[s->adm_wl[a]];
  if (any_row && (!s->ps_adm_flavor || !s->ps_adm_count || !s->ps_adm_usage))
    return fail(h, KB_ERR_INVALID, "reclaim steps: ps_adm_* missing for a row whose record has steps");
  for (int a = 0; a < s->n_adm && any_row; a++) {
    const int w = s->adm_wl[a];
    if (s->wl_rc_start[w + 1] == s->wl_rc_start[w]) continue;
    std::map<int, i64> want, have;
    for (int p = s->wl_ps_start[w]; p < s->wl_ps_start[w + 1]; p++)
      for (int r = 0; r < R; r++) {
        const int f = s->ps_adm_flavor[(size_t)p * R + r];
        const i64 u = s->ps_adm_usage[(size_t)p * R + r];
        const int n = s->ps_adm_count[p];
        if (f < -1 || f >= s->n_flavor || n < 0 || u < 0) return fail(h, KB_ERR_INVALID, "reclaim steps: ps_adm_* out of range");
        if (f >= 0 && n > 0) want[f * R + r] += u / n * std::min(s->ps_count[p], n);
      }
    for (int c = s->adm_use_start[a]; c < s->adm_use_start[a + 1]; c++) have[s->adm_use_fr[c]] += s->adm_use_qty[c];
    for (auto *mp : {&want, &have})
      for (auto it = mp->begin(); it != mp->end();) it = it->second == 0 ? mp->erase(it) : std::next(it);
    if (want != have) return fail(h, KB_ERR_INVALID, "reclaim steps: a row's ps_adm_* do not add up to its adm_use cells");
  }
  return KB_OK;
}
static int32_t drain_validate(kb_handle *h, const kb_snapshot *s, const DrainMode &m, HeldRecords &held) {
  using Check = int32_t (*)(kb_handle *, const kb_snapshot *, const DrainMode &, HeldRecords &);
  held.assign((size_t)std::max(1, s->n_wl), 0);
  for (Check c : {check_replay, check_events, check_latency, check_decay, check_sticky, check_checks, check_pods_ready, check_max_exec,
                  check_quota, check_active, check_reclaim})
    if (int32_t rc = c(h, s, m, held)) return rc;
  return KB_OK;
}

// ---- host precomputation: the tables the device starts from
// n values of a caller's table, or n times v where it passes none
template <class T, class S> static std::vector<T> drain_table_or(const S *src, size_t n, T v) {
  return src ? std::vector<T>(src, src + n) : std::vector<T>(n, v);
}
// the snapshot's rows at the start of an event drain (kb_drain.cuh DrainFin): finish column, phase, evicting byte, and
// per record the PodsReady time of a ready attempt under way.  An eviction under way holds its end time (an evicted
// workload never finishes); a row whose checks run, its verdict time; a row Admitted without PodsReady, its attempt
// (kb_pr_attempt; no failure is used until a timeout is applied); a row with an Admitted time and a limit, not evicting,
// the effective deadline max(D, A, now_ns) where it comes first (kb_exec_clip).
struct DrainRowStart {
  std::vector<i64> finish, pr_at;
  std::vector<uint8_t> phase, evicting;  // evicting: empty unless eviction latency with adm_evict_end_ns
  bool phased;                           // some row starts in another phase than KB_PH_RUN, or may
};
static DrainRowStart drain_row_start(const kb_snapshot *s, const DrainMode &m) {
  const int n = s->n_adm;
  DrainRowStart o;
  o.finish = drain_table_or<i64>(s->adm_finish_ns, (size_t)n, INT64_MAX);
  o.phase.assign((size_t)n, KB_PH_RUN);
  if (m.pr) o.pr_at.assign((size_t)s->n_wl, INT64_MIN);
  if (m.lat && s->adm_evict_end_ns) {
    o.evicting.assign((size_t)n, 0);
    for (int a = 0; a < n; a++)
      if (s->adm_evicted[a]) { o.finish[a] = s->adm_evict_end_ns[a]; o.evicting[a] = 1; }
  }
  o.phased = (m.checks && s->adm_check_end_ns) || (m.pr && s->adm_admitted_ns) || (m.mx && n > 0);
  for (int a = 0; a < n && o.phased; a++) {
    DrainFin f{o.finish[a], KB_PH_RUN};
    if (m.checks && s->adm_check_end_ns && s->adm_check_end_ns[a] != INT64_MIN) f = {s->adm_check_end_ns[a], KB_PH_CHECK};
    const int w = m.replay ? s->adm_wl[a] : -1;
    if (m.pr && s->adm_admitted_ns && s->adm_admitted_ns[a] != INT64_MIN) {
      const i64 t0 = s->adm_admitted_ns[a], d = s->wl_pods_ready_ns[w];
      f = kb_pr_attempt(t0, d, s->wl_pods_ready_fail && s->wl_pods_ready_fail[w] > 0, s->pods_ready_timeout_ns, s->wl_run_ns ? s->wl_run_ns[w] : -1);
      if (f.ph == KB_PH_RUN) o.pr_at[w] = drain_sat_add(t0, d);
    }
    if (m.mx && s->adm_exec_since_ns[a] != INT64_MIN && (o.evicting.empty() || !o.evicting[a]))
      f = kb_exec_clip(f, s->adm_exec_since_ns[a], s->wl_max_exec_s[w], s->wl_exec_acc_s ? s->wl_exec_acc_s[w] : -1, s->now_ns);
    o.finish[a] = f.fin; o.phase[a] = f.ph;
  }
  return o;
}

// reclaim steps: the snapshot's running rows with steps start at their run start (a ready PodsReady attempt under way:
// at its PodsReady time), and their records' PodSetAssignments
struct DrainRcStart { std::vector<i64> next, use; std::vector<int32_t> cur, cnt; std::vector<int8_t> fl; };
static DrainRcStart drain_reclaim_start(const kb_snapshot *s, const DrainMode &m, const std::vector<i64> &pr_at) {
  const int R = s->n_resource;
  const size_t Pz = (size_t)std::max(1, s->n_podset), An = (size_t)std::max(1, s->n_adm);
  DrainRcStart o;
  o.next.assign(An, INT64_MAX); o.cur.assign(An, 0);
  o.fl.assign(Pz * R, -1); o.cnt.assign(Pz, 0); o.use.assign(Pz * R, 0);
  for (int a = 0; a < s->n_adm; a++) {
    const int w = s->adm_wl[a], i = s->wl_rc_start[w];
    if (i == s->wl_rc_start[w + 1]) continue;
    const size_t p0 = s->wl_ps_start[w], p1 = s->wl_ps_start[w + 1];
    memcpy(&o.fl[p0 * R], s->ps_adm_flavor + p0 * R, (p1 - p0) * R);
    memcpy(&o.cnt[p0], s->ps_adm_count + p0, (p1 - p0) * 4);
    memcpy(&o.use[p0 * R], s->ps_adm_usage + p0 * R, (p1 - p0) * R * 8);
    i64 S = s->adm_run_start_ns ? s->adm_run_start_ns[a] : INT64_MIN;
    if (S == INT64_MIN && m.pr && s->adm_admitted_ns && s->adm_admitted_ns[a] != INT64_MIN) S = pr_at[w];
    if (S == INT64_MIN) continue;
    o.cur[a] = i;
    o.next[a] = drain_sat_add(S, s->rc_after_ns[i]);
  }
  return o;
}

// AdmissionFairSharing: queue segments, one per LocalQueue of a ClusterQueue with cq_afs set and one per other
// ClusterQueue, numbered ClusterQueue-major; the initial usage of every LocalQueue (kb_drain.cuh afs_lq_usage); with
// decay, the initial admitted usage of every LocalQueue (the cells of the snapshot's rows)
struct DrainAfs { std::vector<int32_t> seg_start, lq_seg, seg_lq, afs_cqs; std::vector<double> lq_usage; std::vector<i64> lq_adm; };
static int32_t drain_afs_queues(kb_handle *h, const kb_snapshot *s, const DrainMode &m, DrainAfs &o) {
  const int Q = s->n_cq, R = s->n_resource, L = s->n_lq;
  std::vector<int32_t> lq_first((size_t)Q + 1, 0);
  for (int l = 0; l < L; l++) lq_first[s->lq_cq[l] + 1]++;
  for (int q = 0; q < Q; q++) lq_first[q + 1] += lq_first[q];
  o.seg_start.resize((size_t)Q + 1); o.lq_seg.assign((size_t)std::max(1, L), -1); o.lq_usage.assign((size_t)std::max(1, L), 0.0);
  for (int q = 0; q < Q; q++) {
    o.seg_start[q] = (int32_t)o.seg_lq.size();
    if (!s->cq_afs[q]) { o.seg_lq.push_back(-1); continue; }
    o.afs_cqs.push_back(q);
    for (int l = lq_first[q]; l < lq_first[q + 1]; l++) {
      o.lq_seg[l] = (int32_t)o.seg_lq.size(); o.seg_lq.push_back(l);
      const size_t k = (size_t)l * R;
      if (!afs_lq_usage((const i64 *)s->lq_consumed + k, s->lq_consumed_scale + k, s->lq_penalty ? (const i64 *)s->lq_penalty + k : nullptr, s->afs_res_weight,
                        s->lq_weight[l], R, &o.lq_usage[l]))
        return fail(h, KB_ERR_UNSUPPORTED, "afs: consumed usage + entry penalty of a LocalQueue overflows int64");
    }
  }
  o.seg_start[Q] = (int32_t)o.seg_lq.size();
  if (o.seg_lq.empty()) o.seg_lq.push_back(-1);
  if (m.decay) {
    o.lq_adm.assign((size_t)std::max(1, L) * R, 0);
    for (int a = 0; a < s->n_adm; a++)
      if (s->adm_lq[a] >= 0)
        for (int c = s->adm_use_start[a]; c < s->adm_use_start[a + 1]; c++) o.lq_adm[(size_t)s->adm_lq[a] * R + s->adm_use_fr[c] % R] += s->adm_use_qty[c];
  }
  return KB_OK;
}

// NoFit classes (event mode with arrivals and hashes): a dense id per (BestEffortFIFO ClusterQueue, known hash), the
// hashes reclaim steps set included; n = 0: none
struct DrainClasses { int n = 0; std::vector<int32_t> wl_class, cq_class_start, rc_class; };
static DrainClasses drain_nofit_classes(const kb_snapshot *s, const DrainMode &m) {
  const int W = s->n_wl, Q = s->n_cq;
  DrainClasses o;
  if (!m.events || !s->wl_create_ns || !s->wl_sched_hash) return o;
  std::vector<std::pair<std::pair<int32_t, int64_t>, int32_t>> cls;  // a value >= W names step value - W
  for (int w = 0; w < W; w++)
    if (s->wl_sched_hash[w] != 0 && s->cq_strategy[s->wl_cq[w]] != KB_QUEUE_STRICT_FIFO) cls.push_back({{s->wl_cq[w], s->wl_sched_hash[w]}, w});
  if (m.rcl && s->rc_sched_hash)
    for (int w = 0; w < W; w++)
      for (int i = s->wl_rc_start[w]; i < s->wl_rc_start[w + 1]; i++)
        if (s->rc_sched_hash[i] != 0 && s->cq_strategy[s->wl_cq[w]] != KB_QUEUE_STRICT_FIFO) cls.push_back({{s->wl_cq[w], s->rc_sched_hash[i]}, W + i});
  std::sort(cls.begin(), cls.end());
  o.wl_class.assign((size_t)W, -1); o.cq_class_start.assign((size_t)Q + 1, 0); o.rc_class.assign((size_t)std::max(1, m.n_rc), -1);
  for (size_t i = 0; i < cls.size(); i++) {
    if (i > 0 && cls[i].first != cls[i - 1].first) o.n++;
    if (cls[i].second < W) o.wl_class[cls[i].second] = o.n;
    else o.rc_class[cls[i].second - W] = o.n;
    o.cq_class_start[cls[i].first.first + 1] = o.n + 1;
  }
  if (!cls.empty()) o.n++;
  for (int q = 0; q < Q; q++) o.cq_class_start[q + 1] = std::max(o.cq_class_start[q + 1], o.cq_class_start[q]);
  return o;
}

// byte offset of every ClusterQueue's generation in the static tree blocks, -1 = not in a tree
static std::vector<int32_t> drain_blob_gen(const kb_handle *h, int Q) {
  std::vector<int32_t> off((size_t)std::max(1, Q), -1);
  for (int q = 0; q < Q; q++) {
    const int slot = h->root_slot[q];
    if (slot < h->D.nLone) continue;
    const int tr = slot - h->D.nLone, b0 = h->tree_blob_off[tr];
    const TreeBlobHdr *BH = (const TreeBlobHdr *)(h->tree_blob.data() + b0);
    off[q] = b0 + BH->gen + 8 * h->local_idx[q];
  }
  return off;
}

// quota changes: the edits that change nothing (root -1), the root slot and the cohort tree of every other one (the rows
// change only through the edits, in table order, so the rows an edit meets are known here), the next edit of the same
// tree, the ClusterQueues of every root, the place of every ClusterQueue's generation in the static tree blocks
struct DrainQuota { std::vector<int32_t> root, tree, tree_next, cq_start, cq, blob_gen; };
static DrainQuota drain_quota_prep(const kb_handle *h, const kb_snapshot *s, const DrainMode &m) {
  const int Q = s->n_cq, FR = s->n_flavor * s->n_resource, QN = Q + s->n_cohort, NQC = m.n_qc;
  const DevSnap &D = h->D;
  DrainQuota o;
  std::vector<i64> nom(s->nominal, s->nominal + (size_t)QN * FR), bl(s->borrow_limit, s->borrow_limit + (size_t)QN * FR),
      ll(s->lend_limit, s->lend_limit + (size_t)QN * FR);  // the rows each edit meets
  o.root.assign((size_t)NQC, -1); o.tree.assign((size_t)NQC, -1);
  for (int i = 0; i < NQC; i++) {
    const int n = s->qc_node[i];
    const size_t r = (size_t)n * FR, k = (size_t)i * FR, b = (size_t)FR * 8;
    if (!memcmp(&nom[r], s->qc_nominal + k, b) && !memcmp(&bl[r], s->qc_borrow_limit + k, b) && !memcmp(&ll[r], s->qc_lend_limit + k, b)) continue;
    memcpy(&nom[r], s->qc_nominal + k, b); memcpy(&bl[r], s->qc_borrow_limit + k, b); memcpy(&ll[r], s->qc_lend_limit + k, b);
    o.root[i] = h->root_slot[n];
    if (D.tl_subtree && h->root_slot[n] >= D.nLone) o.tree[i] = h->root_slot[n] - D.nLone;  // lone ClusterQueues come first
  }
  o.tree_next.assign((size_t)NQC, NQC);
  std::vector<int32_t> later((size_t)std::max(1, D.nTrees), NQC);
  for (int i = NQC - 1; i >= 0; i--)
    if (o.tree[i] >= 0) { o.tree_next[i] = later[o.tree[i]]; later[o.tree[i]] = i; }
  o.cq_start.assign(h->root_cq_start.begin(), h->root_cq_start.end());
  o.cq.assign((size_t)std::max(1, Q), 0);
  std::vector<int32_t> fill(o.cq_start.begin(), o.cq_start.end() - 1);
  for (int q = 0; q < Q; q++) o.cq[fill[h->root_slot[q]]++] = q;
  o.blob_gen = drain_blob_gen(h, Q);
  return o;
}

// deactivation / reactivation: each edit's previous and next edit of the same record (-1 / n_ac = none)
static void drain_active_links(const kb_snapshot *s, const DrainMode &m, std::vector<int32_t> &next, std::vector<int32_t> &prev) {
  const int NAC = m.n_ac;
  next.assign((size_t)std::max(1, NAC), NAC); prev.assign((size_t)std::max(1, NAC), -1);
  std::vector<int32_t> last((size_t)std::max(1, s->n_wl), -1);
  for (int i = 0; i < NAC; i++) {
    const int w = s->ac_wl[i];
    if (last[w] >= 0) { prev[i] = last[w]; next[last[w]] = i; }
    last[w] = i;
  }
}

// ---- the boundary counters kb_drain_out reports: each row names its slot in DrainDev::counters, how the slot counts,
// the drain's total and per-cycle array, and whether the drain's blocks write it.  A cleared slot is zeroed every
// boundary (kb_run_drain's memsets), a cumulative one counts since the start of the drain (the host differences it), a
// range is the [lo, hi) pair of slots idx, idx + 1 of the edits a boundary applied.
enum { DC_CLEARED, DC_CUMULATIVE, DC_RANGE };
struct DrainCounter { int idx, kind; int64_t *total; int32_t *cycle; bool on; uint32_t seen; };
static std::vector<DrainCounter> drain_counters(kb_drain_out *out, const DrainMode &m) {
  return {{KB_DC_FINISHED, DC_CLEARED, &out->n_finished, out->cycle_finished, m.events, 0},
          {KB_DC_ARRIVED, DC_CLEARED, &out->n_arrived, out->cycle_arrived, m.events, 0},
          {KB_DC_EVICT_DONE, DC_CLEARED, &out->n_evict_done, out->cycle_evict_done, m.lat, 0},
          {KB_DC_CHECK_READY, DC_CUMULATIVE, &out->n_check_ready, nullptr, m.checks, 0},
          {KB_DC_CHECK_RETRY, DC_CUMULATIVE, &out->n_check_retry, out->cycle_check_retry, m.checks, 0},
          {KB_DC_CHECK_REJECTED, DC_CUMULATIVE, &out->n_check_rejected, out->cycle_check_rejected, m.checks, 0},
          {KB_DC_PR_TIMEOUT, DC_CUMULATIVE, &out->n_pods_ready_timeout, out->cycle_pods_ready_timeout, m.pr, 0},
          {KB_DC_PR_DEACTIVATED, DC_CUMULATIVE, &out->n_pods_ready_deactivated, out->cycle_pods_ready_deactivated, m.pr, 0},
          {KB_DC_EXEC_DEACTIVATED, DC_CUMULATIVE, &out->n_max_exec_deactivated, out->cycle_max_exec_deactivated, m.mx, 0},
          {KB_DC_QC_LO, DC_RANGE, &out->n_quota_changes, out->cycle_quota_changes, m.quota, 0},
          {KB_DC_STOPPED, DC_CUMULATIVE, &out->n_stopped, out->cycle_stopped, m.act, 0},
          {KB_DC_RESUMED, DC_CUMULATIVE, &out->n_resumed, out->cycle_resumed, m.act, 0},
          {KB_DC_RECLAIMS, DC_CUMULATIVE, &out->n_reclaims, out->cycle_reclaims, m.rcl, 0}};
}

// ---- one kb_run_drain call (the counterpart of kueue_b200/drain.py _Drain): the mode, the host tables of the plan,
// the device buffers, and the state of the boundary loop
struct DrainRun {
  kb_handle *h; const kb_snapshot *s; kb_drain_out *out;
  DrainMode m;
  std::vector<DrainCounter> counters;
  HeldRecords held;  // held[w]: an admitted row names record w (drain_validate)
  int Q, W, R, FR, Hcap, max_cycles;
  // plan
  int S = 0, L = 0;  // queue segments, LocalQueues
  DrainAfs afs; DrainClasses cls; DrainQuota qc; DrainRowStart rows; DrainRcStart rc;
  std::vector<int32_t> ac_next, ac_prev, rc_blob_gen;
  std::vector<i64> qts, requeue_at, pr_none; std::vector<int32_t> fails, retries, pr_fails, pr_counts, exec_acc;  // records at the start
  size_t Acap = 0, AUcap = 0, sort_bytes = 0, scan_bytes = 0, trace_cap = 0, nR = 1;
  // device buffers
  DrainDev X{};
  AdmRows other{};  // compaction: the other half of the admitted rows' double buffer
  u64 *keys[2] = {}, *arr_keys[2] = {}; int32_t *vals[2] = {}, *arr_vals[2] = {}, *q_count = nullptr;
  char *sort_tmp = nullptr, *scan_tmp = nullptr;
  i64 *create = nullptr; uint8_t *inactive = nullptr;
  // boundary loop
  int n_used = 1, n_live = 0, A_cur = 0, AU_cur = 0, cyc = 0, jumps = 0;
  i64 t = 0, step = 1;
  double gpu_ms = 0;
  float kms[KB_N_KERNELS] = {};  // per-kernel times summed over the cycles (kb_set_profile)
  cudaEvent_t ev_r[2] = {nullptr, nullptr};  // around a re-sort (admission checks, PodsReady)
  bool resort_timed = false;
  ~DrainRun() { for (cudaEvent_t e : ev_r) if (e) cudaEventDestroy(e); }
};
static constexpr int DRAIN_TB = 256;
static int drain_blocks(long long n) { return (int)((n + DRAIN_TB - 1) / DRAIN_TB); }

// the DevSnap's admitted tables are the first nine columns of the current half
static AdmRows drain_snap_rows(const DevSnap &D) {
  AdmRows r{};
  r.cq = const_cast<int32_t *>(D.adm_cq); r.priority = const_cast<int32_t *>(D.adm_priority); r.ts = const_cast<i64 *>(D.adm_ts);
  r.qr_ts = const_cast<i64 *>(D.adm_qr_ts); r.uid = const_cast<i64 *>(D.adm_uid); r.evicted = const_cast<uint8_t *>(D.adm_evicted);
  r.use_start = const_cast<int32_t *>(D.adm_use_start); r.use_fr = const_cast<int32_t *>(D.adm_use_fr); r.use_qty = const_cast<i64 *>(D.adm_use_qty);
  return r;
}
static void drain_point_snap(DevSnap &D, const AdmRows &r) {
  D.adm_cq = r.cq; D.adm_priority = r.priority; D.adm_ts = r.ts; D.adm_qr_ts = r.qr_ts; D.adm_uid = r.uid;
  D.adm_evicted = r.evicted; D.adm_use_start = r.use_start; D.adm_use_fr = r.use_fr; D.adm_use_qty = r.use_qty;
}
// the columns of one half of the admitted rows its blocks need; base: the nine the first half borrows from the DevSnap
static void drain_carve_rows(Arena &a, AdmRows &r, const DrainMode &m, size_t Acap, size_t AUcap, bool base) {
  if (base) {
    r.cq = a.take<int32_t>(Acap); r.priority = a.take<int32_t>(Acap); r.ts = a.take<i64>(Acap);
    r.qr_ts = a.take<i64>(Acap); r.uid = a.take<i64>(Acap); r.evicted = a.take<uint8_t>(Acap);
    r.use_start = a.take<int32_t>(Acap + 1); r.use_fr = a.take<int32_t>(AUcap); r.use_qty = a.take<i64>(AUcap);
  }
  if (m.replay || m.events) r.wl = a.take<int32_t>(Acap);
  if (m.events) r.finish = a.take<i64>(Acap);
  if (m.decay) r.lq = a.take<int32_t>(Acap);
  if (m.lat) r.evicting = a.take<uint8_t>(Acap);
  if (m.requeue || m.mx) r.phase = a.take<uint8_t>(Acap);
  if (m.mx) r.since = a.take<i64>(Acap);
  if (m.rcl) { r.rc_next = a.take<i64>(Acap); r.rc_cur = a.take<int32_t>(Acap); }
}

// after upload_impl: whether rows can die, the host tables, the sizes of the buffers
static int32_t drain_plan(DrainRun &r) {
  kb_handle *h = r.h; const kb_snapshot *s = r.s; DrainMode &m = r.m;
  // evictions happen only where a target search can: without a preemption policy adm_wl only keeps its records queued-out
  m.evict = m.replay && h->preempt_possible;
  m.compact = m.evict || m.events;
  r.S = r.Q;
  if (m.afs) {
    r.L = s->n_lq;
    if (int32_t rc = drain_afs_queues(h, s, m, r.afs)) return rc;
    r.S = r.afs.seg_start[r.Q];
  }
  cub::DoubleBuffer<u64> dk(nullptr, nullptr); cub::DoubleBuffer<int32_t> dv(nullptr, nullptr);
  cub::DeviceRadixSort::SortPairs(nullptr, r.sort_bytes, dk, dv, r.W, 0, 64, h->stream);
  r.sort_bytes += 256;
  r.trace_cap = r.out->trace_wl && r.out->trace_decision ? (size_t)std::max<int64_t>(0, r.out->trace_capacity) : 0;
  r.Acap = (size_t)s->n_adm + h->drain_extra_adm; r.AUcap = (size_t)s->n_adm_use + h->drain_extra_au;  // see drain_boundary
  if (m.compact) cub::DeviceScan::ExclusiveSum(nullptr, r.scan_bytes, (int32_t *)nullptr, (int32_t *)nullptr, (int)r.Acap + 1, h->stream);
  r.nR = (size_t)std::max(1, h->D.nRoots);
  r.cls = drain_nofit_classes(s, m);
  if (m.events) r.rows = drain_row_start(s, m);
  if (m.quota) r.qc = drain_quota_prep(h, s, m);
  if (m.act) drain_active_links(s, m, r.ac_next, r.ac_prev);
  if (m.rcl) { r.rc = drain_reclaim_start(s, m, r.rows.pr_at); r.rc_blob_gen = drain_blob_gen(h, r.Q); }
  // the counter slots [0, n_used) a boundary reads back: the heads; with compaction the evictions, rows, cells and
  // capacity flag; the end flag, re-sort stamp and execution-time status of their blocks; every reported counter
  r.n_used = m.compact ? KB_DC_FULL + 1 : 1;
  if (m.events) r.n_used = std::max(r.n_used, KB_DC_END + 1);
  if (m.requeue) r.n_used = std::max(r.n_used, KB_DC_RESORT + 1);
  if (m.mx) r.n_used = std::max(r.n_used, KB_DC_EXEC_STATUS + 1);
  for (const DrainCounter &c : r.counters)
    if (c.on) r.n_used = std::max(r.n_used, c.idx + (c.kind == DC_RANGE ? 2 : 1));
  return KB_OK;
}

// every buffer of the drain, described once (Arena::carve)
static bool drain_carve(DrainRun &r) {
  const DrainMode &m = r.m;
  DrainDev &X = r.X;
  const int Q = r.Q, R = r.R, FR = r.FR, L = r.L;
  const size_t Wz = (size_t)r.W, Hz = (size_t)r.Hcap, Sz = (size_t)r.S, Lz = (size_t)std::max(1, L), LR = Lz * R, Acap = r.Acap;
  const size_t Pz = (size_t)std::max(1, r.s->n_podset), NQC = (size_t)m.n_qc, NAC = (size_t)m.n_ac, NRCz = (size_t)std::max(1, m.n_rc);
  auto layout = [&](Arena &a) {
    r.keys[0] = a.take<u64>(Wz); r.keys[1] = a.take<u64>(Wz);
    r.vals[0] = a.take<int32_t>(Wz); r.vals[1] = a.take<int32_t>(Wz);
    r.sort_tmp = a.take<char>(r.sort_bytes);
    r.q_count = a.take<int32_t>(Sz + 2);
    X.q_start = a.take<int32_t>(Sz + 2); X.cursor = a.take<int32_t>(Sz); X.wl_state = a.take<uint8_t>(Wz);
    X.first_aside = a.take<int32_t>(Sz);
    X.flag = a.take<int32_t>((size_t)Q + 2); X.pos = a.take<int32_t>((size_t)Q + 2);
    X.e_assumed = a.take<int32_t>(Hz + 2); X.e_ncells = a.take<int32_t>(Hz + 2);
    X.e_adm_off = a.take<int32_t>(Hz + 2); X.e_cell_off = a.take<int32_t>(Hz + 2);
    X.counters = a.take<int32_t>(KB_DC_RECLAIMS + 1);
    X.wl_admit_cycle = a.take<int32_t>(Wz); X.wl_evals = a.take<int32_t>(Wz); X.wl_last_decision = a.take<uint8_t>(Wz);
    if (r.trace_cap) { X.trace_wl = a.take<int32_t>(r.trace_cap); X.trace_dec = a.take<uint8_t>(r.trace_cap); }
    if (m.replay || m.events || m.sticky) { X.wl_seg = a.take<int32_t>(Wz); X.wl_pos = a.take<int32_t>(Wz); }  // sticky: the head's position
    if (m.replay || m.events) X.wl_evictions = a.take<int32_t>(Wz);
    if (m.sticky) X.cq_sticky = a.take<int32_t>((size_t)Q);
    drain_carve_rows(a, X.adm, m, Acap, r.AUcap, false);
    if (m.compact) {
      drain_carve_rows(a, r.other, m, Acap, r.AUcap, true);
      X.adm_dead = a.take<int32_t>(Acap); X.root_mark = a.take<int32_t>(r.nR);
      X.row_live = a.take<int32_t>(Acap + 1); X.row_cells = a.take<int32_t>(Acap + 1);
      X.row_new = a.take<int32_t>(Acap + 1); X.cell_new = a.take<int32_t>(Acap + 1);
      r.scan_tmp = a.take<char>(r.scan_bytes + 256);
    }
    if (m.events) {  // run times, admit / finish times, the clock, the arrival order (sorted pairs and their double
                     // buffers) and the NoFit classes
      if (r.s->wl_run_ns) X.wl_run = a.take<i64>(Wz);
      X.wl_admit_ns = a.take<i64>(Wz); X.wl_finish_ns = a.take<i64>(Wz); X.clock = a.take<i64>(4);
      if (r.s->wl_create_ns) {
        r.arr_keys[0] = a.take<u64>(Wz); r.arr_keys[1] = a.take<u64>(Wz);
        r.arr_vals[0] = a.take<int32_t>(Wz); r.arr_vals[1] = a.take<int32_t>(Wz);
        r.create = a.take<i64>(Wz);
      }
      if (r.cls.n) { X.wl_class = a.take<int32_t>(Wz); X.cq_class_start = a.take<int32_t>((size_t)Q + 1); X.class_nofit = a.take<uint8_t>(r.cls.n); }
    }
    if (m.lat) X.wl_evict = a.take<i64>(Wz);
    if (m.checks) { X.wl_check = a.take<i64>(Wz); X.wl_fail = a.take<int32_t>(Wz); X.wl_retries = a.take<int32_t>(Wz); }
    if (m.pr) {
      X.wl_pr = a.take<i64>(Wz); X.wl_pr_fail = a.take<int32_t>(Wz); X.wl_pr_count = a.take<int32_t>(Wz);
      X.wl_pr_at = a.take<i64>(Wz); X.wl_pr_prev = a.take<i64>(Wz);
    }
    if (m.requeue) { X.wl_ts0 = a.take<i64>(Wz); X.wl_sort_ts = a.take<i64>(Wz); X.wl_requeue_at = a.take<i64>(Wz); X.wl_ready_ns = a.take<i64>(Wz); }
    if (m.deact) X.wl_deactivated = a.take<uint8_t>(Wz);
    if (m.mx) { X.wl_max_exec = a.take<int32_t>(Wz); X.wl_exec_acc = a.take<int32_t>(Wz); }
    if (m.afs) {
      X.seg_start = a.take<int32_t>(r.afs.seg_start.size()); X.lq_seg = a.take<int32_t>(r.afs.lq_seg.size());
      X.seg_lq = a.take<int32_t>(r.afs.seg_lq.size()); X.afs_cqs = a.take<int32_t>(r.afs.afs_cqs.size());
      X.head_seg = a.take<int32_t>(Q); X.wl_lq = a.take<int32_t>(Wz); X.cq_afs = a.take<uint8_t>(Q);
      X.lq_weight = a.take<double>(L); X.lq_consumed = a.take<i64>((size_t)L * R); X.lq_consumed_scale = a.take<int32_t>((size_t)L * R);
      X.lq_penalty = a.take<i64>(LR); X.lq_usage = a.take<double>(Lz);
      X.res_weight = a.take<double>(R); X.milli_mul = a.take<i64>(R);
    }
    if (m.decay) { X.lq_last = a.take<i64>(Lz); X.lq_adm = a.take<i64>(LR); X.afs_samples = a.take<unsigned long long>(1); }
    if (m.quota) {  // the edits and drain_quota_prep's tables
      X.qc_ns = a.take<i64>(NQC); X.qc_node = a.take<int32_t>(NQC);
      X.qc_nominal = a.take<i64>(NQC * FR); X.qc_blimit = a.take<i64>(NQC * FR); X.qc_llimit = a.take<i64>(NQC * FR);
      X.qc_root = a.take<int32_t>(NQC); X.qc_tree = a.take<int32_t>(NQC); X.qc_tree_next = a.take<int32_t>(NQC);
      X.qc_cq_start = a.take<int32_t>(r.nR + 1); X.qc_cq = a.take<int32_t>((size_t)std::max(1, Q)); X.qc_blob_gen = a.take<int32_t>((size_t)std::max(1, Q));
    }
    if (r.s->wl_inactive) r.inactive = a.take<uint8_t>(Wz);
    if (m.act) {  // the edits, their neighbours, and the per-record state of a boundary
      X.ac_ns = a.take<i64>(NAC); X.ac_wl = a.take<int32_t>(NAC); X.ac_on = a.take<uint8_t>(NAC);
      X.ac_next = a.take<int32_t>(NAC); X.ac_prev = a.take<int32_t>(NAC);
      X.wl_ac_from = a.take<int32_t>(Wz); X.wl_stop = a.take<i64>(Wz); X.wl_gone = a.take<i64>(Wz);
    }
    if (m.rcl) {  // the steps, the records' assignments, the generations' blob offsets
      X.wl_rc_start = a.take<int32_t>(Wz + 1); X.rc_after = a.take<i64>(NRCz); X.rc_ps = a.take<int32_t>(NRCz); X.rc_remaining = a.take<int32_t>(NRCz);
      if (r.s->rc_sched_hash) X.rc_hash = a.take<i64>(NRCz);
      if (r.cls.n) X.rc_class = a.take<int32_t>(NRCz);
      X.ps_adm_cnt = a.take<int32_t>(Pz); X.ps_adm_fl = a.take<int8_t>(Pz * R); X.ps_adm_use = a.take<i64>(Pz * R);
      X.rc_blob_gen = a.take<int32_t>((size_t)std::max(1, Q));
    }
  };
  return r.h->drain_arena.carve(layout);
}

// uploads and initial values of the drain's tables
static int32_t drain_upload(DrainRun &r) {
  kb_handle *h = r.h; const kb_snapshot *s = r.s; const DrainMode &m = r.m;
  DrainDev &X = r.X; DevSnap &D = h->D;
  const int W = r.W, Q = r.Q, R = r.R, L = r.L;
  const size_t Wz = (size_t)W, n_adm = (size_t)s->n_adm, LR = (size_t)std::max(1, L) * R;
  X.trace_cap = (long long)r.trace_cap;
  X.cq_usage = const_cast<i64 *>(D.cq_usage); X.wl_last_gen = const_cast<i64 *>(D.wl_last_gen); X.ps_last_tried = const_cast<int8_t *>(D.ps_last_tried);
  X.A_cap = (int)r.Acap; X.AU_cap = (int)r.AUcap;
  // every counter starts at 0, once: the cumulative ones are never cleared, and no kernel before the first boundary
  // writes a counter but k_drain_init_events (the arrived prefix) and k_drain_heads
  CUDA_TRY(h, cudaMemsetAsync(X.counters, 0, (KB_DC_RECLAIMS + 1) * 4, h->stream));
  if (m.replay || m.events) {  // event mode without adm_wl: the rows of the snapshot have no record (-1)
    if (m.replay) CUDA_TRY(h, h2d(h, X.adm.wl, s->adm_wl, n_adm * 4));
    else CUDA_TRY(h, cudaMemsetAsync(X.adm.wl, 0xff, n_adm * 4, h->stream));
    X.wl_has_qr = const_cast<uint8_t *>(D.wl_has_qr);
  }
  if (m.compact) {
    CUDA_TRY(h, cudaMemsetAsync(X.adm_dead, 0, r.Acap * 4, h->stream));
    CUDA_TRY(h, cudaMemsetAsync(X.root_mark, 0, r.nR * 4, h->stream));
  }
  if (m.events) {  // drain_row_start's columns
    if (r.rows.phased) CUDA_TRY(h, h2d(h, X.adm.phase, r.rows.phase.data(), n_adm));
    else if (m.requeue || m.mx) CUDA_TRY(h, cudaMemsetAsync(X.adm.phase, KB_PH_RUN, n_adm, h->stream));
    CUDA_TRY(h, h2d(h, X.adm.finish, r.rows.finish.data(), n_adm * 8));
    if (s->wl_run_ns) CUDA_TRY(h, h2d(h, X.wl_run, s->wl_run_ns, Wz * 8));
    if (r.create) { CUDA_TRY(h, h2d(h, r.create, s->wl_create_ns, Wz * 8)); X.n_arr = W; }
    if (r.cls.n) {
      CUDA_TRY(h, h2d(h, X.wl_class, r.cls.wl_class.data(), Wz * 4));
      CUDA_TRY(h, h2d(h, X.cq_class_start, r.cls.cq_class_start.data(), ((size_t)Q + 1) * 4));
      CUDA_TRY(h, cudaMemsetAsync(X.class_nofit, 0, (size_t)r.cls.n, h->stream));
    }
    if (m.lat) {
      CUDA_TRY(h, h2d(h, X.wl_evict, s->wl_evict_ns, Wz * 8));
      if (!r.rows.evicting.empty()) CUDA_TRY(h, h2d(h, X.adm.evicting, r.rows.evicting.data(), n_adm));
      else CUDA_TRY(h, cudaMemsetAsync(X.adm.evicting, 0, n_adm, h->stream));
    }
  }
  if (m.afs) {
    CUDA_TRY(h, h2d(h, X.seg_start, r.afs.seg_start.data(), r.afs.seg_start.size() * 4));
    CUDA_TRY(h, h2d(h, X.lq_seg, r.afs.lq_seg.data(), r.afs.lq_seg.size() * 4));
    CUDA_TRY(h, h2d(h, X.seg_lq, r.afs.seg_lq.data(), r.afs.seg_lq.size() * 4));
    CUDA_TRY(h, h2d(h, X.afs_cqs, r.afs.afs_cqs.data(), r.afs.afs_cqs.size() * 4));
    CUDA_TRY(h, h2d(h, X.wl_lq, s->wl_lq, Wz * 4));
    CUDA_TRY(h, h2d(h, X.cq_afs, s->cq_afs, (size_t)Q));
    CUDA_TRY(h, h2d(h, X.lq_weight, s->lq_weight, (size_t)L * 8));
    CUDA_TRY(h, h2d(h, X.lq_consumed, s->lq_consumed, (size_t)L * R * 8));
    CUDA_TRY(h, h2d(h, X.lq_consumed_scale, s->lq_consumed_scale, (size_t)L * R * 4));
    if (s->lq_penalty) CUDA_TRY(h, h2d(h, X.lq_penalty, s->lq_penalty, (size_t)L * R * 8));
    else CUDA_TRY(h, cudaMemsetAsync(X.lq_penalty, 0, LR * 8, h->stream));
    CUDA_TRY(h, h2d(h, X.lq_usage, r.afs.lq_usage.data(), (size_t)std::max(1, L) * 8));
    CUDA_TRY(h, h2d(h, X.res_weight, s->afs_res_weight, (size_t)R * 8));
    CUDA_TRY(h, h2d(h, X.milli_mul, s->afs_milli_mul, (size_t)R * 8));
    X.alpha = s->afs_alpha;
    X.n_afs_cq = (int)r.afs.afs_cqs.size();
  }
  if (m.sticky) CUDA_TRY(h, h2d(h, X.cq_sticky, s->cq_sticky, (size_t)Q * 4));
  if (m.requeue) {  // checks / PodsReady: queue-order timestamps (the Evicted time of a record requeued by a check or a
                    // PodsReady timeout), RequeueAt
    r.qts.assign(s->wl_ts, s->wl_ts + W);
    if (s->wl_check_evict_ns)
      for (int w = 0; w < W; w++) if (s->wl_check_evict_ns[w] != INT64_MIN && !r.held[w]) r.qts[w] = s->wl_check_evict_ns[w];
    if (m.pr && s->wl_pods_ready_evict_ns && !s->pods_ready_requeue_creation)
      for (int w = 0; w < W; w++) if (s->wl_pods_ready_evict_ns[w] != INT64_MIN) r.qts[w] = s->wl_pods_ready_evict_ns[w];
    r.requeue_at = drain_table_or<i64>(s->wl_requeue_at_ns, Wz, INT64_MIN);
    X.wl_qts = const_cast<i64 *>(D.wl_ts);
    CUDA_TRY(h, h2d(h, X.wl_ts0, s->wl_ts, Wz * 8));
    CUDA_TRY(h, h2d(h, X.wl_qts, r.qts.data(), Wz * 8));  // the cycle kernels read the queue-order timestamp
    CUDA_TRY(h, h2d(h, X.wl_sort_ts, r.qts.data(), Wz * 8));
    CUDA_TRY(h, h2d(h, X.wl_requeue_at, r.requeue_at.data(), Wz * 8));
  }
  if (m.checks) {
    r.fails = drain_table_or<int32_t>(s->wl_check_fail, Wz, 0);
    r.retries = drain_table_or<int32_t>(s->wl_check_retries, Wz, 0);
    CUDA_TRY(h, h2d(h, X.wl_check, s->wl_check_ns, Wz * 8));
    CUDA_TRY(h, h2d(h, X.wl_fail, r.fails.data(), Wz * 4));
    CUDA_TRY(h, h2d(h, X.wl_retries, r.retries.data(), Wz * 4));
    X.check_base_s = s->check_backoff_base_s; X.check_max_s = s->check_backoff_max_s; X.check_limit = s->check_backoff_limit;
  }
  if (m.pr) {
    r.pr_fails = drain_table_or<int32_t>(s->wl_pods_ready_fail, Wz, 0);
    r.pr_counts = drain_table_or<int32_t>(s->wl_pods_ready_count, Wz, 0);
    r.pr_none.assign(Wz, INT64_MIN);
    CUDA_TRY(h, h2d(h, X.wl_pr, s->wl_pods_ready_ns, Wz * 8));
    CUDA_TRY(h, h2d(h, X.wl_pr_fail, r.pr_fails.data(), Wz * 4));
    CUDA_TRY(h, h2d(h, X.wl_pr_count, r.pr_counts.data(), Wz * 4));
    CUDA_TRY(h, h2d(h, X.wl_pr_at, r.rows.pr_at.data(), Wz * 8));  // a ready attempt under way reaches PodsReady at Admitted + delay
    CUDA_TRY(h, h2d(h, X.wl_pr_prev, r.pr_none.data(), Wz * 8));   // no PodsReady before the attempts under way
    X.pr_timeout = s->pods_ready_timeout_ns; X.pr_base_s = s->pods_ready_backoff_base_s; X.pr_max_s = s->pods_ready_backoff_max_s;
    X.pr_limit = s->pods_ready_backoff_limit; X.pr_creation = s->pods_ready_requeue_creation;
  }
  if (m.mx) {  // the limits, the accumulated times at the start, the Admitted times of the snapshot's rows
    r.exec_acc = drain_table_or<int32_t>(s->wl_exec_acc_s, Wz, -1);
    CUDA_TRY(h, h2d(h, X.wl_max_exec, s->wl_max_exec_s, Wz * 4));
    CUDA_TRY(h, h2d(h, X.wl_exec_acc, r.exec_acc.data(), Wz * 4));
    if (n_adm) CUDA_TRY(h, h2d(h, X.adm.since, s->adm_exec_since_ns, n_adm * 8));
  }
  if ((m.mx || m.blk) && !m.requeue) CUDA_TRY(h, cudaMemsetAsync(X.wl_deactivated, 0, Wz, h->stream));  // (k_drain_init_checks clears it otherwise)
  if (r.inactive) CUDA_TRY(h, h2d(h, r.inactive, s->wl_inactive, Wz));
  if (m.act) {
    const size_t NAC = (size_t)m.n_ac;
    CUDA_TRY(h, h2d(h, X.ac_ns, s->ac_ns, NAC * 8));
    CUDA_TRY(h, h2d(h, X.ac_wl, s->ac_wl, NAC * 4));
    CUDA_TRY(h, h2d(h, X.ac_on, s->ac_active, NAC));
    CUDA_TRY(h, h2d(h, X.ac_next, r.ac_next.data(), NAC * 4));
    CUDA_TRY(h, h2d(h, X.ac_prev, r.ac_prev.data(), NAC * 4));
    X.n_ac = m.n_ac;
  }
  if (m.decay) {
    CUDA_TRY(h, h2d(h, X.lq_last, s->lq_last_update_ns, (size_t)L * 8));
    CUDA_TRY(h, h2d(h, X.lq_adm, r.afs.lq_adm.data(), LR * 8));
    CUDA_TRY(h, h2d(h, X.adm.lq, s->adm_lq, n_adm * 4));
    CUDA_TRY(h, cudaMemsetAsync(X.afs_samples, 0, 8, h->stream));
    X.half_life_ns = s->afs_half_life_ns; X.sampling_ns = s->afs_sampling_ns;
  }
  if (m.quota) {
    const size_t NQC = (size_t)m.n_qc, FRz = (size_t)r.FR;
    CUDA_TRY(h, h2d(h, X.qc_ns, s->qc_ns, NQC * 8));
    CUDA_TRY(h, h2d(h, X.qc_node, s->qc_node, NQC * 4));
    CUDA_TRY(h, h2d(h, X.qc_nominal, s->qc_nominal, NQC * FRz * 8));
    CUDA_TRY(h, h2d(h, X.qc_blimit, s->qc_borrow_limit, NQC * FRz * 8));
    CUDA_TRY(h, h2d(h, X.qc_llimit, s->qc_lend_limit, NQC * FRz * 8));
    CUDA_TRY(h, h2d(h, X.qc_root, r.qc.root.data(), NQC * 4));
    CUDA_TRY(h, h2d(h, X.qc_tree, r.qc.tree.data(), NQC * 4));
    CUDA_TRY(h, h2d(h, X.qc_tree_next, r.qc.tree_next.data(), NQC * 4));
    CUDA_TRY(h, h2d(h, X.qc_cq_start, r.qc.cq_start.data(), r.qc.cq_start.size() * 4));
    CUDA_TRY(h, h2d(h, X.qc_cq, r.qc.cq.data(), r.qc.cq.size() * 4));
    CUDA_TRY(h, h2d(h, X.qc_blob_gen, r.qc.blob_gen.data(), r.qc.blob_gen.size() * 4));
    X.n_qc = m.n_qc;
  }
  if (m.rcl) {
    const size_t NRC = (size_t)m.n_rc;
    CUDA_TRY(h, h2d(h, X.wl_rc_start, s->wl_rc_start, (Wz + 1) * 4));
    if (NRC) {
      CUDA_TRY(h, h2d(h, X.rc_after, s->rc_after_ns, NRC * 8));
      CUDA_TRY(h, h2d(h, X.rc_ps, s->rc_ps, NRC * 4));
      CUDA_TRY(h, h2d(h, X.rc_remaining, s->rc_remaining, NRC * 4));
      if (X.rc_hash) CUDA_TRY(h, h2d(h, X.rc_hash, s->rc_sched_hash, NRC * 8));
      if (X.rc_class) CUDA_TRY(h, h2d(h, X.rc_class, r.cls.rc_class.data(), NRC * 4));
    }
    CUDA_TRY(h, h2d(h, X.ps_adm_fl, r.rc.fl.data(), r.rc.fl.size()));
    CUDA_TRY(h, h2d(h, X.ps_adm_cnt, r.rc.cnt.data(), r.rc.cnt.size() * 4));
    CUDA_TRY(h, h2d(h, X.ps_adm_use, r.rc.use.data(), r.rc.use.size() * 8));
    if (n_adm) {
      CUDA_TRY(h, h2d(h, X.adm.rc_next, r.rc.next.data(), n_adm * 8));
      CUDA_TRY(h, h2d(h, X.adm.rc_cur, r.rc.cur.data(), n_adm * 4));
    }
    CUDA_TRY(h, h2d(h, X.rc_blob_gen, r.rc_blob_gen.data(), r.rc_blob_gen.size() * 4));
  }
  return KB_OK;
}

// per-segment queue order (queueOrderingFunc): stable LSD passes uid -> timestamp -> (segment | priority desc); also
// the re-sort of admission checks and PodsReady (same segments, same q_start)
static cudaError_t drain_sort_queues(DrainRun &r) {
  kb_handle *h = r.h; const DevSnap &D = h->D; DrainDev &X = r.X;
  cudaError_t e = cudaMemsetAsync(r.q_count, 0, sizeof(int32_t) * ((size_t)r.S + 2), h->stream);
  if (e != cudaSuccess) return e;
  cub::DoubleBuffer<u64> dk(r.keys[0], r.keys[1]); cub::DoubleBuffer<int32_t> dv(r.vals[0], r.vals[1]);
  size_t bytes = r.sort_bytes;
  k_drain_keys_uid<<<drain_blocks(r.W), DRAIN_TB, 0, h->stream>>>(D, dk.Current(), dv.Current());
  if ((e = cub::DeviceRadixSort::SortPairs(r.sort_tmp, bytes, dk, dv, r.W, 0, 64, h->stream)) != cudaSuccess) return e;
  k_drain_keys_ts<<<drain_blocks(r.W), DRAIN_TB, 0, h->stream>>>(D, dv.Current(), dk.Current());
  if ((e = cub::DeviceRadixSort::SortPairs(r.sort_tmp, bytes, dk, dv, r.W, 0, 64, h->stream)) != cudaSuccess) return e;
  k_drain_keys_cq<<<drain_blocks(r.W), DRAIN_TB, 0, h->stream>>>(D, X, dv.Current(), dk.Current(), r.q_count);
  int cq_bits = 1; while ((1ll << cq_bits) < (long long)r.S) cq_bits++;
  if ((e = cub::DeviceRadixSort::SortPairs(r.sort_tmp, bytes, dk, dv, r.W, 0, 32 + cq_bits, h->stream)) != cudaSuccess) return e;
  X.q_order = dv.Current();
  return cudaSuccess;
}
// the heads of the next cycle
static void drain_heads(DrainRun &r) {
  kb_handle *h = r.h; const DevSnap &D = h->D; const DrainDev &X = r.X;
  k_drain_flag<<<drain_blocks(r.Q), DRAIN_TB, 0, h->stream>>>(D, X);
  if (X.n_afs_cq) k_drain_afs_heads<<<(X.n_afs_cq + 7) / 8, DRAIN_TB, 0, h->stream>>>(D, X);
  k_scan_i32<<<1, 1024, 0, h->stream>>>(X.flag, X.pos, r.Q);
  k_drain_heads<<<drain_blocks(r.Q), DRAIN_TB, 0, h->stream>>>(D, X, const_cast<int32_t *>(D.heads));
}

// the start of the drain: the queues, the arrival order, every record's state at now_ns, the first heads; one
// synchronisation
static int32_t drain_start(DrainRun &r) {
  kb_handle *h = r.h; const kb_snapshot *s = r.s; const DrainMode &m = r.m;
  DevSnap &D = h->D; DrainDev &X = r.X;
  DrainWords &hw = *reinterpret_cast<DrainWords *>(&h->host_words[64]);
  const int W = r.W, S = r.S, tb = DRAIN_TB;
  CUDA_TRY(h, drain_sort_queues(r));
  if (r.create) {  // arrival order: (creation time, index); the workloads present at the start are its first k_drain_init_events prefix
    cub::DoubleBuffer<u64> dk(r.arr_keys[0], r.arr_keys[1]); cub::DoubleBuffer<int32_t> dv(r.arr_vals[0], r.arr_vals[1]);
    size_t bytes = r.sort_bytes;
    k_drain_keys_create<<<drain_blocks(r.W), tb, 0, h->stream>>>(W, r.create, dk.Current(), dv.Current());
    CUDA_TRY(h, cub::DeviceRadixSort::SortPairs(r.sort_tmp, bytes, dk, dv, W, 0, 64, h->stream));
    X.arr_key = dk.Current(); X.arr_order = dv.Current();
  }
  k_scan_i32<<<1, 1024, 0, h->stream>>>(r.q_count, X.q_start, S);
  k_drain_init<<<std::max(drain_blocks(r.W), drain_blocks(S)), tb, 0, h->stream>>>(D, X, S);
  if (m.events) k_drain_init_events<<<std::max(1, drain_blocks(r.W)), tb, 0, h->stream>>>(D, X, r.create, s->now_ns);
  if (m.replay || m.events || m.sticky) k_drain_init_replay<<<std::max(drain_blocks(r.W), drain_blocks(s->n_adm)), tb, 0, h->stream>>>(D, X, m.replay ? s->n_adm : 0);
  // records in backoff, records inactive at the start, and the first RequeueAt into clock[2] (k_drain_init_events set
  // clock[0] = now_ns)
  if (m.requeue) k_drain_init_checks<<<std::max(1, drain_blocks(r.W)), tb, 0, h->stream>>>(X, W, s->now_ns);
  if (m.blk) k_drain_init_active<<<std::max(1, drain_blocks(r.W)), tb, 0, h->stream>>>(X, W, r.inactive);
  if (m.requeue) k_drain_backoff<<<std::max(1, drain_blocks(r.W)), tb, 0, h->stream>>>(X, W);
  k_drain_advance<<<drain_blocks(S), tb, 0, h->stream>>>(X, S);
  if (m.decay) {  // the samples due at or before now_ns (k_drain_init_events set clock[0] = now_ns), before the first heads
    CUDA_TRY(h, cudaMemsetAsync(D.status, 0, 4, h->stream));
    k_drain_afs_decay<<<std::max(1, drain_blocks(r.L)), tb, 0, h->stream>>>(D, X, r.L);
  }
  drain_heads(r);
  CUDA_TRY(h, cudaMemcpyAsync(&hw.counters[0], X.counters, 4, cudaMemcpyDeviceToHost, h->stream));
  if (m.decay) CUDA_TRY(h, cudaMemcpyAsync(&hw.status, D.status, 4, cudaMemcpyDeviceToHost, h->stream));
  CUDA_TRY(h, cudaStreamSynchronize(h->stream));
  if (m.decay && (hw.status & KBS_AFS_OVERFLOW)) return fail(h, KB_ERR_UNSUPPORTED, "afs: a decayed consumed quantity overflows int64");
  r.n_live = (int)hw.counters[0];
  r.A_cur = s->n_adm; r.AU_cur = s->n_adm_use;
  r.t = s->now_ns;  // the clock: the plain drain steps it by one per cycle
  r.step = s->drain_cycle_ns > 0 ? s->drain_cycle_ns : 1;
  if (m.requeue) {
    CUDA_TRY(h, cudaEventCreate(&r.ev_r[0]));
    CUDA_TRY(h, cudaEventCreate(&r.ev_r[1]));
  }
  return KB_OK;
}

// One boundary, one synchronisation (kueue_b200/drain.py _Drain.boundary): cycle c at t (in event mode, a jump to the
// next event when there are no heads), its decisions and admissions, the evictions; in event mode E, t_{c+1}, the decay
// samples, completions and arrivals; where rows can die (compact) the inadmissible requeue and the compaction over
// [0, bound); then the heads of the next cycle.  A plain drain ends at a cycle without heads or one that neither admits
// nor evicts (the next cycle would see the same snapshot); an event drain when no event is left (*done).
// Capacity: before the compaction the tables hold the live rows plus this cycle's admissions, and every admitted head
// is a workload that holds no row, so the rows stay within A_in + min(W, Hcap * max_cycles) and the cells within
// AU_in + min(P * R, that bound * FR) (a readmitted victim's old cells left with its old row): what upload_impl
// reserved.  An admission past the end is not written and the call fails.
static int32_t drain_boundary(DrainRun &r, bool *done) {
  kb_handle *h = r.h; const DrainMode &m = r.m; kb_drain_out *out = r.out;
  DevSnap &D = h->D; DrainDev &X = r.X;
  DrainWords &hw = *reinterpret_cast<DrainWords *>(&h->host_words[64]);
  const int tb = DRAIN_TB, n_live = r.n_live, sms = std::max(1, h->sm_count);
  const bool jump = n_live == 0;
  *done = jump && !m.events;
  if (*done) return KB_OK;
  const int32_t *n_new_d = jump ? nullptr : X.e_adm_off + n_live;
  if (!jump) {
    D.H = n_live; D.now_ns = r.t;
    D.A = h->preempt_possible ? r.A_cur : 0; D.AU = h->preempt_possible ? r.AU_cur : 0;  // without preemption policies the cycle never looks at the admitted tables
    if (int32_t rc = cycle_enqueue(h)) return rc;
    X.cycle = r.cyc;
  } else {
    CUDA_TRY(h, cudaEventRecord(h->ev2, h->stream));
    X.cycle = -2 - r.jumps;  // stamps of a jump (cycle + 1 < 0) never meet those of a cycle
  }
  X.A = r.A_cur; X.AU = r.AU_cur; X.trace_off = (long long)out->n_decisions;
  kmark(h, KB_K_DRAIN);
  if (m.compact) CUDA_TRY(h, cudaMemsetAsync(X.counters + 1, 0, 4 * 4, h->stream));
  if (m.events) CUDA_TRY(h, cudaMemsetAsync(X.counters + KB_DC_FINISHED, 0, 3 * 4, h->stream));
  int bound = r.A_cur;  // rows the boundary looks at: the tables plus room for this cycle's admissions
  if (!jump) {
    const int nbH = drain_blocks(n_live);
    k_drain_apply<<<nbH, tb, 0, h->stream>>>(D, X);
    k_scan_i32<<<1, 1024, 0, h->stream>>>(X.e_assumed, X.e_adm_off, n_live);
    k_scan_i32<<<1, 1024, 0, h->stream>>>(X.e_ncells, X.e_cell_off, n_live);
    k_drain_admit<<<nbH, tb, 0, h->stream>>>(D, X, r.t);
    if (m.evict) k_drain_evict<<<nbH, tb, 0, h->stream>>>(D, X);
    bound = (int)std::min<size_t>((size_t)r.A_cur + n_live, r.Acap);
  }
  if (m.events) {
    const int nbB = std::max(1, drain_blocks(bound)), nbAc = std::max(1, std::min(drain_blocks(m.n_ac), sms));  // grid-stride over the edits
    k_drain_ev_min<<<nbB, tb, 0, h->stream>>>(X, bound, n_new_d);
    k_drain_ev_next<<<1, 1, 0, h->stream>>>(X, r.t, r.step, jump, n_new_d);
    if (m.quota) k_drain_quota<<<1, 1024, 0, h->stream>>>(D, X);  // step 5: the edits, before the verdicts
    if (m.act) k_drain_active<<<nbAc, tb, 0, h->stream>>>(D, X, 0);  // the edits of records without a row; the stop times
    if (m.decay) k_drain_afs_decay<<<std::max(1, drain_blocks(r.L)), tb, 0, h->stream>>>(D, X, r.L);  // samples due in (t, t_{c+1}], before the completions
    k_drain_finish<<<nbB, tb, 0, h->stream>>>(D, X, bound, n_new_d);
    if (X.arr_key) k_drain_arrive<<<std::max(1, std::min(drain_blocks(r.W), 8 * sms)), tb, 0, h->stream>>>(X);
    // the edits of records that met their own events first, before k_drain_backoff folds the remaining RequeueAts
    // into the next E: a record a timeout or a Retry put in BACKOFF and a later stop deactivated has none
    if (m.act) k_drain_active<<<nbAc, tb, 0, h->stream>>>(D, X, 1);
    if (m.requeue) k_drain_backoff<<<std::max(1, drain_blocks(r.W)), tb, 0, h->stream>>>(X, r.W);
  }
  if (m.compact) {
    k_drain_requeue<<<drain_blocks(r.Q), tb, 0, h->stream>>>(D, X);
    if (m.act) k_drain_advance<<<drain_blocks(r.S), tb, 0, h->stream>>>(X, r.S);  // a deactivated record may sit at a cursor
    const int nbA = drain_blocks(bound + 1);
    k_drain_live<<<nbA, tb, 0, h->stream>>>(X, bound, n_new_d);
    size_t sb = r.scan_bytes;
    CUDA_TRY(h, cub::DeviceScan::ExclusiveSum(r.scan_tmp, sb, X.row_live, X.row_new, bound + 1, h->stream));
    sb = r.scan_bytes;
    CUDA_TRY(h, cub::DeviceScan::ExclusiveSum(r.scan_tmp, sb, X.row_cells, X.cell_new, bound + 1, h->stream));
    k_drain_compact<<<nbA, tb, 0, h->stream>>>(X, r.other, bound);
  }
  drain_heads(r);
  kmark(h, -1);
  CUDA_TRY(h, cudaEventRecord(h->ev_d, h->stream));
  CUDA_TRY(h, cudaMemcpyAsync(&hw.counters[0], X.counters, (size_t)r.n_used * 4, cudaMemcpyDeviceToHost, h->stream));
  if (!jump) CUDA_TRY(h, cudaMemcpyAsync(&hw.n_new, n_new_d, 4, cudaMemcpyDeviceToHost, h->stream));
  if (!m.compact) CUDA_TRY(h, cudaMemcpyAsync(&hw.n_cells, X.e_cell_off + n_live, 4, cudaMemcpyDeviceToHost, h->stream));
  if (m.afs && (!jump || m.decay)) CUDA_TRY(h, cudaMemcpyAsync(&hw.status, D.status, 4, cudaMemcpyDeviceToHost, h->stream));
  if (m.events) CUDA_TRY(h, cudaMemcpyAsync(&hw.t_next, X.clock, 8, cudaMemcpyDeviceToHost, h->stream));
  CUDA_TRY(h, cudaStreamSynchronize(h->stream));
  if (!jump) {
    if (int32_t rc = cycle_finish(h)) return rc;
    if (m.afs && (hw.status & KBS_AFS_OVERFLOW)) return fail(h, KB_ERR_UNSUPPORTED, "afs: an entry penalty overflows int64");
    for (int i = 0; i < KB_N_KERNELS; i++) r.kms[i] += h->stats.kernel_ms[i];
  }
  if (m.decay && (hw.status & KBS_AFS_OVERFLOW)) return fail(h, KB_ERR_UNSUPPORTED, "afs: a decayed consumed quantity overflows int64");
  { float ms = 0; cudaEventElapsedTime(&ms, h->ev2, h->ev_d); r.gpu_ms += ms; }
  if (m.compact && hw.counters[KB_DC_FULL]) return fail(h, KB_ERR_CAPACITY, "kb_run_drain: the admitted tables are full");
  if (m.mx && (hw.counters[KB_DC_EXEC_STATUS] & KBS_EXEC_OVERFLOW))
    return fail(h, KB_ERR_UNSUPPORTED, "max exec: an accumulated execution time leaves int32");
  const int n_new = jump ? 0 : (int)hw.n_new, n_ev = m.evict ? (int)hw.counters[KB_DC_EVICTED] : 0;
  if (!jump) {
    const int cyc = r.cyc;
    if (out->cycle_heads) out->cycle_heads[cyc] = n_live;
    if (out->cycle_admitted) out->cycle_admitted[cyc] = n_new;
    if (out->cycle_evicted) out->cycle_evicted[cyc] = n_ev;
    if (m.events && out->cycle_start_ns) out->cycle_start_ns[cyc] = r.t;
    for (const DrainCounter &c : r.counters)
      if (c.on && c.cycle) c.cycle[cyc] = 0;
    out->n_decisions += n_live; out->n_admitted += n_new; out->n_evicted += n_ev;
    out->n_cycles = ++r.cyc;
  } else {
    r.jumps++;
  }
  for (DrainCounter &c : r.counters) {  // the events of this boundary; those between the start of the last cycle and the next one are that cycle's
    if (!c.on) continue;
    const uint32_t *v = &hw.counters[c.idx];
    int n = (int)v[0];
    if (c.kind == DC_CUMULATIVE) { n = (int)(v[0] - c.seen); c.seen = v[0]; }
    else if (c.kind == DC_RANGE) n = (int)(v[1] - v[0]);
    *c.total += n;
    if (r.cyc > 0 && c.cycle) c.cycle[r.cyc - 1] += n;
  }
  if (m.compact) {  // the compacted half becomes the admitted tables of the next boundary
    r.A_cur = (int)hw.counters[KB_DC_ROWS]; r.AU_cur = (int)hw.counters[KB_DC_CELLS];
    std::swap(X.adm, r.other);
    drain_point_snap(D, X.adm);
  } else {
    r.A_cur += n_new; r.AU_cur += (int)hw.n_cells;
  }
  r.n_live = (int)hw.counters[0];
  *done = m.events ? hw.counters[KB_DC_END] != 0 : n_new == 0 && n_ev == 0;
  if (*done) return KB_OK;
  if (m.requeue && (int32_t)hw.counters[KB_DC_RESORT] == X.cycle + 1) {  // re-sort: the three passes over the queue-order
    // timestamps, positions, cursors from 0, first_aside from the SET_ASIDE positions, then the heads again.  The segments
    // and their lengths do not change, so n_live holds and no synchronisation is added; the events are read at the next one.
    if (r.resort_timed) { float ms = 0; cudaEventElapsedTime(&ms, r.ev_r[0], r.ev_r[1]); out->resort_ms += ms; r.gpu_ms += ms; }
    CUDA_TRY(h, cudaEventRecord(r.ev_r[0], h->stream));
    CUDA_TRY(h, drain_sort_queues(r));
    k_drain_init_replay<<<std::max(1, drain_blocks(r.W)), tb, 0, h->stream>>>(D, X, 0);
    k_drain_resort_reset<<<drain_blocks(r.S), tb, 0, h->stream>>>(X, r.S);
    k_drain_resort_aside<<<std::max(1, drain_blocks(r.W)), tb, 0, h->stream>>>(X, r.W);
    k_drain_advance<<<drain_blocks(r.S), tb, 0, h->stream>>>(X, r.S);
    CUDA_TRY(h, cudaMemcpyAsync(X.wl_sort_ts, X.wl_qts, (size_t)r.W * 8, cudaMemcpyDeviceToDevice, h->stream));
    drain_heads(r);
    CUDA_TRY(h, cudaEventRecord(r.ev_r[1], h->stream));
    r.resort_timed = true;
    out->n_resorts++;
  }
  r.t = m.events ? hw.t_next : r.t + 1;
  return KB_OK;
}

// the end of the drain: the clock, the device time, the tables kb_drain_out asks for
static int32_t drain_results(DrainRun &r) {
  kb_handle *h = r.h; const DrainMode &m = r.m; kb_drain_out *out = r.out;
  const DevSnap &D = h->D; const DrainDev &X = r.X;
  const size_t Wz = (size_t)r.W, L = (size_t)r.L, R = (size_t)r.R, PR = (size_t)D.P * D.R;
  if (m.events) out->end_ns = r.t;
  if (r.resort_timed) {
    CUDA_TRY(h, cudaEventSynchronize(r.ev_r[1]));
    float ms = 0; cudaEventElapsedTime(&ms, r.ev_r[0], r.ev_r[1]); out->resort_ms += ms; r.gpu_ms += ms;
  }
  out->gpu_ms = r.gpu_ms;
  h->stats.last_cycle_gpu_ms = r.gpu_ms;
  memcpy(h->stats.kernel_ms, r.kms, sizeof(r.kms));
  auto d2h = [&](void *dst, const void *src, size_t bytes) { return cudaMemcpyAsync(dst, src, bytes, cudaMemcpyDeviceToHost, h->stream); };
  if (out->wl_admit_cycle) CUDA_TRY(h, d2h(out->wl_admit_cycle, X.wl_admit_cycle, Wz * 4));
  if (out->wl_last_decision) CUDA_TRY(h, d2h(out->wl_last_decision, X.wl_last_decision, Wz));
  if (out->wl_evals) CUDA_TRY(h, d2h(out->wl_evals, X.wl_evals, Wz * 4));
  if (m.events && out->wl_admit_ns) CUDA_TRY(h, d2h(out->wl_admit_ns, X.wl_admit_ns, Wz * 8));
  if (m.events && out->wl_finish_ns) CUDA_TRY(h, d2h(out->wl_finish_ns, X.wl_finish_ns, Wz * 8));
  if (m.decay) {
    if (out->lq_consumed && L) CUDA_TRY(h, d2h(out->lq_consumed, X.lq_consumed, L * R * 8));
    if (out->lq_consumed_scale && L) CUDA_TRY(h, d2h(out->lq_consumed_scale, X.lq_consumed_scale, L * R * 4));
    if (out->lq_last_update_ns && L) CUDA_TRY(h, d2h(out->lq_last_update_ns, X.lq_last, L * 8));
    CUDA_TRY(h, d2h(&out->n_afs_samples, X.afs_samples, 8));
  }
  if (out->wl_evictions) {
    if (m.replay) CUDA_TRY(h, d2h(out->wl_evictions, X.wl_evictions, Wz * 4));
    else memset(out->wl_evictions, 0, Wz * 4);
  }
  if (m.sticky && out->cq_sticky) CUDA_TRY(h, d2h(out->cq_sticky, X.cq_sticky, (size_t)r.Q * 4));
  if (m.checks) {
    if (out->wl_ready_ns) CUDA_TRY(h, d2h(out->wl_ready_ns, X.wl_ready_ns, Wz * 8));
    if (out->wl_check_retries_out) CUDA_TRY(h, d2h(out->wl_check_retries_out, X.wl_retries, Wz * 4));
  }
  if (m.deact && out->wl_deactivated) CUDA_TRY(h, d2h(out->wl_deactivated, X.wl_deactivated, Wz));
  if (m.deact && out->wl_deactivation_reason) CUDA_TRY(h, d2h(out->wl_deactivation_reason, X.wl_deactivated, Wz));
  if (m.mx && out->wl_exec_acc_s_out) CUDA_TRY(h, d2h(out->wl_exec_acc_s_out, X.wl_exec_acc, Wz * 4));
  if (m.pr) {
    if (out->wl_pods_ready_at_ns) CUDA_TRY(h, d2h(out->wl_pods_ready_at_ns, X.wl_pr_at, Wz * 8));
    if (out->wl_pods_ready_count_out) CUDA_TRY(h, d2h(out->wl_pods_ready_count_out, X.wl_pr_count, Wz * 4));
  }
  if (out->ps_flavor && PR) CUDA_TRY(h, d2h(out->ps_flavor, D.ps_flavor, PR));
  if (out->ps_count && D.P) CUDA_TRY(h, d2h(out->ps_count, D.ps_count_out, (size_t)D.P * 4));
  if (out->cq_usage) CUDA_TRY(h, d2h(out->cq_usage, D.cq_usage, (size_t)r.Q * r.FR * 8));
  if (m.rcl && out->ps_remaining_out && D.P) CUDA_TRY(h, d2h(out->ps_remaining_out, D.ps_count, (size_t)D.P * 4));
  if ((m.quota || m.rcl) && out->cq_generation) CUDA_TRY(h, d2h(out->cq_generation, D.cq_generation, (size_t)r.Q * 8));
  const size_t nt = std::min<size_t>(r.trace_cap, (size_t)out->n_decisions);
  if (nt) {
    CUDA_TRY(h, d2h(out->trace_wl, X.trace_wl, nt * 4));
    CUDA_TRY(h, d2h(out->trace_decision, X.trace_dec, nt));
  }
  CUDA_TRY(h, cudaStreamSynchronize(h->stream));
  if (m.deact && out->wl_deactivated)  // the device byte holds the reason (KB_DR_*)
    for (int w = 0; w < r.W; w++) out->wl_deactivated[w] = out->wl_deactivated[w] != 0;
  return KB_OK;
}

// the stages of kb_run_drain: mode, input checks, plan, buffers, uploads and the start, the boundaries, the results
static int32_t drain_impl(kb_handle *h, const kb_snapshot *s, kb_drain_out *out) {
  DrainRun r;
  r.h = h; r.s = s; r.out = out;
  r.m = drain_mode(s);
  r.counters = drain_counters(out, r.m);
  r.Q = s->n_cq; r.W = s->n_wl; r.R = s->n_resource; r.FR = s->n_flavor * s->n_resource;
  r.Hcap = std::min(r.Q, r.W);
  r.max_cycles = std::max(0, out->max_cycles);
  out->n_cycles = 0; out->n_decisions = 0; out->n_admitted = 0; out->gpu_ms = 0; out->n_evicted = 0;
  out->end_ns = s->now_ns; out->n_resorts = 0; out->resort_ms = 0;
  for (const DrainCounter &c : r.counters) *c.total = 0;
  if (int32_t rc = drain_validate(h, s, r.m, r.held)) return rc;
  if (r.m.sticky && out->cq_sticky) memcpy(out->cq_sticky, s->cq_sticky, (size_t)r.Q * 4);  // the slots of a drain that runs no cycle
  out->n_afs_samples = 0;
  if (r.Hcap == 0 || r.max_cycles == 0) {
    if (r.m.rcl && out->ps_remaining_out && s->n_podset) memcpy(out->ps_remaining_out, s->ps_count, (size_t)s->n_podset * 4);
    return KB_OK;
  }
  size_t extra = (size_t)std::min<long long>((long long)r.W, (long long)r.Hcap * r.max_cycles);
  h->drain_extra_adm = extra;
  h->drain_extra_au = std::min<size_t>((size_t)s->n_podset * r.R, extra * (size_t)r.FR);
  h->drain_mode = true;
  h->drain_events = r.m.events;
  kb_snapshot s2 = *s;
  s2.n_heads = r.Hcap; s2.heads = nullptr;
  if (int32_t rc = upload_impl(h, &s2, false)) return rc;
  if (!h->ev_d) cudaEventCreate(&h->ev_d);
  if (int32_t rc = drain_plan(r)) return rc;
  r.X.adm = drain_snap_rows(h->D);  // the first half borrows the DevSnap's columns; drain_carve adds the others
  if (!drain_carve(r)) return fail(h, KB_ERR_CUDA, "kb_run_drain: cudaMalloc of the drain buffer failed");
  if (int32_t rc = drain_upload(r)) return rc;
  if (int32_t rc = drain_start(r)) return rc;
  for (bool done = false; !done && r.cyc < r.max_cycles;)
    if (int32_t rc = drain_boundary(r, &done)) return rc;
  return drain_results(r);
}

extern "C" int32_t kb_run_drain(kb_handle *h, const kb_snapshot *s, kb_drain_out *out) {
  if (!h || !s || !out) return KB_ERR_INVALID;
  int32_t rc = drain_impl(h, s, out);
  h->drain_mode = false; h->drain_events = false; h->drain_extra_adm = 0; h->drain_extra_au = 0;
  if ((s->n_quota_change > 0 && s->qc_ns) || s->wl_rc_start) h->static_gen = 0;  // quota changes or reclaim steps edited the resident static tables
  h->uploaded = false;  // the resident snapshot was consumed (queues advanced, admitted tables grown)
  return rc;
}

// ---------------------------------------------------------------------------
// kb_tas_find: topology-aware placement (kb_tas.cuh)
// ---------------------------------------------------------------------------
extern "C" int32_t kb_tas_find(kb_handle *h, const kb_tas_topology *t, const kb_tas_requests *r, kb_tas_out *out) {
  if (!h || !t || !r || !out) return KB_ERR_INVALID;
  cudaSetDevice(h->device);
  const int L = t->n_levels, ND = t->n_domains, R = t->n_resource, NQ = r->n_req;
  if (L < 1 || ND < 0 || R < 1 || R > 32 || t->pods_resource < 0 || t->pods_resource >= R || NQ < 0) return fail(h, KB_ERR_INVALID, "tas: bad dimensions");
  if (ND == 0) {  // no node of the flavor is schedulable: "no topology domains at level" (:1203-1205) for the first podset of every chain
    for (int q = 0; q < NQ; q++) {
      bool first = q == 0 || r->chain[q] != r->chain[q - 1];
      bool bad = r->level[q] < 0 || r->level[q] >= L || r->slice_level[q] < 0 || r->slice_level[q] >= L || r->level[q] > r->slice_level[q] || r->slice_size[q] < 1;
      out->status[q] = first ? (bad ? KB_TAS_BAD_REQUEST : KB_TAS_NO_FIT) : -1;
      out->asg_start[q] = 0;
    }
    out->asg_start[NQ] = 0; out->n_assigned = 0;
    return KB_OK;
  }
  if (t->level_start[0] != 0 || t->level_start[L] != ND) return fail(h, KB_ERR_INVALID, "tas: level_start must cover [0, n_domains)");
  const int leaf0 = t->level_start[L - 1], NL = ND - leaf0;
  // Children of a domain are contiguous in the next level (lexicographic numbering) and the child ranges of level l
  // tile level l+1 in order, so one [ND+1] table serves as child_start[d] .. child_start[d+1]: the end of the last
  // domain of level l is level_start[l+2], which is also where the children of the first domain of level l+1 start.
  std::vector<int32_t> cstart(ND + 1, ND);
  for (int l = 0; l < L; l++) {
    int a = t->level_start[l], b = t->level_start[l + 1];
    if (b < a) return fail(h, KB_ERR_INVALID, "tas: level_start not monotone");
    for (int d = a; d < b; d++) {
      int p = t->parent[d];
      if (l == 0) { if (p != -1) return fail(h, KB_ERR_INVALID, "tas: level-0 domains have no parent"); continue; }
      if (p < t->level_start[l - 1] || p >= a) return fail(h, KB_ERR_INVALID, "tas: parent must be a domain of the previous level");
      if (d > a && p < t->parent[d - 1]) return fail(h, KB_ERR_INVALID, "tas: domains of a level must be numbered in lexicographic levelValues order (children of one parent contiguous)");
    }
    if (l + 1 < L) {
      int c = t->level_start[l + 1], ce = t->level_start[l + 2];
      for (int d = a; d < b; d++) { cstart[d] = c; while (c < ce && t->parent[c] == d) c++; }
      if (c != ce) return fail(h, KB_ERR_INVALID, "tas: a domain of the next level has no parent in this level");
    }
  }
  // chains, rounds, shape slots
  std::vector<int32_t> pred(std::max(1, NQ), -1), chain_slot(std::max(1, NQ), -1), pos(std::max(1, NQ), 0), slot(std::max(1, NQ), 0);
  int n_chain_slots = 0, n_rounds = 0, max_count = 1;
  for (int q = 0; q < NQ;) {
    int e = q;
    while (e + 1 < NQ && r->chain[e + 1] == r->chain[q]) e++;
    if (e + 1 < NQ && r->chain[e + 1] < r->chain[q]) return fail(h, KB_ERR_INVALID, "tas: chain ids must be non-decreasing");
    int len = e - q + 1;
    int cs = len > 1 ? n_chain_slots++ : -1;
    for (int i = q; i <= e; i++) { pos[i] = i - q; pred[i] = i > q ? i - 1 : -1; chain_slot[i] = cs; }
    n_rounds = std::max(n_rounds, len);
    q = e + 1;
  }
  for (int q = 0; q < NQ; q++) max_count = std::max(max_count, r->count[q]);
  const int ok_words = (NL + 31) / 32;
  std::vector<std::vector<int32_t>> round_req(n_rounds), round_slot_req(n_rounds);
  {
    std::map<std::string, int> shapes;  // round 0: requests with the same shape share the counts
    for (int q = 0; q < NQ; q++) {
      int rd = pos[q];
      round_req[rd].push_back(q);
      if (rd == 0) {
        std::string key((const char *)(r->pod_request + (size_t)q * R), (size_t)R * 8);
        key.append((const char *)&r->request_mask[q], 4);
        uint32_t fl = r->flags[q] & KB_TAS_SIMULATE_EMPTY; key.append((const char *)&fl, 4);
        key.append((const char *)&r->slice_size[q], 4); key.append((const char *)&r->slice_level[q], 4);
        if (r->leaf_ok) key.append((const char *)(r->leaf_ok + (size_t)q * ok_words), (size_t)ok_words * 4);
        auto it = shapes.find(key);
        if (it == shapes.end()) { it = shapes.emplace(key, (int)round_slot_req[0].size()).first; round_slot_req[0].push_back(q); }
        slot[q] = it->second;
      } else { slot[q] = (int)round_slot_req[rd].size(); round_slot_req[rd].push_back(q); }
    }
  }
  size_t max_slots = 1, max_round = 1;
  for (int rd = 0; rd < n_rounds; rd++) { max_slots = std::max(max_slots, round_slot_req[rd].size()); max_round = std::max(max_round, round_req[rd].size()); }
  // CountIn is negative on a leaf whose usage exceeds its free capacity (requests.go:196), or for a podset that follows a
  // simulate-empty one in its chain (the first placed against free alone).  The reference then emits negative counts
  // and more leaves than the podset's count (a negative domain is consumed without covering any pod).  Without either,
  // every listed domain holds at least one pod or slice, so count bounds a request's lists and output region; with
  // one, the kernel writes nothing past either, reports what it needed, and the batch runs again with that much.
  i64 neg_bits = 0;
  for (size_t i = 0; i < (size_t)NL * R; i++) neg_bits |= t->free_capacity[i] | (t->free_capacity[i] - t->tas_usage[i]);
  bool keep_zero = neg_bits < 0;
  for (int q = 1; q < NQ; q++)
    if (pred[q] >= 0 && ((r->flags[q] ^ r->flags[q - 1]) & KB_TAS_SIMULATE_EMPTY)) keep_zero = true;
  std::vector<int32_t> region(std::max(1, NQ)), tmp_start(NQ + 1, 0), n_out_h(std::max(1, NQ));
  for (int q = 0; q < NQ; q++) region[q] = std::max(0, std::min(r->count[q], NL));
  int list_cap = max_count + 8;
  for (int attempt = 0;; attempt++) {
    if (attempt == 64) return fail(h, KB_ERR_CAPACITY, "tas: lists / output regions still too small after 64 runs");
    {
      i64 tot_out = 0;  // offsets are int32 on the device
      for (int q = 0; q < NQ; q++) { tot_out += region[q]; if (tot_out > INT32_MAX - 1) return fail(h, KB_ERR_CAPACITY, "tas: output regions exceed 2^31 entries"); tmp_start[q + 1] = (int32_t)tot_out; }
    }
    // the per-CTA lists stay under 256 MiB: a long list_cap (over-used leaves) runs fewer CTAs, each walking more requests
    const int sel_grid = (int)std::max<size_t>(1, std::min<size_t>({max_round, (size_t)h->sm_count * 8, ((size_t)256 << 20) / ((size_t)24 * list_cap)}));
    // ---- device buffer (grow-only), described once (Arena::carve)
    TasDev T{};
    int32_t *d_asg_start, *d_round, *d_slotreq, *d_leaf, *d_cnt;
    const size_t n_tmp = (size_t)tmp_start[NQ] + 1, n_asg = (size_t)std::max(1, out->capacity);
    auto layout = [&](Arena &a) {
      T.level_start = a.take<int32_t>(L + 1); T.parent = a.take<int32_t>(ND); T.child_start = a.take<int32_t>(ND + 1);
      T.free_cap = a.take<i64>((size_t)NL * R); T.cap_mask = a.take<uint32_t>(NL);
      T.tas_usage = a.take<i64>((size_t)NL * R); T.usage_mask = a.take<uint32_t>(NL);
      T.pod_request = a.take<i64>((size_t)NQ * R); T.request_mask = a.take<uint32_t>(NQ);
      T.flags = a.take<uint32_t>(NQ); T.count = a.take<int32_t>(NQ);
      T.slice_size = a.take<int32_t>(NQ); T.level = a.take<int32_t>(NQ); T.slice_level = a.take<int32_t>(NQ);
      T.slot = a.take<int32_t>(NQ); T.chain_slot = a.take<int32_t>(NQ); T.pred = a.take<int32_t>(NQ);
      if (r->leaf_ok) T.leaf_ok = a.take<uint32_t>((size_t)NQ * ok_words);
      T.state = a.take<int32_t>(max_slots * ND); T.slice = a.take<int32_t>(max_slots * ND);
      T.assumed = a.take<i64>((size_t)n_chain_slots * NL * R); T.assumed_mask = a.take<uint32_t>((size_t)n_chain_slots * NL);
      T.status = a.take<int32_t>(NQ + 1); T.n_out = a.take<int32_t>(NQ + 1);
      d_asg_start = a.take<int32_t>(NQ + 2);
      T.tmp_start = a.take<int32_t>(NQ + 1); T.tmp_leaf = a.take<int32_t>(n_tmp); T.tmp_count = a.take<int32_t>(n_tmp);
      T.lists = a.take<int32_t>((size_t)sel_grid * 6 * list_cap);
      T.overflow = a.take<int32_t>(2);
      d_round = a.take<int32_t>(max_round); d_slotreq = a.take<int32_t>(max_slots);
      d_leaf = a.take<int32_t>(n_asg); d_cnt = a.take<int32_t>(n_asg);
    };
    if (!h->tas_arena.carve(layout)) return fail(h, KB_ERR_CUDA, "tas: cudaMalloc of the device buffer failed");
    T.L = L; T.n_domains = ND; T.n_leaves = NL; T.leaf0 = leaf0; T.R = R; T.pods_res = t->pods_resource; T.n_req = NQ;
    T.ok_words = ok_words; T.list_cap = list_cap; T.keep_zero = keep_zero;
    const size_t nq = (size_t)NQ, nl = (size_t)NL;
    const struct { const void *dst, *src; size_t bytes; } uploads[] = {
        {T.level_start, t->level_start, (size_t)(L + 1) * 4}, {T.parent, t->parent, (size_t)ND * 4}, {T.child_start, cstart.data(), (size_t)(ND + 1) * 4},
        {T.free_cap, t->free_capacity, nl * R * 8}, {T.cap_mask, t->cap_mask, nl * 4}, {T.tas_usage, t->tas_usage, nl * R * 8}, {T.usage_mask, t->usage_mask, nl * 4},
        {T.pod_request, r->pod_request, nq * R * 8}, {T.request_mask, r->request_mask, nq * 4}, {T.flags, r->flags, nq * 4}, {T.count, r->count, nq * 4},
        {T.slice_size, r->slice_size, nq * 4}, {T.level, r->level, nq * 4}, {T.slice_level, r->slice_level, nq * 4},
        {T.slot, slot.data(), nq * 4}, {T.chain_slot, chain_slot.data(), nq * 4}, {T.pred, pred.data(), nq * 4},
        {T.leaf_ok, r->leaf_ok, r->leaf_ok ? nq * ok_words * 4 : 0}, {T.tmp_start, tmp_start.data(), (nq + 1) * 4}};
    for (const auto &u : uploads) CUDA_TRY(h, h2d(h, u.dst, u.src, u.bytes));
    if (n_chain_slots) {
      CUDA_TRY(h, cudaMemsetAsync(T.assumed, 0, (size_t)n_chain_slots * nl * R * 8, h->stream));
      CUDA_TRY(h, cudaMemsetAsync(T.assumed_mask, 0, (size_t)n_chain_slots * nl * 4, h->stream));
    }
    CUDA_TRY(h, cudaMemsetAsync(T.overflow, 0, 8, h->stream));
    if (NQ) CUDA_TRY(h, cudaMemsetAsync(T.n_out, 0, (nq + 1) * 4, h->stream));
    CUDA_TRY(h, cudaEventRecord(h->ev2, h->stream));
    h->kev_n = 0;
    int launches = 0;
    for (int rd = 0; rd < n_rounds; rd++) {
      int ns = (int)round_slot_req[rd].size(), nr = (int)round_req[rd].size();
      CUDA_TRY(h, cudaMemcpyAsync(d_slotreq, round_slot_req[rd].data(), (size_t)ns * 4, cudaMemcpyHostToDevice, h->stream));
      CUDA_TRY(h, cudaMemcpyAsync(d_round, round_req[rd].data(), (size_t)nr * 4, cudaMemcpyHostToDevice, h->stream));
      if (rd == 0) kmark(h, KB_K_TAS_LEAF);
      k_tas_leaf<<<dim3((NL + 255) / 256, ns), 256, 0, h->stream>>>(T, d_slotreq, ns); launches++;
      if (rd == 0) kmark(h, KB_K_TAS_REDUCE);
      for (int l = L - 2; l >= 0; l--) {
        int n = t->level_start[l + 1] - t->level_start[l];
        k_tas_reduce<<<dim3((n + 127) / 128, ns), 128, 0, h->stream>>>(T, d_slotreq, ns, l); launches++;
      }
      if (rd == 0) kmark(h, KB_K_TAS_SELECT);
      k_tas_select<<<std::min(nr, sel_grid), KB_TAS_THREADS, 0, h->stream>>>(T, d_round, nr); launches++;
      if (rd == 0) kmark(h, KB_K_TAS);
    }
    if (NQ) {
      k_scan_i32<<<1, 1024, 0, h->stream>>>(T.n_out, d_asg_start, NQ); launches++;
      k_tas_compact<<<NQ, 64, 0, h->stream>>>(T, d_asg_start, d_leaf, d_cnt, out->capacity); launches++;
    }
    kmark(h, -1);
    CUDA_TRY(h, cudaEventRecord(h->ev3, h->stream));
    CUDA_TRY(h, cudaGetLastError());
    if (NQ) {
      CUDA_TRY(h, cudaMemcpyAsync(out->status, T.status, (size_t)NQ * 4, cudaMemcpyDeviceToHost, h->stream));
      CUDA_TRY(h, cudaMemcpyAsync(out->asg_start, d_asg_start, (size_t)(NQ + 1) * 4, cudaMemcpyDeviceToHost, h->stream));
    } else out->asg_start[0] = 0;
    int32_t ovf[2] = {0, 0};
    CUDA_TRY(h, cudaMemcpyAsync(ovf, T.overflow, 8, cudaMemcpyDeviceToHost, h->stream));
    CUDA_TRY(h, cudaStreamSynchronize(h->stream));
    if (ovf[0]) {  // grow what was short and run again
      CUDA_TRY(h, cudaMemcpy(n_out_h.data(), T.n_out, (size_t)NQ * 4, cudaMemcpyDeviceToHost));
      for (int q = 0; q < NQ; q++) region[q] = std::max(region[q], n_out_h[q]);
      if (ovf[1] + 8 > list_cap) list_cap = std::min(ovf[1], ND) + 8;
      continue;
    }
    out->n_assigned = out->asg_start[NQ];
    int ncopy = std::min(out->n_assigned, out->capacity);
    if (ncopy > 0) {
      CUDA_TRY(h, cudaMemcpy(out->asg_leaf, d_leaf, (size_t)ncopy * 4, cudaMemcpyDeviceToHost));
      CUDA_TRY(h, cudaMemcpy(out->asg_count, d_cnt, (size_t)ncopy * 4, cudaMemcpyDeviceToHost));
    }
    { float ms = 0; cudaEventElapsedTime(&ms, h->ev2, h->ev3); h->stats.last_cycle_gpu_ms = ms; }
    h->stats.kernel_launches = launches;
    for (int i = 0; i < KB_N_KERNELS; i++) h->stats.kernel_ms[i] = 0.f;
    for (int i = 0; i + 1 < h->kev_n; i++) {
      float kms = 0; cudaEventElapsedTime(&kms, h->kev[i], h->kev[i + 1]);
      if (h->kev_id[i] >= 0) h->stats.kernel_ms[h->kev_id[i]] += kms;
    }
    break;
  }
  if (out->n_assigned > out->capacity) return fail(h, KB_ERR_CAPACITY, "tas: assignment buffer too small");
  return KB_OK;
}

extern "C" int32_t kb_tree_eval(kb_handle *h, const kb_snapshot *s, kb_tree_out *out) {
  int32_t rc = kb_upload(h, s);
  if (rc != KB_OK) return rc;
  DevSnap &D = h->D;
  int launches = 0;
  launch_tree(h, &launches);
  k_drs<<<(D.N + 127) / 128, 128, 0, h->stream>>>(D, h->d_drs_rounded, h->d_drs_res, h->d_drs_borrowing);
  CUDA_TRY(h, cudaGetLastError());
  size_t NF = (size_t)D.N * D.FR, QF = (size_t)D.Q * D.FR;
  if (out->subtree_quota) CUDA_TRY(h, cudaMemcpyAsync(out->subtree_quota, D.subtree, NF * 8, cudaMemcpyDeviceToHost, h->stream));
  if (out->usage) CUDA_TRY(h, cudaMemcpyAsync(out->usage, D.usage, NF * 8, cudaMemcpyDeviceToHost, h->stream));
  if (out->available) CUDA_TRY(h, cudaMemcpyAsync(out->available, D.avail, QF * 8, cudaMemcpyDeviceToHost, h->stream));
  if (out->potential_available) CUDA_TRY(h, cudaMemcpyAsync(out->potential_available, D.potential, QF * 8, cudaMemcpyDeviceToHost, h->stream));
  if (out->drs_rounded) CUDA_TRY(h, cudaMemcpyAsync(out->drs_rounded, h->d_drs_rounded, (size_t)D.N * 8, cudaMemcpyDeviceToHost, h->stream));
  if (out->drs_resource) CUDA_TRY(h, cudaMemcpyAsync(out->drs_resource, h->d_drs_res, (size_t)D.N * 4, cudaMemcpyDeviceToHost, h->stream));
  if (out->drs_borrowing) CUDA_TRY(h, cudaMemcpyAsync(out->drs_borrowing, h->d_drs_borrowing, (size_t)D.N, cudaMemcpyDeviceToHost, h->stream));
  CUDA_TRY(h, cudaStreamSynchronize(h->stream));
  if (out->available) for (size_t i = 0; i < QF; i++) if (out->available[i] < 0) out->available[i] = 0;  // Available() clamps at the CQ (clusterqueue_snapshot.go:154-156)
  return KB_OK;
}

extern "C" int32_t kb_set_profile(kb_handle *h, int32_t on) {
  if (!h) return KB_ERR_INVALID;
  h->profile = on != 0;
  return KB_OK;
}

extern "C" int32_t kb_get_stats(const kb_handle *h, kb_stats *out) {
  if (!h || !out) return KB_ERR_INVALID;
  *out = h->stats;
  return KB_OK;
}
