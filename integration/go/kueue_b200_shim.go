// Package scheduler — drop-in shim that routes the decision part of Scheduler.schedule()
// (pkg/scheduler/scheduler.go:245-405) through libkueue_b200.
//
// STATUS: reference-side binding for maintainers.  It is NOT compiled in the repository's build image (there is
// no Go toolchain there); it restates, in the reference's own language and against the reference's own types, the
// host layer that IS built and tested in C++ (include/kueue_b200_host.hpp, tests/test_cpp_host.py) and Python
// (kueue_b200/api.py).  Field-by-field mapping: INTEGRATION.md §3.
//
// Placement: pkg/scheduler/kueue_b200_shim.go, build tag `kueue_b200`.  Nothing else in Kueue changes.

//go:build kueue_b200

package scheduler

/*
#cgo CFLAGS: -I${SRCDIR}/../../third_party/kueue_b200/include
#cgo LDFLAGS: -L${SRCDIR}/../../third_party/kueue_b200 -lkueue_b200
#include "kueue_b200.h"
*/
import "C"

import (
	"fmt"
	"math"
	"runtime"
	"slices"
	"sort"
	"unsafe"

	corev1 "k8s.io/api/core/v1"

	kueue "sigs.k8s.io/kueue/apis/kueue/v1beta2"
	schdcache "sigs.k8s.io/kueue/pkg/cache/scheduler"
	"sigs.k8s.io/kueue/pkg/features"
	"sigs.k8s.io/kueue/pkg/resources"
	afs "sigs.k8s.io/kueue/pkg/util/admissionfairsharing"
	"sigs.k8s.io/kueue/pkg/util/priority"
	utilqueue "sigs.k8s.io/kueue/pkg/util/queue"
	"sigs.k8s.io/kueue/pkg/workload"
)

// kbEvaluator owns one kb_handle (one CUDA device, one stream).  schedule() is single-goroutine
// (scheduler.go:188-194), which is exactly the library's threading contract.
type kbEvaluator struct {
	h         *C.kb_handle
	staticGen int64 // bumped by the cache whenever a ClusterQueue / Cohort spec changes
	// ONE page-locked block per evaluator, carved per cycle (bump allocator, reset at the top of every cycle): no
	// cudaHostAlloc on the cycle's path, nothing leaks, and the per-cycle tables sit in one span the library moves
	// with a single DMA (INTEGRATION.md §3).  It grows (free + allocate twice the size) when a cycle does not fit.
	arena    unsafe.Pointer
	arenaCap uintptr
	arenaOff uintptr
}

func newKBEvaluator(device int) (*kbEvaluator, error) {
	var h *C.kb_handle
	cfg := C.kb_config{device: C.int32_t(device)}
	if rc := C.kb_create(&cfg, &h); rc != 0 {
		return nil, fmt.Errorf("kb_create: %d %s", int(rc), C.GoString(C.kb_last_error(nil)))
	}
	return &kbEvaluator{h: h}, nil
}

// resetArena starts a new cycle: every slice handed out by pinned() in the previous cycle is dead after this call.
func (k *kbEvaluator) resetArena(need uintptr) {
	if need > k.arenaCap {
		if k.arena != nil {
			C.kb_free_pinned(k.arena)
		}
		k.arenaCap = 2 * need
		C.kb_alloc_pinned(&k.arena, C.uint64_t(k.arenaCap))
	}
	k.arenaOff = 0
}

// pinned carves a zeroed slice out of the evaluator's page-locked block (256-byte aligned like the library's device
// arena): the Go GC never moves it and C keeps no Go pointer after the call returns (cgo pointer rules).
func pinned[T any](k *kbEvaluator, n int) []T {
	var zero T
	bytes := (uintptr(max(n, 1))*unsafe.Sizeof(zero) + 255) &^ 255
	if k.arenaOff+bytes > k.arenaCap {
		panic("kueue_b200: per-cycle arena estimate too small") // resetArena sizes it from the snapshot's dimensions
	}
	p := unsafe.Add(k.arena, k.arenaOff)
	k.arenaOff += bytes
	s := unsafe.Slice((*T)(p), n)
	clear(s)
	return s
}

// flatSnapshot is kb_snapshot plus the name tables needed to read the outputs back.
type flatSnapshot struct {
	c         C.kb_snapshot
	cqs       []*schdcache.ClusterQueueSnapshot
	flavors   []kueue.ResourceFlavorReference
	resources []corev1.ResourceName
	admitted  []*workload.Info
}

func (f *flatSnapshot) fr(flavor kueue.ResourceFlavorReference, res corev1.ResourceName) int {
	return slices.Index(f.flavors, flavor)*len(f.resources) + slices.Index(f.resources, res)
}

const noLimit = int64(^uint64(0) >> 1) // KB_NO_LIMIT

// flatten: cache.Snapshot + queues.Heads -> SoA.  Same layout rules as kb::FlatSnapshot (kueue_b200_host.hpp):
// ClusterQueues first then Cohorts, fr = flavor*R + resource, resources sorted by name.
func (s *Scheduler) flatten(snap *schdcache.Snapshot, heads []workload.Info, gen int64) *flatSnapshot {
	f := &flatSnapshot{}
	cqNames := snap.ClusterQueuesNames()
	slices.Sort(cqNames)
	cohortNames := make([]kueue.CohortReference, 0)
	for name := range snap.Cohorts() {
		cohortNames = append(cohortNames, name)
	}
	slices.Sort(cohortNames)
	resSet := map[corev1.ResourceName]struct{}{}
	addFR := func(fr resources.FlavorResource) { // every flavor-resource that can index a table must be in the universe
		if !slices.Contains(f.flavors, fr.Flavor) {
			f.flavors = append(f.flavors, fr.Flavor)
		}
		resSet[fr.Resource] = struct{}{}
	}
	for _, n := range cqNames {
		cq := snap.ClusterQueue(n)
		f.cqs = append(f.cqs, cq)
		for _, rg := range cq.ResourceGroups {
			for _, fl := range rg.Flavors {
				if !slices.Contains(f.flavors, fl) {
					f.flavors = append(f.flavors, fl)
				}
			}
			for r := range rg.CoveredResources {
				resSet[r] = struct{}{}
			}
		}
		for fr := range cq.ResourceNode.Usage { // usage on a flavor the ClusterQueue no longer defines
			addFR(fr)
		}
		for _, wi := range cq.Workloads { // admitted usage (preemption candidates)
			for fr := range wi.FlavorResourceUsage() {
				addFR(fr)
			}
		}
	}
	for _, name := range cohortNames { // quotas defined at cohort level only
		for fr := range snap.Cohort(name).ResourceNode.Quotas {
			addFR(fr)
		}
	}
	for i := range heads {
		for _, ps := range heads[i].TotalRequests {
			for r := range ps.Requests {
				resSet[r] = struct{}{}
			}
		}
	}
	for r := range resSet {
		f.resources = append(f.resources, r)
	}
	sort.Slice(f.resources, func(i, j int) bool { return f.resources[i] < f.resources[j] }) // DRS tie-break compares names
	Q, C_, F, R := len(cqNames), len(cohortNames), len(f.flavors), len(f.resources)
	N, FR := Q+C_, F*R
	k := s.kb
	{ // size the page-locked block for this cycle: node tables + entries + admitted workloads + outputs, with slack
		nAdm, nPs := 0, 0
		for _, cq := range f.cqs {
			nAdm += len(cq.Workloads)
		}
		for i := range heads {
			nPs += len(heads[i].TotalRequests)
		}
		k.resetArena(uintptr(N*FR*32+N*64+Q*64+nAdm*(64+16*R)+len(heads)*128+nPs*(R*12+64)) + 1<<20)
	}

	parent := pinned[int32](k, N)
	weight := pinned[float64](k, N)
	nominal, blimit, llimit := pinned[int64](k, N*FR), pinned[int64](k, N*FR), pinned[int64](k, N*FR)
	usage := pinned[int64](k, Q*FR)
	for i := range blimit {
		blimit[i], llimit[i] = noLimit, noLimit
	}
	quotas := func(n int, q map[resources.FlavorResource]schdcache.ResourceQuota) {
		for fr, rq := range q {
			c := n*FR + f.fr(fr.Flavor, fr.Resource)
			nominal[c] = rq.Nominal
			if rq.BorrowingLimit != nil {
				blimit[c] = *rq.BorrowingLimit
			}
			if rq.LendingLimit != nil {
				llimit[c] = *rq.LendingLimit
			}
		}
	}
	cohortIdx := func(name kueue.CohortReference) int32 { return int32(Q + slices.Index(cohortNames, name)) }
	// ---- ClusterQueue tables
	within, reclaim, bwc := pinned[uint8](k, Q), pinned[uint8](k, Q), pinned[uint8](k, Q)
	hasThr, thr := pinned[uint8](k, Q), pinned[int32](k, Q)
	wcb, wcp, pref, strat, cqGen := pinned[uint8](k, Q), pinned[uint8](k, Q), pinned[uint8](k, Q), pinned[uint8](k, Q), pinned[int64](k, Q)
	var rgStart, rgMask, rgFlStart, rgFl []int32
	rgStart, rgFlStart = append(rgStart, 0), append(rgFlStart, 0)
	for i, cq := range f.cqs {
		parent[i] = -1
		if cq.HasParent() {
			parent[i] = cohortIdx(cq.Parent().GetName())
		}
		weight[i] = cq.FairWeight
		quotas(i, cq.ResourceNode.Quotas)
		for fr, q := range cq.ResourceNode.Usage {
			usage[i*FR+f.fr(fr.Flavor, fr.Resource)] = q
		}
		within[i], reclaim[i] = policyCode(cq.Preemption.WithinClusterQueue), policyCode(cq.Preemption.ReclaimWithinCohort)
		if b := cq.Preemption.BorrowWithinCohort; b != nil && b.Policy != kueue.BorrowWithinCohortPolicyNever {
			bwc[i] = C.KB_POLICY_LOWER_PRIORITY
			if b.MaxPriorityThreshold != nil {
				hasThr[i], thr[i] = 1, *b.MaxPriorityThreshold
			}
		}
		wcb[i], wcp[i], pref[i] = fungibilityCodes(cq.FlavorFungibility)
		if s.queues.QueueingStrategy(cq.Name) == kueue.StrictFIFO { // read by kb_run_drain's requeue rules
			strat[i] = C.KB_QUEUE_STRICT_FIFO
		}
		cqGen[i] = cq.AllocatableResourceGeneration
		for _, rg := range cq.ResourceGroups {
			var mask int32
			for r := range rg.CoveredResources {
				mask |= 1 << slices.Index(f.resources, r)
			}
			rgMask = append(rgMask, mask)
			for _, fl := range rg.Flavors {
				rgFl = append(rgFl, int32(slices.Index(f.flavors, fl)))
			}
			rgFlStart = append(rgFlStart, int32(len(rgFl)))
		}
		rgStart = append(rgStart, int32(len(rgMask)))
	}
	for j, name := range cohortNames {
		co := snap.Cohort(name)
		parent[Q+j] = -1
		if co.HasParent() {
			parent[Q+j] = cohortIdx(co.Parent().GetName())
		}
		weight[Q+j] = co.FairWeight
		quotas(Q+j, co.ResourceNode.Quotas)
	}
	// ---- admitted workloads (preemption candidates), per ClusterQueue in name order
	var admCq, admPrio, admUseStart, admFr []int32
	var admTs, admQr, admUID, admQty []int64
	var admEv []uint8
	admUseStart = append(admUseStart, 0)
	for i, cq := range f.cqs {
		keys := make([]workload.Reference, 0, len(cq.Workloads))
		for k := range cq.Workloads {
			keys = append(keys, k)
		}
		slices.Sort(keys)
		for _, k := range keys {
			wi := cq.Workloads[k]
			f.admitted = append(f.admitted, wi)
			admCq, admPrio = append(admCq, int32(i)), append(admPrio, priority.Priority(wi.Obj))
			admTs = append(admTs, s.workloadOrdering.GetQueueOrderTimestamp(wi.Obj).UnixNano())
			admQr = append(admQr, quotaReservedNs(wi.Obj)) // INT64_MIN when the condition is missing (ordering.go:93-100)
			admEv = append(admEv, b2u(workload.IsEvicted(wi.Obj)))
			for fr, q := range wi.FlavorResourceUsage() {
				admFr, admQty = append(admFr, int32(f.fr(fr.Flavor, fr.Resource))), append(admQty, q)
			}
			admUseStart = append(admUseStart, int32(len(admFr)))
		}
	}
	uidRank(f.admitted, &admUID) // dense ranks consistent with the UID string order
	// ---- entries of this cycle
	var wlCq, wlPrio, wlPsStart, psCount, psMin, psMask []int32
	var wlTs, wlUID, wlGen, psReq []int64
	var psOk []uint64
	var psLast []int8
	var psGroup []int32 // PodSetGroupName as a per-workload id, -1 = none (flavorassigner.go:613-616)
	anyGroup := false
	wlPsStart = append(wlPsStart, 0)
	for i := range heads {
		w := &heads[i]
		ci := slices.IndexFunc(f.cqs, func(c *schdcache.ClusterQueueSnapshot) bool { return c.Name == w.ClusterQueue })
		wlCq, wlPrio = append(wlCq, int32(ci)), append(wlPrio, priority.Priority(w.Obj))
		wlTs = append(wlTs, s.workloadOrdering.GetQueueOrderTimestamp(w.Obj).UnixNano())
		gen := int64(-1)
		if w.LastAssignment != nil {
			gen = w.LastAssignment.ClusterQueueGeneration
		}
		wlGen = append(wlGen, gen)
		var groupNames []string
		for pi, ps := range w.TotalRequests {
			gid := int32(-1)
			if tr := w.Obj.Spec.PodSets[pi].TopologyRequest; tr != nil && tr.PodSetGroupName != nil {
				k := slices.Index(groupNames, *tr.PodSetGroupName)
				if k < 0 {
					groupNames, k = append(groupNames, *tr.PodSetGroupName), len(groupNames)
				}
				gid, anyGroup = int32(k), true
			}
			psGroup = append(psGroup, gid)
			row := make([]int64, R)
			last := make([]int8, R)
			var mask int32
			for r, q := range ps.Requests {
				ri := slices.Index(f.resources, r)
				row[ri], mask = q, mask|1<<ri // TotalRequests already holds Count pods (workload.go:567-598)
			}
			for ri := range last {
				last[ri] = -1
			}
			if w.LastAssignment != nil && pi < len(w.LastAssignment.LastTriedFlavorIdx) {
				for r, idx := range w.LastAssignment.LastTriedFlavorIdx[pi] {
					last[slices.Index(f.resources, r)] = int8(idx)
				}
			}
			minCount := int32(-1)
			if mc := w.Obj.Spec.PodSets[pi].MinCount; mc != nil && features.Enabled(features.PartialAdmission) {
				minCount = *mc
			}
			psReq, psLast = append(psReq, row...), append(psLast, last...)
			psMask, psCount, psMin = append(psMask, mask), append(psCount, ps.Count), append(psMin, minCount)
			psOk = append(psOk, s.eligibleFlavors(w, pi, f.cqs[ci], f.flavors)) // checkFlavorForPodSets flavorassigner.go:899-944
		}
		wlPsStart = append(wlPsStart, int32(len(psCount)))
	}
	wlUIDRank(heads, &wlUID)
	headsIdx := make([]int32, len(heads))
	for i := range headsIdx {
		headsIdx[i] = int32(i)
	}
	// ---- struct (cp32 / cp64 / ... copy a Go slice into the evaluator's pinned block: pinned[T](k, len) + copy)
	c := &f.c
	c.n_cq, c.n_cohort, c.n_flavor, c.n_resource = C.int32_t(Q), C.int32_t(C_), C.int32_t(F), C.int32_t(R)
	c.n_rg, c.n_wl, c.n_podset = C.int32_t(len(rgMask)), C.int32_t(len(heads)), C.int32_t(len(psCount))
	c.n_adm, c.n_adm_use, c.n_heads = C.int32_t(len(admCq)), C.int32_t(len(admFr)), C.int32_t(len(heads))
	c.pods_resource = C.int32_t(slices.Index(f.resources, corev1.ResourcePods))
	c.flags, c.now_ns, c.static_generation = C.uint32_t(s.kbFlags()), C.int64_t(s.clock.Now().UnixNano()), C.int64_t(gen)
	c.parent, c.fair_weight = (*C.int32_t)(&parent[0]), (*C.double)(&weight[0])
	c.nominal, c.borrow_limit, c.lend_limit = (*C.int64_t)(&nominal[0]), (*C.int64_t)(&blimit[0]), (*C.int64_t)(&llimit[0])
	c.cq_usage = (*C.int64_t)(&usage[0])
	// Incremental form (kb_snapshot.usage_delta_*, INTEGRATION.md "Usage deltas"): once a call carried the full table with
	// KB_F_USAGE_RESIDENT, a cache that tracks which ClusterQueues it touched since the previous cycle passes only those rows:
	//   c.n_usage_delta, c.usage_delta_cq, c.usage_delta_rows = n, &dirtyCQ[0], &dirtyRows[0]   (c.cq_usage may stay nil)
	// This shim always sends the full table.
	c.cq_within_cq, c.cq_reclaim_within, c.cq_borrow_within = (*C.uint8_t)(&within[0]), (*C.uint8_t)(&reclaim[0]), (*C.uint8_t)(&bwc[0])
	c.cq_has_bwc_threshold, c.cq_bwc_threshold = (*C.uint8_t)(&hasThr[0]), (*C.int32_t)(&thr[0])
	c.cq_when_can_borrow, c.cq_when_can_preempt, c.cq_preference = (*C.uint8_t)(&wcb[0]), (*C.uint8_t)(&wcp[0]), (*C.uint8_t)(&pref[0])
	c.cq_strategy, c.cq_generation = (*C.uint8_t)(&strat[0]), (*C.int64_t)(&cqGen[0])
	c.cq_rg_start, c.rg_res_mask = cp32(rgStart), (*C.uint32_t)(unsafe.Pointer(cp32(rgMask)))
	c.rg_flavor_start, c.rg_flavors = cp32(rgFlStart), cp32(rgFl)
	c.wl_cq, c.wl_priority, c.wl_ts, c.wl_uid, c.wl_last_gen = cp32(wlCq), cp32(wlPrio), cp64(wlTs), cp64(wlUID), cp64(wlGen)
	c.wl_ps_start, c.ps_req, c.ps_req_mask = cp32(wlPsStart), cp64(psReq), (*C.uint32_t)(unsafe.Pointer(cp32(psMask)))
	c.ps_count, c.ps_min_count, c.ps_flavor_ok, c.ps_last_tried = cp32(psCount), cp32(psMin), cpU64(psOk), cpI8(psLast)
	c.adm_cq, c.adm_priority, c.adm_ts, c.adm_qr_ts, c.adm_uid = cp32(admCq), cp32(admPrio), cp64(admTs), cp64(admQr), cp64(admUID)
	c.adm_evicted, c.adm_use_start, c.adm_use_fr, c.adm_use_qty = cpU8(admEv), cp32(admUseStart), cp32(admFr), cp64(admQty)
	c.heads = cp32(headsIdx)
	// Eviction replay in kb_run_drain (kb_snapshot.adm_wl, INTEGRATION.md): before the copies above, append one pending
	// record per admitted workload (its ClusterQueue, priority, queue-order timestamp, UID and podsets with full counts, as
	// it would be requeued) and keep its index:
	//   admWl[a] = int32(len(wlCq)); wlCq = append(wlCq, admCq[a]); ...   then c.adm_wl = cp32(admWl)
	// This shim runs single cycles and leaves c.adm_wl nil.
	// Arrivals and completions in kb_run_drain (INTEGRATION.md): a queue simulation fills one creation time per pending
	// workload and one run time, plus one finish time per admitted workload, and the length of one cycle:
	//   c.wl_create_ns, c.wl_run_ns, c.adm_finish_ns = cp64(wlCreate), cp64(wlRun), cp64(admFinish); c.drain_cycle_ns = C.int64_t(cycleNs)
	// With eviction replay it may also fill each workload's eviction latency (until its pods are gone) and, for the
	// admitted workloads already evicted, the time their quota is released (read where adm_evicted is set):
	//   c.wl_evict_ns, c.adm_evict_end_ns = cp64(wlEvict), cp64(admEvictEnd)
	// The sticky workload of every ClusterQueue (INTEGRATION.md) comes from an accessor in pkg/cache/queue, since the
	// field sw is unexported, mapped to its pending index (-1 = none):
	//   c.cq_sticky = cp32(cqSticky)   // after kb_run_drain, kb_drain_out.cq_sticky is written back through a setter
	// Admission checks (INTEGRATION.md): a modelled check delay and fail count per workload, and the start state read from
	// Status.AdmissionChecks[*].RetryCount, Status.RequeueState.RequeueAt, the Evicted condition (reason AdmissionCheck)
	// and ProvisioningRequestConfig.Spec.RetryStrategy:
	//   c.wl_check_ns, c.wl_check_fail, c.wl_check_retries = cp64(chkNs), cp32(chkFail), cp32(retryCount)
	//   c.wl_check_evict_ns, c.wl_requeue_at_ns, c.adm_check_end_ns = cp64(evictedAt), cp64(requeueAt), cp64(checkEnd)
	//   c.check_backoff_base_s, c.check_backoff_max_s, c.check_backoff_limit = base, max, limit
	// WaitForPodsReady (INTEGRATION.md): a modelled PodsReady delay and fail count per workload, the settings from
	// Configuration.WaitForPodsReady (timeout, RequeuingStrategy; BlockAdmission true keeps the Go path), and the start
	// state from Status.RequeueState.Count / RequeueAt and the Admitted, PodsReady and Evicted (reason PodsReadyTimeout)
	// conditions:
	//   c.wl_pods_ready_ns, c.wl_pods_ready_fail, c.wl_pods_ready_count = cp64(readyNs), cp32(readyFail), cp32(requeueCount)
	//   c.wl_pods_ready_evict_ns, c.adm_admitted_ns = cp64(timeoutEvictedAt), cp64(admittedNotReadyAt)
	//   c.pods_ready_timeout_ns, c.pods_ready_backoff_base_s, c.pods_ready_backoff_max_s = timeout, base, max
	//   c.pods_ready_backoff_limit, c.pods_ready_requeue_creation = limitOrMinus1, creation
	// MaximumExecutionTimeSeconds (INTEGRATION.md): the limit from Spec.MaximumExecutionTimeSeconds (nil = 0), the
	// accumulated time from Status.AccumulatedPastExecutionTimeSeconds (nil = -1), and each admitted row's Admitted time
	// from the Admitted condition's LastTransitionTime (math.MinInt64 while its checks are not all Ready):
	//   c.wl_max_exec_s, c.wl_exec_acc_s, c.adm_exec_since_ns = cp32(maxExecS), cp32(accS), cp64(admittedAt)
	// Quota changes (INTEGRATION.md): planned ClusterQueue / Cohort edits, one per node and time, sorted by time, each
	// with the node's full rows after the change; kb_drain_out.cq_generation is written back after the drain:
	//   c.n_quota_change, c.qc_ns, c.qc_node = C.int32_t(len(editNs)), cp64(editNs), cp32(editNode)
	//   c.qc_nominal, c.qc_borrow_limit, c.qc_lend_limit = cp64(editNominal), cp64(editBorrow), cp64(editLend)
	// Deactivation and reactivation (INTEGRATION.md): the start state from !workload.IsActive (0 when active, else the
	// reason of the deactivation in force: 1 Rejected, 2 RequeuingLimitExceeded, 3 MaximumExecutionTimeExceeded, 4 a
	// user's stop, read from the Evicted condition's reason), and planned stop / resume edits sorted by time:
	//   c.wl_inactive = cpU8(inactiveReason)
	//   c.n_active_change, c.ac_ns, c.ac_wl, c.ac_active = C.int32_t(len(acNs)), cp64(acNs), cp32(acWl), cpU8(acActive)
	// Reclaim steps (INTEGRATION.md): ps_count / ps_req after Status.ReclaimablePods (spec Count - reclaimable), planned
	// steps per record (the podset's count after each step, relative to the run start), each admitted row's
	// Admission.PodSetAssignments[].Flavors / Count / ResourceUsage, and its run start from the Admitted condition's
	// LastTransitionTime (the PodsReady condition's with waitForPodsReady; math.MinInt64 while the row does not run);
	// Status.ReclaimablePods = spec Count - kb_drain_out.ps_remaining_out is written back after the drain:
	//   c.n_reclaim, c.wl_rc_start, c.rc_after_ns, c.rc_ps, c.rc_remaining = C.int32_t(len(rcAfter)), cp32(rcStart), cp64(rcAfter), cp32(rcPs), cp32(rcRemaining)
	//   c.ps_adm_flavor, c.ps_adm_count, c.ps_adm_usage, c.adm_run_start_ns = cp8(admFlavor), cp32(admCount), cp64(admUsage), cp64(runStart)
	// They stay nil here: a single cycle ignores them.
	if anyGroup { // optional table: NULL when no podset is grouped
		c.ps_group = cp32(psGroup)
	}
	return f
}

// flattenAFS fills the AdmissionFairSharing tables of a drain snapshot (kb_snapshot.wl_lq ..., include/kueue_b200.h)
// from the queue manager and the Configuration; wlQueue[w] is the LocalQueue key of pending workload w.  Without
// afs.Enabled the tables stay NULL.  A consumed quantity in inf.Dec form has no (value, scale) pair: the caller runs the
// Go path.
func (s *Scheduler) flattenAFS(f *flat, wlQueue []utilqueue.LocalQueueReference) error {
	if !afs.Enabled(s.admissionFairSharing) {
		return nil
	}
	R := len(f.resources)
	var lqKeys []utilqueue.LocalQueueReference // ClusterQueue-major
	var lqCq []int32
	var lqWeight []float64
	for ci, cq := range f.cqs {
		for _, key := range s.queues.LocalQueuesOf(cq.Name) { // sorted keys of the LocalQueues feeding cq
			lqKeys, lqCq = append(lqKeys, key), append(lqCq, int32(ci))
			lqWeight = append(lqWeight, s.queues.LocalQueueFairSharingWeight(key)) // Weight.AsApproximateFloat64(), 1.0 when nil
		}
	}
	cqAfs := make([]uint8, len(f.cqs))
	for ci, cq := range f.cqs {
		on, _ := afs.ResourceWeights(cq.AdmissionScope, s.admissionFairSharing)
		cqAfs[ci] = b2u(on)
	}
	consumed, scale, penalty := make([]int64, len(lqKeys)*R), make([]int32, len(lqKeys)*R), make([]int64, len(lqKeys)*R)
	for l, key := range lqKeys {
		if entry, ok := s.queues.AfsConsumedResources.Get(key); ok {
			for r, q := range entry.Resources {
				v, sc, ok := q.AsScaledInt64Pair() // (value, scale) of the int64Amount form; false for inf.Dec
				if !ok {
					return fmt.Errorf("afs: consumed %s of %s is not an int64Amount", r, key)
				}
				consumed[l*R+slices.Index(f.resources, r)], scale[l*R+slices.Index(f.resources, r)] = v, int32(sc)
			}
		}
		for r, q := range s.queues.AfsEntryPenalties.Peek(key) {
			penalty[l*R+slices.Index(f.resources, r)] = q.MilliValue()
		}
	}
	resWeight, milliMul := make([]float64, R), make([]int64, R)
	for ri, r := range f.resources {
		resWeight[ri], milliMul[ri] = 1, 1000
		if w, ok := s.admissionFairSharing.ResourceWeights[r]; ok {
			resWeight[ri] = w
		}
		if r == corev1.ResourceCPU {
			milliMul[ri] = 1 // the library keeps cpu in milli-units (pkg/resources/requests.go:104-109)
		}
	}
	wlLq := make([]int32, len(wlQueue))
	for w, key := range wlQueue {
		wlLq[w] = int32(slices.Index(lqKeys, key))
	}
	cfg := s.admissionFairSharing
	alpha := 0.0
	if cfg.UsageHalfLifeTime.Seconds() != 0 { // calculateAlphaRate (admission_fair_sharing.go): Go's math.Pow bits
		alpha = 1.0 - math.Pow(0.5, cfg.UsageSamplingInterval.Seconds()/cfg.UsageHalfLifeTime.Seconds())
	}
	c := &f.c
	c.n_lq, c.wl_lq, c.lq_cq, c.cq_afs = C.int32_t(len(lqKeys)), cp32(wlLq), cp32(lqCq), cpU8(cqAfs)
	c.lq_weight, c.lq_consumed, c.lq_consumed_scale = cpF64(lqWeight), cp64(consumed), cp32(scale)
	c.lq_penalty, c.afs_res_weight, c.afs_milli_mul, c.afs_alpha = cp64(penalty), cpF64(resWeight), cp64(milliMul), C.double(alpha)
	// Decay of consumed usage in an event drain (INTEGRATION.md): a LocalQueue without a cache entry is initialised as
	// initializeAfsIfNeeded does (consumed = its admitted usage, LastUpdate = now), then
	//   c.afs_half_life_ns, c.afs_sampling_ns = C.int64_t(cfg.UsageHalfLifeTime.Nanoseconds()), C.int64_t(cfg.UsageSamplingInterval.Nanoseconds())
	//   c.lq_last_update_ns, c.adm_lq = cp64(lastUpdate), cp32(admLq)   // entry.LastUpdate.UnixNano(); LocalQueue per admitted row, -1 for none
	// and after kb_run_drain: s.queues.AfsConsumedResources.Set(key, consumed from out.lq_consumed / lq_consumed_scale,
	// time.Unix(0, out.lq_last_update_ns[l])).  A single cycle leaves them nil.
	return nil
}

// scheduleKB replaces nominate + makeIterator + the decision part of the loop (scheduler.go:255-401) and replays
// the side effects in the order the library committed the entries.
func (s *Scheduler) scheduleKB(heads []workload.Info, snap *schdcache.Snapshot) ([]entry, error) {
	f := s.flatten(snap, heads, s.kb.staticGen)
	H, P, R := len(heads), int(f.c.n_podset), len(f.resources)
	k := s.kb // outputs come from the same per-cycle block as the inputs (flatten reset it)
	decision, mode := pinned[uint8](k, H), pinned[uint8](k, H)
	borrow, rank := pinned[int32](k, H), pinned[int32](k, H)
	psFlavor, psMode, psTried := pinned[int8](k, P*R), pinned[int8](k, P*R), pinned[int8](k, P*R)
	psCount, tgtStart := pinned[int32](k, P), pinned[int32](k, H+1)
	capT := 4*int(f.c.n_adm) + 1024
	tgtAdm, tgtReason := pinned[int32](k, capT), pinned[uint8](k, capT)
	out := C.kb_cycle_out{decision: (*C.uint8_t)(&decision[0]), mode: (*C.uint8_t)(&mode[0]), borrow: (*C.int32_t)(&borrow[0]),
		commit_rank: (*C.int32_t)(&rank[0]), ps_flavor: (*C.int8_t)(&psFlavor[0]), ps_res_mode: (*C.int8_t)(&psMode[0]),
		ps_tried_idx: (*C.int8_t)(&psTried[0]), ps_count: (*C.int32_t)(&psCount[0]), tgt_start: (*C.int32_t)(&tgtStart[0]),
		tgt_adm: (*C.int32_t)(&tgtAdm[0]), tgt_reason: (*C.uint8_t)(&tgtReason[0]), tgt_capacity: C.int32_t(capT)}
	runtime.LockOSThread() // CUDA context affinity; kb_run_cycle is blocking and not re-entrant per handle
	rc := C.kb_run_cycle(s.kb.h, &f.c, &out)
	runtime.UnlockOSThread()
	if rc != 0 { // any error: the caller runs the stock Go cycle, outputs are not consumed
		return nil, fmt.Errorf("kb_run_cycle: %d %s", int(rc), C.GoString(C.kb_last_error(s.kb.h)))
	}
	type ranked struct {
		entry
		root, rank int32
	}
	entries := make([]ranked, H)
	row := 0
	for e := range heads {
		en := &entries[e]
		en.rank = rank[e]
		en.Info = heads[e]
		en.clusterQueueSnapshot = f.cqs[slices.IndexFunc(f.cqs, func(c *schdcache.ClusterQueueSnapshot) bool { return c.Name == heads[e].ClusterQueue })]
		en.assignment = s.assignmentFromRows(f, &heads[e], row, psFlavor, psMode, psTried, psCount, int(borrow[e])) // Flavors/Mode/TriedFlavorIdx/Count/Usage
		row += len(heads[e].TotalRequests)
		for k := tgtStart[e]; k < tgtStart[e+1]; k++ {
			en.preemptionTargets = append(en.preemptionTargets, s.targetFrom(f.admitted[tgtAdm[k]], tgtReason[k])) // preemption.go:111-115
		}
		switch decision[e] {
		case C.KB_DEC_ASSUMED:
			en.status = assumed // admit() is replayed by the caller (scheduler.go:397-400)
		case C.KB_DEC_PREEMPTING:
			en.status = nominated // IssuePreemptions (:344-359)
		case C.KB_DEC_SKIPPED_OVERLAP, C.KB_DEC_SKIPPED_NO_FIT:
			en.status = skipped
		}
	}
	// replay order: the iterator's pop order inside every root cohort (commit_rank, scheduler.go:269).  The rank
	// travels WITH the entry so the comparator stays consistent while the slice is permuted; root cohorts are
	// independent, so interleaving them by rank is as good as any other order.
	sort.SliceStable(entries, func(i, j int) bool { return entries[i].rank < entries[j].rank })
	ordered := make([]entry, H)
	for i := range entries {
		ordered[i] = entries[i].entry
	}
	return ordered, nil
}

func policyCode(p kueue.PreemptionPolicy) uint8 {
	switch p {
	case kueue.PreemptionPolicyLowerPriority:
		return C.KB_POLICY_LOWER_PRIORITY
	case kueue.PreemptionPolicyLowerOrNewerEqualPriority:
		return C.KB_POLICY_LOWER_OR_NEWER_EQUAL_PRIORITY
	case kueue.PreemptionPolicyAny:
		return C.KB_POLICY_ANY
	}
	return C.KB_POLICY_NEVER
}

func b2u(b bool) uint8 {
	if b {
		return 1
	}
	return 0
}

// Small helpers left to the integrator (each a few lines): fungibilityCodes, quotaReservedNs, uidRank / wlUIDRank,
// cp32 / cp64 / cpU8 / cpI8 / cpU64 / cpF64 (copy a Go slice into pinned memory and return the C pointer),
// LocalQueuesOf / LocalQueueFairSharingWeight (queue-manager lookups), Quantity.AsScaledInt64Pair (the int64Amount
// fields of a resource.Quantity),
// (*Scheduler).eligibleFlavors (checkFlavorForPodSets per flavor -> bitmask), kbFlags (feature gates -> KB_F_*),
// assignmentFromRows and targetFrom (output rows -> flavorassigner.Assignment / preemption.Target).
