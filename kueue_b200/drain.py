"""Drain mode (SURVEY.md §8d): iterate scheduling cycles over a snapshot whose pending tables hold whole queues.

This module is the HOST DEFINITION of the drain (numpy bookkeeping around any single-cycle evaluator); the product
path is kb_run_drain (include/kueue_b200.h), which keeps the queue layer on the device.  tests/test_drain.py runs this
loop on the oracle and compares kb_run_drain with it cycle by cycle.

  * per ClusterQueue the pending workloads are ordered once by queueOrderingFunc
    (pkg/cache/queue/cluster_queue.go:636-685: priority desc, queue-order timestamp, UID);
  * every cycle takes the current head of every ClusterQueue (queues.Heads, manager.go:770-794), runs ONE cycle and
    applies its decisions the way schedule() + requeueAndUpdate (scheduler.go:405-418,823-850) do:
      - Assumed: the workload leaves the queue, its Assignment.Usage is added to the ClusterQueue usage and it joins
        the admitted tables (a preemption candidate of later cycles);
      - every other entry keeps `LastAssignment = &assignment.LastState` (scheduler.go:494): the next attempt starts
        after the flavors already tried (ps_tried_idx -> ps_last_tried, ClusterQueueGeneration -> wl_last_gen);
        a Preempting entry gets LastAssignment = nil (scheduler.go:345);
      - StrictFIFO: the entry stays the head (requeue is immediate, cluster_queue.go:622-624);
      - BestEffortFIFO: skipped entries (FailedAfterNomination) and pending preemptions stay (immediate requeue);
        NoFit / Preempt-without-targets entries stay when LastAssignment.PendingFlavors() (cluster_queue.go:372,
        workload.go:163-176) and otherwise go to the inadmissible set: the next workload becomes the head;
      - BestEffortFIFO, mode NoFit, known SchedulingHash: every queued workload of the same equivalence class moves to
        the inadmissible set as well (handleInadmissibleHash, cluster_queue.go:408-425; scheduler.go:292-300);
  * the drain ends with the first cycle that admits nothing and evicts nothing (no cluster event can change the outcome
    after that).  Without `adm_wl` evictions are not replayed: a Preempting entry keeps its place and its targets stay
    admitted.

Queue state: every pending workload is QUEUED, SET_ASIDE (the inadmissible set: BestEffortFIFO requeue or the hash
bulk move) or HELD (holds quota: admitted in the drain, or named by `adm_wl`).  The head of a queue is its first QUEUED
workload in the static order; the cursor of a segment is the position of that workload (no QUEUED workload before it).

Eviction replay (the snapshot carries `adm_wl`, include/kueue_b200.h).  In the reference an eviction completes
asynchronously (the job is suspended, the pods terminate); the drain takes the limit in which every eviction issued in
cycle c completes before cycle c+1.  After cycle c, in this order:
  1. the decisions are applied as above;
  2. every target of every Preempting entry leaves the admitted tables (the QuotaReserved -> Pending transition of
     workload_controller.go:973-1004): its cells leave its ClusterQueue's usage (cache.DeleteWorkload), its row is
     removed (the other rows keep their order) and its pending record `adm_wl[row]` is QUEUED again with
     LastAssignment nil (wl_last_gen = -1, ps_last_tried = -1, HasQuotaReservation false).  Preemption evictions set
     no RequeueState (only PodsReady timeouts do, workload_controller.go:827-832), so the requeue is immediate.
     Targets that already carried adm_evicted count too (IssuePreemptions, preemption.go:183-186); evictions under way
     before the drain are not completed;
  3. QueueAssociatedInadmissibleWorkloadsAfter (manager.go:670-697 -> notifyRetryInadmissibleWithoutLock,
     inadmissible_workloads.go:128-223): for every root cohort with an evicted workload in its tree (the ClusterQueue
     itself when it has no cohort) every SET_ASIDE workload of its ClusterQueues is QUEUED again, keeping its
     LastAssignment; noFitSchedulingHashes is cleared with them (`requeue_inadmissible`);
  4. the head of every queue in cycle c+1 is its first QUEUED workload: a requeued victim takes the place its
     priority, timestamp and UID give it (with PrioritySortingWithinCohort the queue-order timestamp of a preempted
     workload is its creation timestamp, workload.go:1174-1193, so the static order holds).

AdmissionFairSharing (the snapshot carries `wl_lq` and the LocalQueue tables, include/kueue_b200.h): the queue of a
ClusterQueue with `cq_afs` set is one segment per LocalQueue, each in the static order above with its own cursor.
  * the head is the minimum of (LocalQueue usage by cmp.Compare, -priority, timestamp, UID) over the segment heads
    (queueOrderingFunc with enableAdmissionFs, cluster_queue.go:636-685; kb_run_drain refuses a sticky workload here,
    and without preemption none arises).  After penalties the reference's Pop re-heapifies in map order (rebuildAll,
    cluster_queue.go:494-531; heap.go:115-123, 166-172) and may return a workload that is not the minimum: the true
    minimum is this definition's canonical rule;
  * LocalQueue usage is `lq_usage` (Info.CalcLocalQueueFSUsage, workload.go:391-427), summed in resource-index order
    (the reference sums over a map, in random order: resource-index order is the canonical choice);
  * every admission adds its entry penalty to its LocalQueue (`entry_penalty`; scheduler.go:727-742,946-960) before
    the next cycle; consumed usage does not decay inside a drain, except in event mode with `lq_last_update_ns` (below);
  * StrictFIFO keeps its head (the next cycle picks the minimum again), BestEffortFIFO advances the head's own segment,
    handleInadmissibleHash sets aside the workloads of the class in every segment of the ClusterQueue.

Event mode (the snapshot carries `wl_create_ns`, `wl_run_ns` or `adm_finish_ns`, include/kueue_b200.h): arrivals and
completions on a simulated clock, as the reference's scheduler performance runner drives them (generator.go creates
workloads at fixed intervals; controller.go:100-160 finishes each one runtimeMs after its admission, an eviction
restarting that clock).  The clock t starts at now_ns; cycle c runs at t_c (its now_ns and the QuotaReserved time of
its admissions).  Two more states: ABSENT (not created yet, in no queue) and FINISHED (never requeued).  A pending event
is the finish time of a live admitted row or the creation time of an ABSENT workload; INT64_MAX means never.
  1. no queue has a head: t jumps to E, the earliest pending event, and steps 5-7 apply the events at E without
     counting a cycle; without E the drain ends;
  2. cycle c runs at t_c, its decisions are applied as above;  3. evictions are replayed as above (with `adm_wl`);
  4. a cycle that admitted or evicted: t_{c+1} = t_c + step (drain_cycle_ns, <= 0 means 1).  A quiet cycle, the stop
     rule of the plain drain, waits instead: t_{c+1} = max(t_c + step, E); without E the drain ends;
  5. completions (workload_controller.go:936-952): every live row with finish <= t_{c+1} finishes, a row admitted in
     cycle c included (it never enters the tables).  Its cells leave its ClusterQueue's usage (cache.DeleteWorkload),
     its row is removed, its record becomes FINISHED and its root cohort tree is marked.  A row admitted at t finishes
     at t + wl_run_ns[w] (saturating at INT64_MAX); an evicted workload loses its finish time and a readmission restarts
     the full run time;
  6. arrivals (AddOrUpdateWorkload -> PushOrUpdate, manager.go:524-560): every ABSENT workload with create <= t_{c+1}
     joins its queue; the cursor moves back to it if it comes earlier.  In a BestEffortFIFO ClusterQueue a workload
     whose known scheduling hash is in the ClusterQueue's NoFit set goes straight to SET_ASIDE (cluster_queue.go:288-293;
     `NoFitSets`);
  7. the inadmissible requeue (`requeue_inadmissible`) over every root tree marked in step 3 or 5; it clears the NoFit
     sets of the ClusterQueues it visits;
  8. the heads of cycle c+1.
Steps 5-7 only set state bytes and lower cursors: their order does not change the result.  Waiting in a quiet cycle is
the canonical choice; with every run time < 0 and every creation <= now_ns the drain is the plain drain.  The drain
stops before cycle max_cycles.  Events applied before cycle 0 count only in the totals; the events applied between the
start of cycle c and the start of cycle c+1 are cycle c's (`finished`, `arrived`, `evict_done`).

Eviction latency (event mode, the snapshot carries `wl_evict_ns` and `adm_wl`, include/kueue_b200.h).  In the
reference IssuePreemptions only sets the Evicted condition (preemption.go:175-215); the quota is released once the job
is stopped and its pods are gone (reconciler.go:576-590, UnsetQuotaReservationWithCondition), then the workload leaves
the cache and its root tree is requeued (workload_controller.go:973-1004).  `wl_evict_ns[w]` is that time.  Step 3
becomes the issue, the release moves to step 5:
  3. issue at t_c: every target row of every Preempting entry that is not already evicting gets adm_evicted = 1 and the
     end time t_c + wl_evict_ns[adm_wl[row]] (saturating), which replaces its finish time (an evicted workload never
     finishes, the runner's controller.go:119-127).  It counts in `evicted`, `wl_evictions` and the active-cycle rule;
     the row keeps its cells in the usage and stays in the tables (a candidate ordered first, ordering.go:41-47), its
     record stays HELD.  A target that is already evicting gets nothing ("Preemption ongoing", preemption.go:183-186):
     a cycle whose Preempting entries only re-target evicting rows is quiet and waits for E;
  5. complete: every evicting row with end <= t_{c+1} leaves the tables (its cells leave the usage), its record is
     QUEUED with LastAssignment nil and HasQuotaReservation false, the cursor moves back, its root tree is marked, and
     it counts in `evict_done`.  E includes these end times.
Rows with adm_evicted set before the drain complete at `adm_evict_end_ns` (never targeted as new evictions) when the
snapshot carries it; without it they are issued like any other row when targeted.  With every wl_evict_ns <=
max(drain_cycle_ns, 1) and no `adm_evict_end_ns` the drain equals the drain without latency: every issued eviction
completes at the next boundary, and steps 5-7 do not depend on their order.

Decay of the AdmissionFairSharing consumed usage (event mode, the snapshot carries `lq_last_update_ns` and `adm_lq`,
include/kueue_b200.h), as the LocalQueue reconciler decays it (localqueue_controller.go:210-229,363-398):
  1. state per LocalQueue of an AFS ClusterQueue: `consumed[r]` as int64Amount (value, scale), 0 = an absent key; `last`,
     the entry's LastUpdate; `adm[r]`, the admitted usage in library units (the cells with fr % R == r of the
     LocalQueue's live rows);
  2. Decay(consumed, adm, elapsed) = MulByFloat(consumed, 1 - a) (+) MulByFloat(adm, a) with a = 1 - 0.5^(elapsed /
     half-life) (CalculateDecayedConsumed, admission_fair_sharing.go:39-66): MulByFloat(q, f) = int64(float64(
     MilliValue(q)) * f) milli-units (resource.go:72-99), `milli_value` rounds a finer scale away from zero
     (negativeScaleInt64), the MilliValue of adm[r] is adm[r] * afs_milli_mul[r], and every resource is written back as
     (milli, -3).  Durations go through Duration.Seconds() (`seconds`) before the division; 0.5^x is `half_pow`;
  3. samples: the next one is due at last + sampling.  At the start every sample due at or before now_ns is taken; at
     every boundary t -> t' (a cycle boundary or a jump) every sample due in (t, t'], in time order, with a =
     afs_alpha (one interval elapsed: the caller's calculateAlphaRate(sampling, half-life)); with half-life 0 a sample
     resets consumed to empty.  Each sample sets last to its due time.  A boundary's samples run before its
     completions.  Once a sample leaves consumed unchanged, so would every later one of the boundary (adm is constant
     there): last goes to the last due time;
  4. an admission at t_c of a workload of LocalQueue l (workload_controller.go:965-971,1030-1056): its cells join
     adm[l], consumed = Decay(consumed, adm, t_c - last) (+) entry penalty, last = t_c.  The pending penalties
     (`lq_penalty`) are not touched: the ones of the snapshot stay pending for the whole drain;
  5. a completion takes its row's cells out of adm[adm_lq[row]] at the boundary, after the samples; consumed changes at
     the next sample;
  6. the LocalQueue usage of the queue order is recomputed whenever consumed changes.
Canonical choices: samples do not wake the clock (a quiet cycle still waits for the next arrival or completion); the
early resample while penalties are pending (HasPendingFor, localqueue_controller.go:219) is not modelled; 0.5^x is
`half_pow`, the library's afs_half_pow (kb_drain.cuh) restated operation for operation, not Go's platform-dependent
math.Pow.  A drain that runs no cycle takes no sample.

The sticky workload (the snapshot carries `cq_sticky`, include/kueue_b200.h).  In the reference a BestEffortFIFO
ClusterQueue keeps a preemptor that waits for its evictions at its head (stickyWorkload, cluster_queue.go:64-93; kueue#6929,
kueue#7101): RequeueIfNotPresent (:609-619) sets `sw` to a workload requeued with RequeueReasonPendingPreemption (the
entry issued preemptions, scheduler.go:344-358; targets already evicting count, preemption.go:183-194), queueOrderingFunc
(:656-665) orders it first after the AFS LocalQueue usage and before priority, and only `delete` (:330-340) clears it,
which for a drain is the admission (Pending -> QuotaReserved calls queues.DeleteWorkload, workload_controller.go:965-966).
One slot per ClusterQueue, -1 = none, seeded from the table:
  1. heads (step 8): a ClusterQueue whose sticky workload is QUEUED takes it as its head; otherwise the head is the first
     QUEUED workload as above.  A SET_ASIDE sticky workload has no effect and is first again once it is requeued (`sw`
     survives the inadmissible set: fair_sharing_test.go:866);
  2. after the decisions (step 1): an ASSUMED head that is its ClusterQueue's sticky workload clears the slot; a
     Preempting head of a BestEffortFIFO ClusterQueue becomes the sticky workload (one value per ClusterQueue: a new one
     replaces the old); every other decision leaves the slot alone, a sticky head that goes NoFit and is set aside too;
  3. arrivals, completions, releases and the inadmissible requeue only change state bytes: steps 5-7 stay
     order-independent.
The head may lie past the cursor, so queue movement uses the head's own position: set-aside and first_aside use it, the
cursor moves only by the advance loop, and the scheduling-hash bulk move excludes the head by identity (the popped head
is not in the heap; the workload at the cursor is an ordinary queued one).  With every slot -1 at the start the drain
equals the drain without the table when (a) there is no `adm_wl` and no event table (nothing before a Preempting head
ever becomes queued again), (b) every ClusterQueue is StrictFIFO, or (c) no ClusterQueue has a preemption policy.
Preemption expectations are not modelled: the drain observes an eviction at once.

Admission checks (event mode, the snapshot carries `wl_check_ns` and `adm_wl`, include/kueue_b200.h).  In the reference
a workload of a ClusterQueue with admission checks reserves quota and becomes Admitted once every check is Ready
(SetQuotaReservation workload.go:830-853, SyncAdmittedCondition admissionchecks.go:36-70); the performance runner starts
its run clock at Admitted (controller.go:62-72,131).  Two more states: BACKOFF (evicted by a check, waiting for RequeueAt)
and DEACTIVATED (never queued again).  Every record has a mutable queue-order timestamp `qts`: `wl_check_evict_ns` when
set (for a record adm_wl does not name), otherwise `wl_ts`, the creation timestamp.  Additions to the loop:
  1. an admission at t_c of a workload with wl_check_ns > 0 reserves quota and starts attempt k = RetryCount + 1; its
     row is checking and its verdict comes at t_c + wl_check_ns (saturating), kept in the finish column.  With 0 the
     row is Ready at t_c, exactly as without the tables (wl_check_fail is then not read);
  2. verdicts are events: E includes them, and in step 5 they are applied before the boundary's completions
     (ProvisioningRequest controller.go:536-580, attempt numbering :249-263, provisioning.go:76-89):
       - Ready (no failure left): wl_ready_ns = verdict, finish = verdict + wl_run_ns (saturating); the row may finish
         in the same boundary;
       - Retry (a failing attempt with k <= check_backoff_limit): the row's cells leave the usage, the row is removed,
         its root tree is marked (reconcileCheckBasedEviction workload_controller.go:650-678: the workload holds no pods,
         so the quota goes at once; :973-1004 requeues the tree).  The record goes to BACKOFF with RequeueAt = verdict +
         WaitTime(k), RetryCount = k (resetChecksOnEviction admissionchecks.go:88-109, UpdateAdmissionCheckRequeueState
         :250-262), qts = verdict (GetQueueOrderTimestamp workload.go:1180-1182) and LastAssignment nil;
       - Rejected (k > limit): released the same way, the record is DEACTIVATED (SetDeactivationTarget,
         workload_controller.go:386-433,656-671);
       - a failing attempt uses up one unit of wl_check_fail (INT32_MAX: every attempt fails);
  3. a BACKOFF record whose RequeueAt <= t_{c+1} arrives through step 6, NoFit rule included (workload_controller.go:
     330-350,362-375 -> AddOrUpdateWorkload / PushOrUpdate); E includes the RequeueAt times;
  4. an admission resets qts to wl_ts (SetQuotaReservation resets Evicted); the new row's adm_ts is wl_ts;
  5. a preempted row whose checks are running holds no pods: with wl_evict_ns it is released at the next boundary
     (its end time is t_c).  The attempt under way is dropped: it is not counted and uses up no failure (canonical);
  6. the cycle sees qts as the heads' wl_ts (entry order scheduler.go:808, fair_sharing_iterator.go:196; preemption
     policy preemption_policy.go:39-40), and each segment's order is by qts: when a record enters its queue with a qts
     other than the key the order was built with, the order is rebuilt before the next heads (`n_resorts`): every
     cursor at its first QUEUED workload, first_aside at the first SET_ASIDE one;
  7. with every wl_check_ns = 0, every wl_check_fail = 0 and no start-state tables the drain equals the drain without
     the tables.
WaitTime(k) is `check_wait_s`: wait.NewBackoff(base, max, 2, 0.0001).WaitTime(k) (pkg/util/wait/backoff.go:35-60)
truncated to whole seconds, exact below 10,000 s (kb_run_drain refuses a strategy whose longest reachable wait,
`check_wait_bound_s`, is not below it).  It is min(base * 2^(k-1), max or infinity), except that with base > max > 0 the
first Step returns the base uncapped (attempt 1 waits base, later ones max): the reference accepts such a strategy.  Start state:
`adm_check_end_ns` (rows whose checks run, INT64_MIN = Admitted), `wl_requeue_at_ns` (records in backoff; one at or
before now_ns is queued at the start), `wl_check_retries`.  Verdicts applied between the start of cycle c and of c+1
are cycle c's (`check_retry`, `check_rejected`); those before cycle 0 count in the totals only.

WaitForPodsReady (event mode, the snapshot carries `wl_pods_ready_ns` and `adm_wl`, include/kueue_b200.h).  A workload
whose pods are not all Ready within `pods_ready_timeout_ns` of its Admitted condition is evicted (PodsReadyTimeout,
reconcileNotReadyTimeout / admittedNotReadyWorkload workload_controller.go:805-835,1106-1130), requeued after a backoff
(UpdateRequeueState workload.go:707-722) and deactivated past backoffLimitCount (triggerDeactivation :840-855).  It uses
the BACKOFF / DEACTIVATED states, RequeueAt, `qts` and the re-sort of the admission checks.  An attempt is one admission:
  1. it starts at Admitted: the reservation at t_c without a check delay, else the Ready verdict time;
  2. it fails if the record has failures left in wl_pods_ready_fail (it uses one up; INT32_MAX = every attempt fails) or
     wl_pods_ready_ns > pods_ready_timeout_ns; otherwise it is ready (a delay equal to the timeout is ready: a canonical
     tie-break).  A ready attempt reaches PodsReady at Admitted + wl_pods_ready_ns and finishes at PodsReady + wl_run_ns
     (saturating), with no event of its own;
  3. a failing attempt has an event at T = Admitted + timeout (saturating; E includes it), applied after the boundary's
     verdicts and before its completions.  With pods_ready_backoff_limit >= 0 and Count + 1 > limit: deactivation, Count
     = 0.  Otherwise Count += 1 (saturating at INT32_MAX), RequeueAt = T + WaitTime(Count) (saturating), and under the
     Eviction timestamp qts = T (GetQueueOrderTimestamp workload.go:1174-1182; Creation leaves it);
  4. the timed-out row is evicted at T: with wl_evict_ns it is an evicting row until T + latency (it keeps its cells, a
     preemptor that targets it is ongoing), without it is released by the boundary that applies T.  At release its cells
     leave the usage, its root tree is requeued, and the record goes to DEACTIVATED or BACKOFF (rule 3 of the checks
     queues it, in the same boundary when RequeueAt <= t_{c+1}) with LastAssignment nil (jobframework/reconciler.go:
     576-590, workload_controller.go:323-375,973-1004).  Neither a completion nor a preemption eviction is counted;
  5. a row preempted while its attempt waits (before PodsReady, or before T) loses it: not counted, no failure used
     (workload_controller.go:808-811), wl_pods_ready_at keeps its previous value; the row goes as any preempted row;
  6. an admission resets qts to wl_ts; Count survives a ready attempt;
  7. start state: wl_pods_ready_count, adm_admitted_ns (a row whose pods are not ready: its attempt runs from that
     Admitted time by rules 2-3 in place of adm_finish_ns), wl_requeue_at_ns, wl_pods_ready_evict_ns (qts under Eviction);
  8. with every delay 0, every fail 0 and no start-state tables the drain equals the drain without the block.
WaitTime(k) is `pods_ready_wait_ns`: wait.NewBackoff(base, max, 2, 0.0001).WaitTime(k) without jitter, in nanoseconds
(the reference's RequeueAt carries a jitter below wait * 1e-4 at second precision).  Timeouts applied between the start of
cycle c and of c+1 are cycle c's (`pods_ready_timeout`, `pods_ready_deactivated`).  blockAdmission and recoveryTimeout
are not modelled.

MaximumExecutionTimeSeconds (event mode, the snapshot carries `wl_max_exec_s` and `adm_wl`, include/kueue_b200.h).  A
workload that has spent spec.maximumExecutionTimeSeconds (`max`, 0 = nil) in the Admitted state, summed over its
admissions in status.accumulatedPastExecutionTimeSeconds (`acc`, -1 = nil, read as 0), is deactivated with reason
MaximumExecutionTimeExceeded and never requeued (workload_types.go:71-77,658-662):
  1. every row has an Admitted time A (`exec_since`): the reservation t_c without a check delay, else the Ready verdict
     time; a row whose checks run has none (SyncAdmittedCondition admissionchecks.go:36-70).  A row of a record with a
     limit has the deadline D = A + (max - acc) * 1e9 (saturating, `exec_deadline`) and the effective deadline
     max(D, A, now_ns) (reconcileMaxExecutionTime workload_controller.go:619-646: remaining = (max - acc) s - (now - A),
     acting on remaining <= 0), so a negative max - acc or a snapshot row past its limit expires at the first boundary;
  2. the finish column holds the earlier of the row's own next event (its finish, or T of a failing PodsReady attempt)
     and the effective deadline; a row whose deadline came first is EXPIRE.  A tie goes to the own event (a finish at
     the deadline finishes, a PodsReady timeout at the deadline is a timeout).  `apply_expiries` runs in step 5 after the
     verdicts and the timeouts, before the completions;
  3. at expiry (`exec_deactivate`): reason MaximumExecutionTimeExceeded (SetDeactivationTarget; the inactive branch
     :316-321,386-420 evicts and clears RequeueState: Count 0, no RequeueAt), acc = nil.  A PodsReady attempt still
     waiting is dropped (not counted, no failure used, wl_pods_ready_at back to its previous value).  The row is evicted at
     the effective deadline: an evicting row until deadline + latency with wl_evict_ns (a preemptor that targets it is
     ongoing), else released by the boundary that applies it.  At release the record is DEACTIVATED;
  4. every release of a row with an Admitted time (a completed preemption, a PodsReady-timeout release, an expiry
     release; `exec_release`) adds d = `exec_seconds`(t - A) to acc, or sets acc = d when nil (UnsetQuotaReservation
     workload.go:684-704 turns Admitted false at the release, so termination latency counts).  t is the eviction's end,
     T or the effective deadline without latency, t_c for a preemption without latency.  Completions and rows whose
     checks run add nothing.  A release at or after the row's D of a record not deactivated yet (RequeuingLimitExceeded
     sets DeactivationTarget first, :840-851) applies rule 3 there instead of the requeue or the backoff (both reconcilers
     run while the reservation is held, :509-536): acc ends as d of that attempt, and it counts at that boundary;
  5. condition times keep nanoseconds; with every limit nil and no start state the drain equals the drain without the
     block except for `wl_exec_acc_s`.
`exec_seconds` is int32(Duration.Seconds()): float64(sec) + float64(nsec) / 1e9, truncated per attempt; from about 2^24 s
the float sum can round up to sec + 1.  A value or a sum outside int32 raises ExecOverflow (kb_run_drain:
KB_ERR_UNSUPPORTED).  Deactivations between the start of cycle c and of c+1 are cycle c's (`max_exec_deactivated`).

ClusterQueue and Cohort quota changes (event mode, the snapshot carries `qc_ns`, `qc_node`, `qc_nominal`,
`qc_borrow_limit` and `qc_lend_limit`, include/kueue_b200.h).  Edit i replaces the three quota rows of node qc_node[i]
at qc_ns[i].  In the reference a spec update reaches the cache (updateClusterQueue clusterqueue.go:130-145 ->
updateQuotasAndResourceGroups :199-209; updateCohort cohort.go:44-52) and the queue manager (UpdateClusterQueue with
specUpdated, clusterqueue_controller.go:384; AddOrUpdateCohort manager.go:251-262):
  1. every edit time is a pending event: E includes the next edit not applied yet, a quiet cycle waits for it, with no
     head the clock jumps to it; after the last edit the stop rule is as before;
  2. at a boundary t -> t' every edit with qc_ns in (t, t'] is applied in table order (`apply_quota_changes`), in step
     5 before the verdicts: its rows replace the node's in the `static` tables the cycles see (of two edits of one node
     in one boundary the later wins);
  3. an edit whose three rows equal the node's current rows changes nothing (updateQuotasAndResourceGroups returns
     false, specUpdated is false): no bump, no requeue.  It still counts in `quota_changes`;
  4. every other edit adds 1 to the generation (AllocatableResourceGeneration) of every ClusterQueue of the node's root
     tree, or of the ClusterQueue alone without a cohort (updateCohortTreeResources resource_node.go:168-198 ->
     updateClusterQueueResourceNode :160-165), so every remembered LastAssignment there is outdated
     (lastAssignmentOutdated flavorassigner.go:533); and it marks the root tree for the requeue of step 7
     (notifyRetryInadmissibleWithoutLock inadmissible_workloads.go:206-223), which clears its NoFit sets;
  5. nothing is evicted: admitted rows keep their cells, usage above the new quota stays;
  6. the LastAssignment of an entry that stays pending records the current generation (`gen`);
  7. the block composes with every block above: none of their rules reads quotas.
Every cycle's snapshot carries a static_generation that changes with the rows (`static_generation_after`; 0 stays
"none"), so an evaluator that keeps static tables resident never reuses old quotas.  Edits applied between the start
of cycle c and of c+1 are cycle c's (`quota_changes`); `cq_generation` holds the generations after the drain.

Deactivation and reactivation (the snapshot carries `ac_ns`, `ac_wl`, `ac_active` (event mode) and / or `wl_inactive`;
both need `adm_wl`, include/kueue_b200.h).  Edit i sets spec.active of record ac_wl[i] to ac_active[i] at ac_ns[i]
(kueuectl stop / resume workload).  An Update that leaves a workload inactive takes the `status == Finished || !active`
branch (workload_controller.go:937-952): queues.DeleteWorkload and cache.DeleteWorkload at once, whatever the status, so
the quota goes when spec.active turns false, not when the pods are gone.  Reason 4 (USER) is a deactivation without a
DeactivationTarget.
  1. edit times are events (E, the quiet wait, the jump).  At a boundary the edits due are applied in table order per
     record; a record's own events (arrival, finish, verdict, PodsReady timeout, expiry, eviction end, RequeueAt) at or
     before an edit's time come first.  `apply_active_first` applies the edits of records that hold no row and are
     present; a record that is ABSENT or holds a row waits at its edit for `apply_active_rest` (after the row events and
     arrivals), and the first stop of an active row-holding record sets its stop time d for `apply_row_stops`, which runs
     before each row phase and stops a row whose next own event comes after d (a tie goes to the own event);
  2. stop of an active record without a row (QUEUED, SET_ASIDE, BACKOFF): DEACTIVATED, reason USER, RequeueState
     cleared (Count 0, no RequeueAt; the inactive branch :386-420), the sticky slot cleared (delete, cluster_queue.go:
     330-340), the root tree marked (QueueAssociatedInadmissibleWorkloadsAfter, manager.go:676-697);
  3. stop at d of an active record holding a row (running, checks under way, waiting for PodsReady, evicting): the cells
     leave the usage at d, the row goes, the root tree is marked, RequeueState is cleared, a waiting PodsReady attempt is
     dropped (as at an expiry), a check attempt under way is dropped (not counted, no failure used), LastAssignment nil,
     DEACTIVATED with reason USER.  A row with an Admitted time adds exec_seconds(t - A) to acc (`exec_release`): t is the
     QuotaReserved unset, after the pods terminate (jobframework/reconciler.go:576-590): the end of an eviction under way,
     else d + wl_evict_ns (d without it).  acc is not reset (only MaximumExecutionTimeExceeded resets it, :635);
  4. stop of an inactive record (any state) or a FINISHED one: nothing; it counts in `active_changes` only;
  5. resume of a DEACTIVATED record (any reason): reason 0, LastAssignment nil (its queue entry was deleted), Count 0 (as
     the deactivation left it), and it joins its queue by step 6 (`enqueue`: the NoFit rule, its LocalQueue's segment).
     wl_check_retries does not change: resetChecksOnEviction (admissionchecks.go:88-109) keeps a Pending check's
     RetryCount, and the drain keeps it at every eviction it replays.  A resume of any other record changes nothing:
     an active one, or one holding a row while the eviction of its deactivation (MaximumExecutionTimeExceeded,
     RequeuingLimitExceeded) is under way (canonical);
  6. qts does not change: a deactivation sets Evicted(Deactivated) only on a workload that is not evicted, and
     GetQueueOrderTimestamp (workload.go:1174-1193) reads the creation time for that reason; an evicted record keeps
     its condition and timestamp.  A resumed record with a qts other than its sort key re-sorts the queues (`resort`);
  7. `wl_inactive` 1-4: the record starts DEACTIVATED with that reason, in no queue, without RequeueAt;
  8. after the inadmissible requeue every cursor moves to its first QUEUED workload (a deactivated record may sit at a
     cursor or at first_aside);
  9. with no edit and every wl_inactive 0 the drain equals the drain without the block.
Edits applied between the start of cycle c and of c+1 are cycle c's (`active_changes`, and `stopped` / `resumed` for
those that changed the state); wl_deactivated / wl_deactivation_reason describe the state at the end.

Reclaim steps (event mode, the snapshot carries `wl_rc_start`, `rc_after_ns`, `rc_ps`, `rc_remaining` and `adm_wl`,
include/kueue_b200.h).  ReclaimablePods: the Job, JobSet, TrainJob and Pod integrations write Status.ReclaimablePods as
pods succeed (job_controller.go:213-227) and the cache counts only the pods still needed.  Step i of record w lowers
podset rc_ps[i] to rc_remaining[i] pods rc_after_ns[i] after the run starts:
  1. the run start S (`rc_begin`): the reservation t_c without a check delay, else the Ready verdict; with
     WaitForPodsReady the PodsReady time of a ready attempt (a failing attempt has no run).  A snapshot row starts at
     adm_run_start_ns, or at the PodsReady time of a ready attempt under way.  A readmission replays from the first step;
  2. step i is an event at S + rc_after_ns[i] (saturating; `next_event` includes it while the row can take it).  It
     applies while the row runs (`rc_live`): not checking, not evicting, phase RUN or EXPIRE, strictly before the
     finish column (its finish or its effective MaximumExecutionTimeSeconds deadline); a step at the finish is dropped,
     a row whose preemption is issued takes none.  A stop of the record at d takes the steps at or before d first
     (`apply_row_stops`: the step is an own event).  A step whose rc_remaining is not below the podset's count changes
     nothing and is not counted;
  3. `apply_reclaims` runs in step 5 after the quota edits, the verdicts and the stops they allow, the AFS samples, and
     before the timeouts, expiries and completions: none of those changes a running row before its finish column, so
     the steps it applies are those the order of the issue names.  A record's steps at one instant are one update;
  4. a step that lowers podset p from c to r (`reclaim_row`; totalRequestsFromAdmission workload.go:600-645): the
     record's ps_count[p] = r and ps_req[p] = ps_req[p] // c * r (totalRequestsFromPodSets :567-598); the row's usage of
     p becomes U0 // n * min(r, n) per resource on its flavor, U0 and n the admission's ResourceUsage and Count (`adm_use`,
     `adm_cnt`, `adm_fl`: the drain's admission, or ps_adm_*); the difference leaves the row's cells, the ClusterQueue
     usage and, under decay, the LocalQueue's admitted usage.  Once per update (workload_controller.go:1005-1014): the
     ClusterQueue's generation + 1 (deleteWorkload clusterqueue.go:477-491), its root tree marked for step 7, the
     record's scheduling hash = rc_sched_hash of the step (0 without the table);
  5. finishes and releases leave the generation alone; the block composes with every block above.
With no step that lowers a count the drain equals the drain without the block but for `ps_remaining`.  Steps applied
between the start of cycle c and of c+1 are cycle c's (`reclaims`, indices of the steps).
"""
from __future__ import annotations

import math
from dataclasses import dataclass, field
from typing import Callable, List

import numpy as np

from . import abi
from .shard import _csr_take


@dataclass
class DrainResult:
    cycles: int = 0
    admitted: List[np.ndarray] = field(default_factory=list)   # per cycle: global pending indices admitted
    heads: List[np.ndarray] = field(default_factory=list)      # per cycle: global pending indices evaluated
    decisions: List[np.ndarray] = field(default_factory=list)  # per cycle: KB_DEC_* per entry
    cq_usage: np.ndarray | None = None                         # final ClusterQueue usage [Q][FR]
    evicted: List[np.ndarray] = field(default_factory=list)    # per cycle: pending indices evicted (replay only)
    wl_evictions: np.ndarray | None = None                     # [n_wl] times each pending record was evicted
    wl_admit_cycle: np.ndarray | None = None                   # [n_wl] cycle of its last admission if it holds quota, else -1
    state: np.ndarray | None = None                            # [n_wl] final QUEUED / SET_ASIDE / HELD
    adm: dict | None = None                                    # final admitted tables (adm_* plus adm_wl when replaying)
    # event mode
    cycle_start_ns: List[int] = field(default_factory=list)    # per cycle: t_c
    finished: List[np.ndarray] = field(default_factory=list)   # per cycle: pending indices finished (-1: a row without one)
    arrived: List[np.ndarray] = field(default_factory=list)    # per cycle: pending indices arrived
    n_finished: int = 0                                        # including the events applied before cycle 0
    n_arrived: int = 0
    wl_admit_ns: np.ndarray | None = None                      # [n_wl] time of its last admission, INT64_MIN = never
    wl_finish_ns: np.ndarray | None = None                     # [n_wl] finish time, INT64_MAX = not finished
    end_ns: int = 0                                            # the clock when the drain stopped
    # eviction latency (wl_evict_ns in the snapshot; empty / 0 otherwise)
    evict_done: List[np.ndarray] = field(default_factory=list) # per cycle: pending indices whose eviction completed
    n_evict_done: int = 0                                      # including the completions applied before cycle 0
    # decay of consumed usage (lq_last_update_ns in the snapshot; None / 0 otherwise)
    lq_consumed: np.ndarray | None = None                      # [n_lq][R] int64Amount values after the drain
    lq_consumed_scale: np.ndarray | None = None                # [n_lq][R] their scales
    lq_last_update_ns: np.ndarray | None = None                # [n_lq] LastUpdate
    n_afs_samples: int = 0                                     # samples due over the drain (fixed-point skips included)
    # sticky workload (cq_sticky in the snapshot; None / empty otherwise)
    cq_sticky: np.ndarray | None = None                        # [n_cq] the slots after the drain, -1 = none
    sticky_heads: List[np.ndarray] = field(default_factory=list)  # per cycle: heads the rule chose over the first queued
    # admission checks (wl_check_ns in the snapshot; None / empty / 0 otherwise)
    check_retry: List[np.ndarray] = field(default_factory=list)     # per cycle: pending indices that went to Retry
    check_rejected: List[np.ndarray] = field(default_factory=list)  # per cycle: pending indices that were Rejected
    n_check_ready: int = 0                                     # verdicts, those before cycle 0 included
    n_check_retry: int = 0
    n_check_rejected: int = 0
    wl_ready_ns: np.ndarray | None = None                      # [n_wl] time of the last Admitted, INT64_MIN = none
    wl_check_retries: np.ndarray | None = None                 # [n_wl] final RetryCount
    wl_deactivated: np.ndarray | None = None                   # [n_wl] 1 = deactivated (Rejected, or the blocks below)
    wl_queue_ts: np.ndarray | None = None                      # [n_wl] final queue-order timestamps
    n_resorts: int = 0
    resort_orders: List[dict] = field(default_factory=list)    # the rebuilt queue state after every re-sort
    # WaitForPodsReady (wl_pods_ready_ns in the snapshot; None / empty / 0 otherwise); wl_deactivated also marks its
    # deactivations
    pods_ready_timeout: List[np.ndarray] = field(default_factory=list)      # per cycle: records timed out and requeued
    pods_ready_timeout_at: List[np.ndarray] = field(default_factory=list)   # per cycle: [n, 2] their T and RequeueAt
    pods_ready_deactivated: List[np.ndarray] = field(default_factory=list)  # per cycle: records deactivated by a timeout
    n_pods_ready_timeout: int = 0                              # those before cycle 0 included
    n_pods_ready_deactivated: int = 0
    wl_pods_ready_at: np.ndarray | None = None                 # [n_wl] last PodsReady time, INT64_MIN = none
    wl_pods_ready_count: np.ndarray | None = None              # [n_wl] final RequeueState.Count
    # MaximumExecutionTimeSeconds (wl_max_exec_s in the snapshot; None / empty / 0 otherwise); wl_deactivated also marks
    # its deactivations
    max_exec_deactivated: List[np.ndarray] = field(default_factory=list)  # per cycle: records deactivated
    n_max_exec_deactivated: int = 0                            # those before cycle 0 included
    wl_exec_acc_s: np.ndarray | None = None                    # [n_wl] final accumulated seconds, -1 = nil
    exec_spans: List[tuple] = field(default_factory=list)      # (record, Admitted time, release time, seconds added)
    wl_deactivation_reason: np.ndarray | None = None           # [n_wl] 0 none, 1 Rejected, 2 RequeuingLimitExceeded, 3 this
    # quota changes (qc_ns in the snapshot; None / empty / 0 otherwise)
    quota_changes: List[np.ndarray] = field(default_factory=list)  # per cycle: indices of the edits applied
    n_quota_changes: int = 0                                   # those before cycle 0 included (no-op edits too)
    cq_generation: np.ndarray | None = None                    # [n_cq] the generations after the drain
    static_generations: List[int] = field(default_factory=list)  # per cycle: the static_generation its snapshot carried
    # deactivation / reactivation (ac_ns or wl_inactive in the snapshot; empty / 0 otherwise); wl_deactivated and
    # wl_deactivation_reason describe the state at the end
    active_changes: List[np.ndarray] = field(default_factory=list)  # per cycle: indices of the edits applied
    stopped: List[np.ndarray] = field(default_factory=list)    # per cycle: records a stop deactivated
    resumed: List[np.ndarray] = field(default_factory=list)    # per cycle: records a resume reactivated
    n_active_changes: int = 0                                  # edits applied, those before cycle 0 and no-op edits included
    n_stopped: int = 0
    n_resumed: int = 0
    # reclaim steps (wl_rc_start in the snapshot; None / empty / 0 otherwise); cq_generation is written with it
    reclaims: List[np.ndarray] = field(default_factory=list)  # per cycle: indices of the steps that lowered a count
    n_reclaims: int = 0                                        # those before cycle 0 included
    ps_remaining: np.ndarray | None = None                     # [n_podset] the counts after reclaim at the end

    @property
    def n_evicted(self) -> int:
        return int(sum(len(e) for e in self.evicted))

    @property
    def n_admitted(self) -> int:
        return int(sum(len(a) for a in self.admitted))

    @property
    def n_decisions(self) -> int:
        return int(sum(len(h) for h in self.heads))


# RequeueReason (pkg/cache/queue/cluster_queue.go:55-66) of an entry that was not admitted, from the cycle's decision:
# entries that were nominated and then lost the admit loop are "FailedAfterNomination" (requeueAndUpdate
# scheduler.go:825-828), a Preempting entry waits for its evictions ("PendingPreemption", scheduler.go:339-346), NoFit and
# Preempt-without-targets entries keep the generic reason.
REASON_GENERIC, REASON_FAILED_AFTER_NOMINATION, REASON_NAMESPACE_MISMATCH, REASON_PENDING_PREEMPTION = (
    "", "FailedAfterNomination", "NamespaceMismatch", "PendingPreemption")


def requeue_reason(decision: int) -> str:
    if decision in (abi.DEC_NOFIT, abi.DEC_PREEMPT_NO_TARGETS):
        return REASON_GENERIC
    if decision == abi.DEC_PREEMPTING:
        return REASON_PENDING_PREEMPTION
    return REASON_FAILED_AFTER_NOMINATION  # skipped in the admit loop


def pending_flavors(last_tried) -> bool:
    """AssignmentClusterQueueState.PendingFlavors (workload.go:163-176): some podset resource still has a flavor to
    try.  `last_tried`: LastTriedFlavorIdx as rows of per-resource indices (-1 = exhausted / absent), or None."""
    if last_tried is None:
        return False
    return bool((np.asarray(last_tried) != -1).any())


def requeue_goes_inadmissible(strict_fifo: bool, reason: str, last_tried) -> bool:
    """RequeueIfNotPresent + requeueIfNotPresent (cluster_queue.go:362-393,609-633) inside a drain: no
    QueueInadmissibleWorkloads call happens between Pop and the requeue and no backoff is pending, so the workload
    returns to the heap iff the requeue is immediate or flavors are pending; otherwise it joins the inadmissible set."""
    if strict_fifo:
        immediate = reason != REASON_NAMESPACE_MISMATCH
    else:
        immediate = reason in (REASON_FAILED_AFTER_NOMINATION, REASON_PENDING_PREEMPTION, "PreemptionFailed")
    return not (immediate or pending_flavors(last_tried))


QUEUED, SET_ASIDE, HELD, ABSENT, FINISHED, BACKOFF, DEACTIVATED = 0, 1, 2, 3, 4, 5, 6  # queue state (kb_drain.cuh KB_WS_*)
NEVER = np.iinfo(np.int64).max  # an event time that never comes
UNSET = np.iinfo(np.int64).min
ALL_FAIL = np.iinfo(np.int32).max  # wl_check_fail / wl_pods_ready_fail: every attempt fails
# phase of a row (kb_drain.cuh KB_PH_*): its finish column holds the finish, T of a PodsReady attempt, the end of an
# eviction by a timeout or an expiry, the effective MaximumExecutionTimeSeconds deadline
RUN, WAIT, TIMED_OUT, EXPIRE = 0, 2, 3, 4
REJECTED, REQUEUING_LIMIT, MAX_EXEC, USER = 1, 2, 3, 4  # deactivation reasons (kb_drain_out.wl_deactivation_reason)
_S = 1_000_000_000
_I32_MAX = 2**31 - 1
MAX_BACKOFF_S = 10_000  # below it the reference's jittered, truncated WaitTime is exact


def wait_time(base_ns: int, cap_ns: int, factor: float, iteration: int) -> int:
    """Backoff.WaitTime (pkg/util/wait/backoff.go:35-60) without jitter: wait.Backoff.Step `iteration` times (the
    duration grows by `factor` in float64 and is capped at Cap, after which Steps is 0 and Step returns Cap), stopping
    at the cap.  cap_ns 0 = MaxInt64 / ceil(factor).  A base of 0 stays 0 at every Step."""
    if int(base_ns) == 0:
        return 0
    cap = cap_ns if cap_ns else int(float(2**63 - 1) / math.ceil(factor))
    dur, capped, out = int(base_ns), False, 0
    for _ in range(iteration):
        out = dur
        if not capped:
            x = float(dur) * factor
            if x >= 2.0**63 or int(x) > cap:  # a product past int64 is past the cap too
                dur, capped = cap, True
            else:
                dur = int(x)
        if out == cap:
            break
    return out


def check_wait_s(k: int, base_s: int, max_s: int) -> int:
    """RequeueAfterSeconds of admission-check attempt k: WaitTime(k) of wait.NewBackoff(base, max, 2, 0.0001) without
    jitter, in whole seconds (kb_drain.cuh kb_check_wait_ns).  The first Step returns the base uncapped, so with
    base > max > 0 attempt 1 waits base and every later one max; otherwise it is min(base * 2^(k-1), max or infinity)."""
    return wait_time(int(base_s) * 1_000_000_000, int(max_s) * 1_000_000_000, 2.0, int(k)) // 1_000_000_000


def pods_ready_wait_ns(k: int, base_s: int, max_s: int) -> int:
    """WaitTime of PodsReady requeue k: wait.NewBackoff(base, max, 2, 0.0001).WaitTime(k) without jitter, in
    nanoseconds (kb_drain.cuh kb_pods_ready_wait_ns)"""
    return wait_time(int(base_s) * 1_000_000_000, int(max_s) * 1_000_000_000, 2.0, int(k))


class ExecOverflow(ValueError):
    """An attempt's seconds or the accumulated time leaves int32 (kb_run_drain: KB_ERR_UNSUPPORTED)."""


def exec_seconds(d_ns: int) -> int:
    """int32(time.Duration(d_ns).Seconds()) for d_ns >= 0 (SyncAdmittedCondition admissionchecks.go:73-80; kb_drain.cuh
    kb_exec_seconds): float64(sec) + float64(nsec) / 1e9, truncated.  ExecOverflow when it leaves int32."""
    sec, nsec = divmod(int(d_ns), _S)
    x = float(sec) + float(nsec) / 1e9
    if x >= 2.0**31:
        raise ExecOverflow(d_ns)
    return int(x)


def exec_deadline(admitted_ns: int, max_s: int, acc_s: int) -> int:
    """the MaximumExecutionTimeSeconds deadline A + (max - acc) s (acc -1 = nil, read as 0), saturating both ways
    (kb_drain.cuh kb_exec_deadline)"""
    return max(min(int(admitted_ns) + (int(max_s) - max(int(acc_s), 0)) * _S, NEVER), UNSET)


def check_quota_changes(snap) -> None:
    """the refusals of the quota-change tables (kb_run_drain: KB_ERR_INVALID): ValueError"""
    a = snap.arrays
    if not any(k in a for k in abi.QUOTA_CHANGE_FIELDS):
        return
    if not all(k in a for k in abi.QUOTA_CHANGE_FIELDS):
        raise ValueError("quota changes: a NULL table with n_quota_change > 0")
    N, Q, FR, R = snap.n_nodes, snap.n_cq, snap.n_fr, snap.n_resource
    ns, node = a["qc_ns"].astype(np.int64), a["qc_node"].astype(np.int64)
    nom, bl, ll = (a[k].reshape(-1, FR).astype(np.int64) for k in ("qc_nominal", "qc_borrow_limit", "qc_lend_limit"))
    if (ns <= snap.now_ns).any():
        raise ValueError("quota changes: qc_ns at or before now_ns")
    if (np.diff(ns) < 0).any():
        raise ValueError("quota changes: qc_ns decreasing")
    if ((node < 0) | (node >= N)).any():
        raise ValueError("quota changes: qc_node out of range")
    if ((nom < 0) | (nom == abi.KB_NO_LIMIT)).any():
        raise ValueError("quota changes: a negative nominal or KB_NO_LIMIT in a nominal row")
    if ((bl < 0) | (ll < 0)).any():
        raise ValueError("quota changes: a negative limit")
    covered = np.zeros((Q, FR), bool)  # the cells a ClusterQueue's resource groups cover
    for q in range(Q):
        for g in range(int(a["cq_rg_start"][q]), int(a["cq_rg_start"][q + 1])):
            for f in a["rg_flavors"][int(a["rg_flavor_start"][g]):int(a["rg_flavor_start"][g + 1])]:
                for r in range(R):
                    if int(a["rg_res_mask"][g]) >> r & 1:
                        covered[q, int(f) * R + r] = True
    rows = [a[k].reshape(N, FR) for k in ("nominal", "borrow_limit", "lend_limit")]
    for i in np.flatnonzero(node < Q):
        q = int(node[i])
        for new, old in zip((nom[i], bl[i], ll[i]), rows):
            if (new[~covered[q]] != old[q][~covered[q]]).any():
                raise ValueError("quota changes: a ClusterQueue cell its resource groups do not cover")


def check_active_changes(snap) -> None:
    """the refusals of the deactivation / reactivation tables (kb_run_drain: KB_ERR_INVALID): ValueError"""
    a = snap.arrays
    if not any(k in a for k in abi.ACTIVE_FIELDS):
        return
    if "adm_wl" not in a:
        raise ValueError("active changes: the tables need adm_wl")
    if "ac_ns" in a or "ac_wl" in a or "ac_active" in a:
        if not all(k in a for k in ("ac_ns", "ac_wl", "ac_active")):
            raise ValueError("active changes: a NULL table with n_active_change > 0")
        ns, w, act = (a[k].astype(np.int64) for k in ("ac_ns", "ac_wl", "ac_active"))
        if (ns <= snap.now_ns).any():
            raise ValueError("active changes: ac_ns at or before now_ns")
        if (np.diff(ns) < 0).any():
            raise ValueError("active changes: ac_ns decreasing")
        if ((w < 0) | (w >= snap.n_wl)).any():
            raise ValueError("active changes: ac_wl out of range")
        if ((act != 0) & (act != 1)).any():
            raise ValueError("active changes: ac_active neither 0 nor 1")
        if "wl_create_ns" in a and (ns <= a["wl_create_ns"].astype(np.int64)[w]).any():
            raise ValueError("active changes: an edit at or before its record's wl_create_ns")
    if "wl_inactive" in a:
        ina = a["wl_inactive"].astype(np.int64)
        if (ina > USER).any():
            raise ValueError("active changes: wl_inactive above 4")
        if (ina[a["adm_wl"].astype(np.int64)] != 0).any():
            raise ValueError("active changes: an inactive start record that adm_wl names")
        if "wl_create_ns" in a and ((ina != 0) & (a["wl_create_ns"].astype(np.int64) > snap.now_ns)).any():
            raise ValueError("active changes: an inactive start record created after now_ns")


class ReclaimUnsupported(ValueError):
    """Steps on a record that can be partially admitted (kb_run_drain: KB_ERR_UNSUPPORTED)."""


def check_reclaims(snap) -> None:
    """the refusals of the reclaim-step tables (kb_run_drain: KB_ERR_INVALID): ValueError; ReclaimUnsupported"""
    a = snap.arrays
    if not any(k in a for k in abi.RECLAIM_FIELDS):
        return
    if "adm_wl" not in a:
        raise ValueError("reclaim steps: the tables need adm_wl")
    if not all(k in a for k in ("wl_rc_start", "rc_after_ns", "rc_ps", "rc_remaining")):
        raise ValueError("reclaim steps: a NULL table (wl_rc_start, rc_after_ns, rc_ps, rc_remaining)")
    W, R, F = snap.n_wl, snap.n_resource, snap.n_flavor
    st = a["wl_rc_start"].astype(np.int64)
    n = len(a["rc_after_ns"])
    if (len(st) != W + 1 or st[0] != 0 or (np.diff(st) < 0).any() or st[-1] != n or len(a["rc_ps"]) != n
            or len(a["rc_remaining"]) != n or ("rc_sched_hash" in a and len(a["rc_sched_hash"]) != n)):
        raise ValueError("reclaim steps: wl_rc_start is not a CSR of the steps")
    ps_start = a["wl_ps_start"].astype(np.int64)
    after, ps, rem = (a[k].astype(np.int64) for k in ("rc_after_ns", "rc_ps", "rc_remaining"))
    rec = np.repeat(np.arange(W), np.diff(st))
    if ((ps < ps_start[rec]) | (ps >= ps_start[rec + 1])).any():
        raise ValueError("reclaim steps: rc_ps outside its record")
    if (after <= 0).any() or ((np.diff(after) < 0) & (rec[1:] == rec[:-1])).any():
        raise ValueError("reclaim steps: rc_after_ns <= 0 or decreasing within a record")
    last = {}
    for i in range(n):
        if rem[i] < 0 or rem[i] > last.get(int(ps[i]), rem[i]):
            raise ValueError("reclaim steps: rc_remaining negative or increasing within a podset")
        last[int(ps[i])] = int(rem[i])
    cnt, req = a["ps_count"].astype(np.int64), a["ps_req"].reshape(-1, R).astype(np.int64)
    for p in last:
        if cnt[p] > 0 and (req[p] % cnt[p] != 0).any():
            raise ValueError("reclaim steps: ps_req of a podset with steps not divisible by its ps_count")
    has = np.diff(st) > 0
    if snap.flags & abi.F_PARTIAL_ADMISSION:
        for w in np.flatnonzero(has):
            if (a["ps_min_count"][ps_start[w]:ps_start[w + 1]] >= 0).any():
                raise ReclaimUnsupported("reclaim steps: steps on a record that can be partially admitted")
    adm_wl = a["adm_wl"].astype(np.int64)
    if "adm_run_start_ns" in a:
        rs = a["adm_run_start_ns"].astype(np.int64)
        if ((rs != UNSET) & (rs > snap.now_ns)).any():
            raise ValueError("reclaim steps: adm_run_start_ns after now_ns")
        idle = a["adm_evicted"].astype(bool).copy()
        for k in ("adm_check_end_ns", "adm_admitted_ns"):
            if k in a:
                idle |= a[k].astype(np.int64) != UNSET
        if ((rs != UNSET) & idle).any():
            raise ValueError("reclaim steps: adm_run_start_ns on a row that is not running")
    rows = [row for row in range(snap.n_adm) if has[adm_wl[row]]]
    if not rows:
        return
    if not all(k in a for k in ("ps_adm_flavor", "ps_adm_count", "ps_adm_usage")):
        raise ValueError("reclaim steps: ps_adm_* missing for a row whose record has steps")
    fl, acnt, use = a["ps_adm_flavor"].reshape(-1, R).astype(np.int64), a["ps_adm_count"].astype(np.int64), a["ps_adm_usage"].reshape(-1, R).astype(np.int64)
    us = a["adm_use_start"]
    for row in rows:
        w = adm_wl[row]
        p0, p1 = ps_start[w], ps_start[w + 1]
        if (fl[p0:p1] < -1).any() or (fl[p0:p1] >= F).any() or (acnt[p0:p1] < 0).any() or (use[p0:p1] < 0).any():
            raise ValueError("reclaim steps: ps_adm_* out of range")
        want = {}
        for p in range(p0, p1):
            for r in range(R):
                if fl[p, r] >= 0 and acnt[p] > 0:
                    fr = int(fl[p, r]) * R + r
                    want[fr] = want.get(fr, 0) + int(use[p, r]) // int(acnt[p]) * min(int(cnt[p]), int(acnt[p]))
        have = {}
        for k in range(int(us[row]), int(us[row + 1])):
            have[int(a["adm_use_fr"][k])] = have.get(int(a["adm_use_fr"][k]), 0) + int(a["adm_use_qty"][k])
        if {f: q for f, q in want.items() if q} != {f: q for f, q in have.items() if q}:
            raise ValueError("reclaim steps: a row's ps_adm_* do not add up to its adm_use cells")


def static_generation_after(base: int, changes: int, n_edits: int) -> int:
    """kb_snapshot.static_generation of a cycle after `changes` row-changing edits of a drain whose snapshot carries
    `base`: 0 stays none, otherwise one value per state of the rows that is not 0"""
    if base == 0 or changes == 0:
        return base
    g = base + changes
    return g if g != 0 else base + n_edits + 1


def check_wait_bound_s(base_s: int, max_s: int, limit: int) -> int:
    """the longest RequeueAfterSeconds a Retry can get (attempts 1..limit, 0 when limit is 0): WaitTime is constant once
    capped, which takes fewer than 64 doublings of a base of at least 1 s"""
    return max((check_wait_s(k, base_s, max_s) for k in range(1, min(int(limit), 64) + 1)), default=0)


class NoFitSets:
    """noFitSchedulingHashes of every ClusterQueue: handleInadmissibleHash inserts the hash of a NoFit head
    (cluster_queue.go:408-425, :414), queueInadmissibleWorkloads clears the set (inadmissible_workloads.go:174), and
    PushOrUpdate sets a new workload aside when its known hash is in the set of a BestEffortFIFO ClusterQueue
    (cluster_queue.go:288-293)."""

    def __init__(self):
        self.sets = {}

    def insert(self, cq: int, hsh: int) -> None:
        self.sets.setdefault(int(cq), set()).add(int(hsh))

    def clear(self, cq: int) -> None:
        self.sets.pop(int(cq), None)

    def arrival_goes_aside(self, cq: int, strict_fifo: bool, hsh: int) -> bool:
        return not strict_fifo and hsh != 0 and int(hsh) in self.sets.get(int(cq), ())


def finish_time(admit_ns: int, run_ns: int) -> int:
    """Finish time of a row admitted at admit_ns: admit + run saturating at INT64_MAX; run < 0 never finishes."""
    return NEVER if run_ns < 0 else min(int(admit_ns) + int(run_ns), NEVER)


def root_of(parent) -> np.ndarray:
    """Root node of every node of the cohort forest (a ClusterQueue without a cohort is its own root)."""
    parent = np.asarray(parent, np.int64)
    root = np.arange(len(parent))
    for _ in range(len(parent)):
        up = parent[root]
        nxt = np.where(up >= 0, up, root)
        if np.array_equal(nxt, root):
            break
        root = nxt
    return root


def requeue_inadmissible(parent, n_cq: int, notified, aside):
    """QueueAssociatedInadmissibleWorkloads for the ClusterQueues `notified` (notifyRetryInadmissibleWithoutLock +
    requeueWorkloadsCohort + queueInadmissibleWorkloads, inadmissible_workloads.go:128-223): every root of their cohort
    trees is visited once, and every set-aside workload of every ClusterQueue of a visited tree returns to its queue
    (the ClusterQueue's noFitSchedulingHashes are cleared with them).  `aside`: {cq: [workloads]}.
    Returns ({cq: [workloads moved]}, visited roots in ascending order)."""
    root = root_of(parent)
    roots = sorted({int(root[int(q)]) for q in notified})
    moved = {}
    for q in range(n_cq):
        if int(root[q]) in roots and aside.get(q):
            moved[q] = list(aside[q])
    return moved, roots


class AfsOverflow(ValueError):
    """A quantity sum leaves int64: the reference would switch to inf.Dec (kb_run_drain: KB_ERR_UNSUPPORTED)."""


AFS_MAX_SCALE = 22
_I64 = 2**63


def _int64(v: int) -> int:
    if not -_I64 <= v < _I64:
        raise AfsOverflow(v)
    return v


def quantity_add(a, b):
    """int64Amount.Add (apimachinery amount.go:162-199) on (value, scale) pairs: a zero operand keeps the other's scale,
    otherwise the sum is aligned to the smaller scale (positiveScaleInt64 + int64Add, AfsOverflow when they fail)."""
    (av, as_), (bv, bs) = a, b
    if bv == 0:
        return av, as_
    if av == 0:
        return bv, bs
    if as_ == bs:
        return _int64(av + bv), as_
    if as_ > bs:
        return _int64(_int64(av * 10**(as_ - bs)) + bv), bs
    return _int64(av + _int64(bv * 10**(bs - as_))), as_


def pow10(n: int) -> float:
    """math.Pow10 for |n| <= 22: 10^n exactly, and 1 / 10^-n (not a product with 1e-n) for negative n."""
    return float(10**n) if n >= 0 else 1.0 / float(10**-n)


def quantity_float(v: int, s: int) -> float:
    """Quantity.AsApproximateFloat64 (quantity.go:468-483) of the int64Amount (v, s)."""
    return float(v) if s == 0 else float(v) * pow10(s)


def compare_usage(a: float, b: float) -> int:
    """cmp.Compare on float64: NaN sorts before every other value, two NaNs are equal."""
    an, bn = a != a, b != b
    if an or bn:
        return 0 if an and bn else (-1 if an else 1)
    return -1 if a < b else (1 if a > b else 0)


def lq_usage(consumed, scale, penalty_milli, res_weight, lq_weight) -> float:
    """Info.CalcLocalQueueFSUsage (workload.go:391-427) of one LocalQueue: sum_r weight_r * AsApproximateFloat64(
    consumed_r (+) penalty_r) in resource-index order, divided by the LocalQueue's fair-sharing weight (1.0 when nil).
    `consumed` / `scale`: int64Amount per resource (0 = absent); `penalty_milli`: AfsEntryPenalties in milli-units."""
    usage = 0.0
    for r in range(len(consumed)):
        v, s = quantity_add((int(consumed[r]), int(scale[r])), (int(penalty_milli[r]), -3))
        if v == 0:
            continue  # a zero quantity adds what an absent key adds: nothing
        usage += float(res_weight[r]) * quantity_float(v, s)
    with np.errstate(divide="ignore", invalid="ignore"):
        return float(np.float64(usage) / np.float64(lq_weight))


# ---- decay of consumed usage: restatements of kb_drain.cuh afs_half_pow / afs_seconds / afs_alpha_of / afs_milli / afs_decay
_LN2HI, _LN2LO, _LOG2E = 6.93147180369123816490e-01, 1.90821492927058770002e-10, 1.44269504088896338700e+00
_EXP_P = (1.66666666666666657415e-01, -2.77777777770155933842e-03, 6.61375632143793436117e-05, -1.65339022054652515390e-06,
          4.13813679705723846039e-08)


def half_pow(x: float) -> float:
    """0.5^x for x >= 0, operation for operation as kb_drain.cuh afs_half_pow: Go's Pow for base 0.5 (x = yi + yf with
    |yf| <= 0.5, exp(yf * Log(0.5)) by the fdlibm reduction and polynomial of Go's exp, then ldexp by -yi)."""
    yi = float(math.trunc(x))
    yf = x - yi
    if yf > 0.5:
        yf -= 1.0
        yi += 1.0
    if yi >= 2048.0:
        return 0.0
    v = yf * -0.6931471805599453
    if -3.725290298461914e-09 < v < 3.725290298461914e-09:
        a = 1.0 + v
    else:
        p1, p2, p3, p4, p5 = _EXP_P
        k = int(_LOG2E * v - 0.5) if v < 0 else int(_LOG2E * v + 0.5)
        hi = v - float(k) * _LN2HI
        lo = float(k) * _LN2LO
        r = hi - lo
        t = r * r
        c = r - t * (p1 + t * (p2 + t * (p3 + t * (p4 + t * p5))))
        a = math.ldexp(1.0 - ((lo - (r * c) / (2.0 - c)) - hi), k)
    return math.ldexp(a, -int(yi))


def _cdiv(a: int, b: int):
    """C's truncating a / b and a % b"""
    q, r = divmod(abs(a), b)
    return (q, r) if a >= 0 else (-q, -r)


def seconds(d_ns: int) -> float:
    """time.Duration.Seconds(): float64(d / 1e9) + float64(d % 1e9) / 1e9"""
    q, r = _cdiv(int(d_ns), 1_000_000_000)
    return float(q) + float(r) / 1e9


def alpha_of(elapsed_ns: int, half_life_ns: int) -> float:
    """calculateAlphaRate(elapsed.Seconds(), halfLife.Seconds()) with half_pow: 0 when the half-life is 0"""
    return 0.0 if half_life_ns == 0 else 1.0 - half_pow(seconds(elapsed_ns) / seconds(half_life_ns))


def milli_value(v: int, s: int) -> int:
    """Quantity.MilliValue of the int64Amount (v, s): a coarser scale multiplies (AfsOverflow when it leaves int64), a
    finer one divides and rounds away from zero (negativeScaleInt64, apimachinery math.go:166-198)."""
    if s >= -3:
        return _int64(v * 10**(s + 3))
    q, rem = _cdiv(v, 10**(-3 - s))
    return q + (1 if v > 0 else -1) if rem else q


def decay_quantities(cons, scale, adm, milli_mul, alpha: float):
    """CalculateDecayedConsumed of one LocalQueue: MulByFloat(consumed, 1 - alpha) (+) MulByFloat(admitted, alpha), every
    resource as (milli, -3).  Returns (values, changed)."""
    keep = 1.0 - alpha
    out, changed = [], False
    for r in range(len(cons)):
        old = milli_value(int(cons[r]), int(scale[r]))
        mul, q = int(milli_mul[r]), int(adm[r])
        if q > (2**63 - 1) // mul or q < -((2**63 - 1) // mul):
            raise AfsOverflow(q)
        v = _int64(int(float(old) * keep) + int(float(q * mul) * alpha))
        changed |= v != int(cons[r]) or int(scale[r]) != -3
        out.append(v)
    return out, changed


def entry_penalty(req_rows, mask_rows, milli_mul, alpha: float):
    """CalculateEntryPenalty (admission_fair_sharing.go) of one workload in milli-units per resource:
    int64(float64(MilliValue(SumTotalRequests_r)) * alpha), over the full TotalRequests (the keys of Requests only)."""
    R = len(milli_mul)
    out = []
    for r in range(R):
        total = sum(int(q) for q, m in zip(req_rows[:, r], mask_rows) if int(m) >> r & 1)
        milli = _int64(_int64(total) * int(milli_mul[r]))
        out.append(int(float(milli) * alpha))
    return out


def _queue_order(a, Q, ts=None):
    """Pending workloads in queueOrderingFunc order per segment: (order, start[S+1], seg_start[Q+1], seg_lq[S]).  A
    segment is a ClusterQueue, or one LocalQueue of a ClusterQueue with AdmissionFairSharing (numbered
    ClusterQueue-major)."""
    cq = a["wl_cq"].astype(np.int64)
    if "wl_lq" in a:
        afs = a["cq_afs"].astype(bool)
        n_lq_of = np.bincount(a["lq_cq"].astype(np.int64), minlength=Q)
        nseg = np.where(afs, n_lq_of, 1)
        seg_start = np.concatenate([[0], np.cumsum(nseg)])
        lq_first = np.concatenate([[0], np.cumsum(n_lq_of)])
        seg_lq = np.full(int(seg_start[-1]), -1, np.int64)
        for q in np.flatnonzero(afs):
            seg_lq[seg_start[q]:seg_start[q + 1]] = np.arange(lq_first[q], lq_first[q + 1])
        lq = a["wl_lq"].astype(np.int64)
        seg = np.where(afs[cq], seg_start[cq] + lq - lq_first[cq], seg_start[cq])
    else:
        seg_start, seg_lq, seg = np.arange(Q + 1), np.full(Q, -1, np.int64), cq
    S = int(seg_start[-1])
    order = np.lexsort((a["wl_uid"], a["wl_ts"] if ts is None else ts, -a["wl_priority"].astype(np.int64), seg))
    start = np.zeros(S + 1, np.int64)
    np.add.at(start, seg + 1, 1)
    return order, np.cumsum(start), seg_start, seg_lq


_ADM_ROW_KEYS = ("adm_cq", "adm_priority", "adm_ts", "adm_qr_ts", "adm_uid", "adm_evicted")
_ADM_KEYS = _ADM_ROW_KEYS + ("adm_use_start", "adm_use_fr", "adm_use_qty")
# DrainResult's per-cycle event lists (`_Drain.log`); each has its total n_<name> but pods_ready_timeout_at, the [n, 2]
# times beside pods_ready_timeout
_EVENT_LISTS = ("finished", "arrived", "evict_done", "check_retry", "check_rejected", "pods_ready_timeout",
                "pods_ready_timeout_at", "pods_ready_deactivated", "max_exec_deactivated", "quota_changes", "active_changes",
                "stopped", "resumed", "reclaims")


class _Rows:
    """The admitted tables of a drain.  `adm` holds the snapshot's columns (the cells of row i are adm_use_start[i] ..
    adm_use_start[i + 1]); every block the snapshot carries adds a column (None otherwise), exported under its key:
      wl        the pending record, -1 = a row of an event snapshot without adm_wl     adm_wl
      finish    the finish column: the next event of the row (see RUN .. EXPIRE)       adm_finish_ns
      evicting  an eviction is under way (eviction latency)                            adm_evicting
      since     the Admitted time, UNSET = none (MaximumExecutionTimeSeconds)          adm_exec_since_ns
      checking  the admission checks run                                               adm_checking
      phase     RUN / WAIT / TIMED_OUT / EXPIRE (WaitForPodsReady, max exec)           adm_pods_ready_phase
      lq        the LocalQueue (decay of consumed usage)                               -
      rc_next   the time of the row's next reclaim step, NEVER = none                  -
      rc_cur    the index of that step                                                 -
    Rows join and leave only through `append` and `remove`, which move their cells in and out of the ClusterQueue usage
    (cache.AddWorkload / DeleteWorkload) and keep every column aligned."""
    COLUMNS = {"wl": "adm_wl", "finish": "adm_finish_ns", "evicting": "adm_evicting", "since": "adm_exec_since_ns",
               "checking": "adm_checking", "phase": "adm_pods_ready_phase", "lq": None, "rc_next": None, "rc_cur": None}

    def __init__(self, a, usage):
        self.adm = {k: a[k].copy() for k in _ADM_KEYS}
        self.usage = usage
        self.wl = self.finish = self.evicting = self.since = self.checking = self.phase = self.lq = None
        self.rc_next = self.rc_cur = None

    def _columns(self):
        return [c for c in self.COLUMNS if getattr(self, c) is not None]

    def append(self, cells, **cols):
        """new rows at the end: `cells` holds one {flavor-resource: quantity} per row, `cols` the new rows' values of
        every snapshot column but the cells and of every block column"""
        adm, usage = self.adm, self.usage
        start, fr, qty = [int(adm["adm_use_start"][-1])], [], []
        for cqi, row_cells in zip(cols["adm_cq"], cells):
            for f, q in row_cells.items():
                usage[int(cqi), f] += q
                fr.append(f); qty.append(q)
            start.append(start[-1] + len(row_cells))
        cols.update(adm_use_start=np.asarray(start[1:], np.int32), adm_use_fr=np.asarray(fr, np.int32),
                    adm_use_qty=np.asarray(qty, np.int64))
        for k in _ADM_KEYS:
            adm[k] = np.concatenate([adm[k], cols[k]])
        for c in self._columns():
            setattr(self, c, np.concatenate([getattr(self, c), cols[c]]))

    def remove(self, rows):
        """rows leave the tables; the other rows keep their order"""
        adm, usage = self.adm, self.usage
        us, uf, uq = adm["adm_use_start"], adm["adm_use_fr"], adm["adm_use_qty"]
        for row in rows:
            cqi = int(adm["adm_cq"][row])
            for k in range(int(us[row]), int(us[row + 1])):
                usage[cqi, int(uf[k])] -= int(uq[k])
        keep = np.ones(len(adm["adm_cq"]), bool)
        keep[rows] = False
        cnt = np.diff(us.astype(np.int64))
        cell_keep = np.repeat(keep, cnt)
        for k in _ADM_ROW_KEYS:
            adm[k] = adm[k][keep]
        adm["adm_use_fr"], adm["adm_use_qty"] = uf[cell_keep], uq[cell_keep]
        adm["adm_use_start"] = np.concatenate([[0], np.cumsum(cnt[keep])]).astype(np.int32)
        for c in self._columns():
            setattr(self, c, getattr(self, c)[keep])

    def export(self, hide=()):
        """DrainResult.adm: the snapshot's columns, then every block column but those in `hide` under its key"""
        out = dict(self.adm)
        for c, key in self.COLUMNS.items():
            if key is not None and c not in hide and getattr(self, c) is not None:
                out[key] = getattr(self, c)
        return out


def drain(snap: abi.FlatSnapshot, run_cycle: Callable[[abi.FlatSnapshot], abi.CycleOut], max_cycles: int = 10_000) -> DrainResult:
    return _Drain(snap).run(run_cycle, max_cycles)


class _Drain:
    """The state of one drain: the queues, the records, the admitted tables (`rows`) and the blocks the snapshot
    carries.  The methods named in the module docstring are its rules; `run` iterates the cycles and the boundaries."""

    def __init__(self, snap: abi.FlatSnapshot):
        self.snap = snap
        a = self.a = snap.arrays
        Q, R, FR = self.Q, self.R, self.FR = snap.n_cq, snap.n_resource, snap.n_fr
        W = snap.n_wl
        checks = self.checks = "wl_check_ns" in a
        pr = self.pr = "wl_pods_ready_ns" in a                         # WaitForPodsReady
        backoff = self.backoff = checks or pr                          # BACKOFF / DEACTIVATED, RequeueAt, mutable qts
        mx = self.mx = "wl_max_exec_s" in a                            # MaximumExecutionTimeSeconds
        if mx and "adm_wl" not in a:
            raise ValueError("wl_max_exec_s needs adm_wl")
        qts = self.qts = a["wl_ts"].astype(np.int64).copy()            # queue-order timestamps (checks, PodsReady: mutable)
        if backoff:
            if "adm_wl" not in a:
                raise ValueError("wl_check_ns / wl_pods_ready_ns need adm_wl")
            held0 = np.zeros(W, bool)
            held0[a["adm_wl"].astype(np.int64)] = True
            if "wl_check_evict_ns" in a:
                ce = a["wl_check_evict_ns"].astype(np.int64)
                qts[:] = np.where((ce != UNSET) & ~held0, ce, qts)
            if pr and "wl_pods_ready_evict_ns" in a and not snap.pods_ready_requeue_creation:  # rule 7 (Eviction timestamp)
                pe = a["wl_pods_ready_evict_ns"].astype(np.int64)
                qts[:] = np.where(pe != UNSET, pe, qts)
        self.order, self.qstart, seg_start, self.seg_lq = _queue_order(a, Q, qts)
        self.seg_start = seg_start
        self.sort_ts = qts.copy()                                      # the keys the order was built with
        qlen = self.qlen = np.diff(self.qstart)
        afs_cq = self.afs_cq = a["cq_afs"].astype(bool) if "wl_lq" in a else np.zeros(Q, bool)
        replay = self.replay = "adm_wl" in a
        check_quota_changes(snap)
        quota = self.quota = "qc_ns" in a and len(a["qc_ns"]) > 0     # ClusterQueue / Cohort quota changes
        check_active_changes(snap)
        act = self.act = "ac_ns" in a and len(a["ac_ns"]) > 0         # deactivation / reactivation edits
        self.blk = act or "wl_inactive" in a                           # the block (its start state alone needs no events)
        check_reclaims(snap)
        rc = self.rc = "wl_rc_start" in a                              # reclaim steps
        events = self.events = any(k in a for k in abi.EVENT_FIELDS) or quota or act or rc
        self.step = max(1, int(snap.drain_cycle_ns)) if events else 1
        create = self.create = a.get("wl_create_ns")
        self.run_ns = a.get("wl_run_ns")
        lat = self.lat = a.get("wl_evict_ns")  # eviction latency: issue at t_c, release at the end time
        if lat is not None and not replay:
            raise ValueError("wl_evict_ns needs adm_wl")
        state = self.state = np.full(W, QUEUED, np.uint8)
        self.seg_of = np.zeros(W, np.int64)                            # segment of every pending workload
        self.pos_of = np.zeros(W, np.int64)                            # its position in the segment's static order
        self.index_segments()
        self.usage = a["cq_usage"].reshape(Q, FR).astype(np.int64).copy()
        rows = self.rows = _Rows(a, self.usage)
        self.res = DrainResult()
        if replay:
            rows.wl = a["adm_wl"].astype(np.int64).copy()
        if events:  # the record of every row (-1: a row of the snapshot without adm_wl) and its finish time
            if not replay:
                rows.wl = np.full(snap.n_adm, -1, np.int64)
            rows.finish = a["adm_finish_ns"].astype(np.int64).copy() if "adm_finish_ns" in a else np.full(snap.n_adm, NEVER, np.int64)
            if create is not None:
                state[create > snap.now_ns] = ABSENT
            if lat is not None:
                rows.evicting = np.zeros(snap.n_adm, bool)
                if "adm_evict_end_ns" in a:  # evictions under way before the drain complete at their end time
                    rows.evicting = a["adm_evicted"].astype(bool).copy()
                    rows.finish[rows.evicting] = a["adm_evict_end_ns"][rows.evicting]
        if replay:
            state[a["adm_wl"].astype(np.int64)] = HELD  # holds quota: out of every queue
        self.requeue_at = np.full(W, UNSET, np.int64)                  # RequeueAt of a BACKOFF record
        if backoff and "wl_requeue_at_ns" in a:  # records in backoff at the start
            ra = a["wl_requeue_at_ns"].astype(np.int64)
            state[ra > snap.now_ns] = BACKOFF
            self.requeue_at[ra > snap.now_ns] = ra[ra > snap.now_ns]
        deactivated = self.deactivated = np.zeros(W, np.uint8)        # 0, or the reason (REJECTED, REQUEUING_LIMIT, MAX_EXEC, USER)
        if "wl_inactive" in a:  # rule 7 of deactivation: inactive records start DEACTIVATED, in no queue, without RequeueAt
            ina = a["wl_inactive"].astype(np.uint8)
            deactivated[ina != 0] = ina[ina != 0]
            state[ina != 0] = DEACTIVATED
            self.requeue_at[ina != 0] = UNSET
        if checks:  # rule 1: attempt state; start state of the rows whose checks run
            self.chk_ns = a["wl_check_ns"].astype(np.int64)
            self.chk_fail = a["wl_check_fail"].astype(np.int64).copy() if "wl_check_fail" in a else np.zeros(W, np.int64)
            self.retries = a["wl_check_retries"].astype(np.int64).copy() if "wl_check_retries" in a else np.zeros(W, np.int64)
            rows.checking = np.zeros(snap.n_adm, bool)
            if "adm_check_end_ns" in a:
                ce = a["adm_check_end_ns"].astype(np.int64)
                rows.checking = ce != UNSET
                rows.finish[rows.checking] = ce[rows.checking]
            self.ready_ns = np.full(W, UNSET, np.int64)
        if pr or mx:
            rows.phase = np.full(snap.n_adm, RUN, np.int64)
        if pr:  # rules 2 and 7: attempt state, and the rows whose pods are not ready at the start
            self.pr_ns = a["wl_pods_ready_ns"].astype(np.int64)
            self.pr_fail = a["wl_pods_ready_fail"].astype(np.int64).copy() if "wl_pods_ready_fail" in a else np.zeros(W, np.int64)
            self.pr_count = a["wl_pods_ready_count"].astype(np.int64).copy() if "wl_pods_ready_count" in a else np.zeros(W, np.int64)
            self.pr_at = np.full(W, UNSET, np.int64)                   # last PodsReady time
            self.pr_prev = self.pr_at.copy()                           # its value before the attempt under way
            if "adm_admitted_ns" in a:
                for row in np.flatnonzero(a["adm_admitted_ns"] != UNSET):
                    rows.finish[row], rows.phase[row] = self.pr_attempt(int(rows.wl[row]), int(a["adm_admitted_ns"][row]))
        if mx:  # rule 1: limits, accumulated times, the Admitted time of every row; the start rows' effective deadlines
            self.exec_max = a["wl_max_exec_s"].astype(np.int64)
            self.acc = a["wl_exec_acc_s"].astype(np.int64).copy() if "wl_exec_acc_s" in a else np.full(W, -1, np.int64)
            if snap.n_adm and "adm_exec_since_ns" not in a:
                raise ValueError("wl_max_exec_s needs adm_exec_since_ns when the snapshot has admitted rows")
            rows.since = a["adm_exec_since_ns"].astype(np.int64).copy() if snap.n_adm else np.zeros(0, np.int64)
            for row in range(snap.n_adm):
                if rows.since[row] == UNSET or (rows.evicting is not None and rows.evicting[row]):
                    continue
                rows.finish[row], e = self.exec_clip(int(rows.wl[row]), int(rows.since[row]), int(rows.finish[row]), int(snap.now_ns))
                if e:
                    rows.phase[row] = EXPIRE
        self.ps_start = a["wl_ps_start"].astype(np.int64)
        self.ps_req = a["ps_req"].reshape(-1, R)
        self.ps_cnt = a["ps_count"]                                    # the counts after reclaim (reclaim steps: mutable)
        self.shash = a.get("wl_sched_hash")
        if rc:  # rule 1 of reclaim steps: the steps, the admissions' assignments, the running rows of the snapshot
            self.ps_req, self.ps_cnt = self.ps_req.astype(np.int64).copy(), self.ps_cnt.astype(np.int64).copy()
            self.shash = self.shash.astype(np.int64).copy() if self.shash is not None else None
            self.rc_start, self.rc_after, self.rc_ps, self.rc_rem = (a[k].astype(np.int64) for k in (
                "wl_rc_start", "rc_after_ns", "rc_ps", "rc_remaining"))
            self.rc_hash = a["rc_sched_hash"].astype(np.int64) if "rc_sched_hash" in a else None
            P = len(self.ps_cnt)
            self.adm_fl, self.adm_cnt, self.adm_use = np.full((P, R), -1, np.int64), np.zeros(P, np.int64), np.zeros((P, R), np.int64)
            rows.rc_next, rows.rc_cur = np.full(snap.n_adm, NEVER, np.int64), np.zeros(snap.n_adm, np.int64)
            rs = a["adm_run_start_ns"].astype(np.int64) if "adm_run_start_ns" in a else np.full(snap.n_adm, UNSET, np.int64)
            for row in range(snap.n_adm):
                w = int(rows.wl[row])
                if self.rc_start[w] == self.rc_start[w + 1]:
                    continue
                p = slice(int(self.ps_start[w]), int(self.ps_start[w + 1]))
                self.adm_fl[p] = a["ps_adm_flavor"].reshape(-1, R)[p]
                self.adm_cnt[p] = a["ps_adm_count"][p]
                self.adm_use[p] = a["ps_adm_usage"].reshape(-1, R)[p]
                S = int(rs[row])
                if S == UNSET and pr and "adm_admitted_ns" in a and a["adm_admitted_ns"][row] != UNSET:
                    S = int(self.pr_at[w])  # a ready attempt under way: its PodsReady time (UNSET for a failing one)
                if S != UNSET:
                    self.rc_begin(row, w, S)
        self.sticky = a["cq_sticky"].astype(np.int64).copy() if "cq_sticky" in a else None  # sticky workload per ClusterQueue
        self.cursor = np.zeros(len(qlen), np.int64)
        self.first_aside = qlen.copy()                                 # smallest SET_ASIDE position per segment (qlen = none)
        self.nofit = NoFitSets()
        for s in range(len(qlen)):
            self.advance(s)
        decay = self.decay = events and "wl_lq" in a and "lq_last_update_ns" in a
        if afs_cq.any() or decay:
            L = len(a["lq_cq"])
            self.penalty = (a["lq_penalty"].reshape(L, R).astype(object) if "lq_penalty" in a else np.zeros((L, R), object))
            self.consumed, self.cscale = a["lq_consumed"].reshape(L, R), a["lq_consumed_scale"].reshape(L, R)
            if decay:  # rule 1: mutable consumed usage, LastUpdate and the admitted usage of the snapshot's rows
                self.consumed, self.cscale = self.consumed.astype(object), self.cscale.astype(np.int64)
                self.lq_last = a["lq_last_update_ns"].astype(np.int64).copy()
                self.lq_afs = afs_cq[a["lq_cq"].astype(np.int64)]
                rows.lq = a["adm_lq"].astype(np.int64).copy() if "adm_lq" in a else np.zeros(0, np.int64)
                self.ladm = np.zeros((L, R), object)
                us = a["adm_use_start"]
                for row in np.flatnonzero(rows.lq >= 0):
                    for k in range(int(us[row]), int(us[row + 1])):
                        self.ladm[rows.lq[row], int(a["adm_use_fr"][k]) % R] += int(a["adm_use_qty"][k])
                self.hl, self.samp = int(snap.afs_half_life_ns), int(snap.afs_sampling_ns)
                self.n_samples = 0
            self.lqu = {int(l): self.usage_of(l) for l in self.seg_lq if l >= 0}
        self.first_seg = seg_start[:-1]
        self.strict = a["cq_strategy"].astype(bool)  # KB_QUEUE_STRICT_FIFO = 1
        self.last_gen = a["wl_last_gen"].astype(np.int64).copy()       # LastAssignment.ClusterQueueGeneration, -1 = nil
        self.last_tried = a["ps_last_tried"].reshape(-1, R).copy()     # LastAssignment.LastTriedFlavorIdx
        self.has_qr = a["wl_has_quota_reservation"].copy() if "wl_has_quota_reservation" in a else None
        self.admit_cycle = np.full(W, -1, np.int64)
        self.evictions = np.zeros(W, np.int64)
        self.admit_ns = np.full(W, np.iinfo(np.int64).min, np.int64)
        self.finish_ns = np.full(W, NEVER, np.int64)
        self.root = root_of(a["parent"])
        self.static = {k: v for k, v in a.items() if not (k.startswith(("wl_", "ps_", "adm_")) or k in ("heads", "cq_usage") +
                                                          abi.AFS_FIELDS + abi.AFS_DECAY_FIELDS + abi.STICKY_FIELDS +
                                                          abi.QUOTA_CHANGE_FIELDS + abi.ACTIVE_FIELDS + abi.RECLAIM_FIELDS)}
        self.gen = a["cq_generation"].astype(np.int64).copy()          # AllocatableResourceGeneration (rule 4 of quota changes)
        self.static_gen, self.qc_next, self.qc_rowed = int(snap.static_generation), 0, 0
        # edits that can change the static tables: quota changes, and reclaim updates (the generations)
        self.n_gen_edits = (len(a["qc_ns"]) if quota else 0) + (len(a["rc_after_ns"]) if rc else 0)
        if quota:
            self.qc_ns, self.qc_node = a["qc_ns"].astype(np.int64), a["qc_node"].astype(np.int64)
            self.qc_rows = [a[k].reshape(-1, FR) for k in ("qc_nominal", "qc_borrow_limit", "qc_lend_limit")]
            self.static.update({k: a[k].reshape(snap.n_nodes, FR).astype(np.int64).copy()
                                for k in ("nominal", "borrow_limit", "lend_limit")})
        if act:  # deactivation / reactivation edits
            self.ac_ns, self.ac_wl, self.ac_on = (a[k].astype(np.int64) for k in ("ac_ns", "ac_wl", "ac_active"))
        # per boundary: the stop times of row-holding records, the edits left for after the row events and arrivals, the
        # time a deferred record's row went
        self.ac_next, self.stop_at, self.deferred, self.row_gone = 0, {}, {}, {}
        self.covers_pods = np.zeros(Q, bool)
        if snap.pods_resource >= 0:
            for q in range(Q):
                masks = a["rg_res_mask"][a["cq_rg_start"][q]:a["cq_rg_start"][q + 1]]
                self.covers_pods[q] = bool(np.any(masks & (1 << snap.pods_resource)))
        if events and create is not None:  # ABSENT workloads in (create, index) order; `arr_next` is the first not arrived
            arr_order = np.lexsort((np.arange(W), create))
            self.arr_order = arr_order[create[arr_order] > snap.now_ns]
        else:
            self.arr_order = np.zeros(0, np.int64)
        self.arr_next = 0
        self.t = int(snap.now_ns)

    # ---- queues
    def index_segments(self):
        """seg_of / pos_of of every pending workload from the order"""
        order, qstart = self.order, self.qstart
        for s in range(len(self.qlen)):
            self.seg_of[order[qstart[s]:qstart[s + 1]]] = s
            self.pos_of[order[qstart[s]:qstart[s + 1]]] = np.arange(self.qlen[s])

    def advance(self, s):
        """the cursor of segment s to its first QUEUED workload"""
        cursor, qlen, state, order, q0 = self.cursor, self.qlen, self.state, self.order, self.qstart[s]
        while cursor[s] < qlen[s] and state[order[q0 + cursor[s]]] != QUEUED:
            cursor[s] += 1

    def set_aside(self, w):
        self.state[w] = SET_ASIDE
        s = self.seg_of[w]
        self.first_aside[s] = min(self.first_aside[s], self.pos_of[w])

    def queue(self, w):
        """w is QUEUED: the cursor of its segment moves back to it if it comes earlier"""
        self.state[w] = QUEUED
        s = self.seg_of[w]
        self.cursor[s] = min(self.cursor[s], self.pos_of[w])

    def enqueue(self, w):
        """step 6 for one record: PushOrUpdate, with the NoFit rule of a BestEffortFIFO ClusterQueue"""
        q = int(self.a["wl_cq"][w])
        if self.shash is not None and self.nofit.arrival_goes_aside(q, bool(self.strict[q]), int(self.shash[w])):
            self.set_aside(w)
        else:
            self.queue(w)

    def usage_of(self, l):
        return lq_usage(self.consumed[l], self.cscale[l], self.penalty[l], self.a["afs_res_weight"], self.a["lq_weight"][l])

    def afs_head_seg(self, q):
        """segment of the head of AFS ClusterQueue q, -1 = nothing queued"""
        a, cursor, qlen, order, qstart, lqu, seg_lq = self.a, self.cursor, self.qlen, self.order, self.qstart, self.lqu, self.seg_lq
        best, bkey = -1, None
        for s in range(int(self.seg_start[q]), int(self.seg_start[q + 1])):
            if cursor[s] >= qlen[s]:
                continue
            w = order[qstart[s] + cursor[s]]
            key = (int(a["wl_priority"][w]), int(a["wl_ts"][w]), int(a["wl_uid"][w]))
            if best >= 0:
                c = compare_usage(lqu[int(seg_lq[s])], lqu[int(seg_lq[best])])
                if c > 0 or (c == 0 and (-key[0], key[1], key[2]) >= (-bkey[0], bkey[1], bkey[2])):
                    continue
            best, bkey = s, key
        return best

    def resort(self):
        """rule 6: rebuild the order when a queued or set-aside record carries a key other than the one it was sorted by"""
        state, qts, cursor, first_aside, qlen, res = self.state, self.qts, self.cursor, self.first_aside, self.qlen, self.res
        if not self.backoff or not (((state == QUEUED) | (state == SET_ASIDE)) & (qts != self.sort_ts)).any():
            return
        self.order, self.qstart, _, _ = _queue_order(self.a, self.Q, qts)
        self.sort_ts = qts.copy()
        self.index_segments()
        for s in range(len(qlen)):
            cursor[s] = 0
            self.advance(s)
            seg = self.order[self.qstart[s]:self.qstart[s + 1]]
            aside = np.flatnonzero(state[seg] == SET_ASIDE)
            first_aside[s] = int(aside[0]) if len(aside) else qlen[s]
        res.n_resorts += 1
        res.resort_orders.append(dict(order=self.order.copy(), qstart=self.qstart.copy(), qts=qts.copy(), state=state.copy(),
                                      cursor=cursor.copy(), first_aside=first_aside.copy(), seg_of=self.seg_of.copy(),
                                      pos_of=self.pos_of.copy()))

    def requeue(self, notified):
        """step 7: the inadmissible requeue in the root cohort trees of `notified`"""
        order, qstart, state, cursor, first_aside = self.order, self.qstart, self.state, self.cursor, self.first_aside
        seg_start = self.seg_start
        aside = {}
        for q in range(self.Q):
            for s in range(int(seg_start[q]), int(seg_start[q + 1])):
                seg = order[qstart[s] + first_aside[s]:qstart[s + 1]]
                aside.setdefault(q, []).extend(int(w) for w in seg[state[seg] == SET_ASIDE])
        moved, roots = requeue_inadmissible(self.a["parent"], self.Q, sorted(notified), aside)
        for ws in moved.values():
            state[np.asarray(ws, np.int64)] = QUEUED
        for q in np.flatnonzero(np.isin(self.root[:self.Q], roots)):
            self.nofit.clear(q)
            for s in range(int(seg_start[q]), int(seg_start[q + 1])):
                cursor[s] = min(cursor[s], first_aside[s])
                first_aside[s] = self.qlen[s]

    # ---- records and rows
    def log(self, name, vals):
        """files events of the boundary under way in DrainResult: into the list of the last cycle (the events between
        the start of cycle c and of c+1 are cycle c's) and into the total, or into the total only before cycle 0"""
        res = self.res
        if name != "pods_ready_timeout_at":
            setattr(res, "n_" + name, getattr(res, "n_" + name) + len(vals))
        if res.cycles and len(vals):
            lst = getattr(res, name)
            lst[-1] = np.concatenate([lst[-1], np.asarray(vals, np.int64)])

    def forget(self, w):
        """a released record: LastAssignment nil, no reservation"""
        self.last_gen[w] = -1
        self.last_tried[int(self.ps_start[w]):int(self.ps_start[w + 1])] = -1
        if self.has_qr is not None:
            self.has_qr[w] = 0
        self.admit_cycle[w] = -1

    def release(self, w):
        """the record of an evicted row returns to its queue with LastAssignment nil (workload_controller.go:973-1004);
        preemption sets no RequeueState, so the requeue is immediate"""
        self.forget(w)
        self.queue(w)

    def clear_requeue(self, w):
        """RequeueState cleared: Count 0, no RequeueAt"""
        if self.pr:
            self.pr_count[w] = 0
        self.requeue_at[w] = UNSET

    def drop_attempt(self, w, t):
        """a PodsReady attempt still waiting at t is dropped: not counted, no failure used"""
        if self.pr and self.pr_at[w] > t:
            self.pr_at[w] = self.pr_prev[w]

    def evict_row(self, row, w, t0):
        """an eviction issued at t0 on a row (eviction latency): evicting until t0 + latency"""
        rows = self.rows
        rows.evicting[row] = True
        rows.adm["adm_evicted"][row] = 1
        rows.finish[row] = min(t0 + int(self.lat[w]), NEVER)

    def lq_release(self, row):
        """rule 5 of decay: a row's cells leave its LocalQueue's admitted usage"""
        rows = self.rows
        if self.decay and rows.lq[row] >= 0 and self.afs_cq[int(rows.adm["adm_cq"][row])]:
            us = rows.adm["adm_use_start"]
            for k in range(int(us[row]), int(us[row + 1])):
                self.ladm[rows.lq[row], int(rows.adm["adm_use_fr"][k]) % self.R] -= int(rows.adm["adm_use_qty"][k])

    def pr_attempt(self, w, t0):
        """rules 1-2 of WaitForPodsReady: the attempt of record w Admitted at t0 -> (finish column, phase)"""
        d = int(self.pr_ns[w])
        timeout = int(self.snap.pods_ready_timeout_ns)
        if self.pr_fail[w] > 0 or d > timeout:
            return min(t0 + timeout, NEVER), WAIT
        self.pr_prev[w] = self.pr_at[w]
        self.pr_at[w] = min(t0 + d, NEVER)
        return (finish_time(int(self.pr_at[w]), int(self.run_ns[w])) if self.run_ns is not None else NEVER), RUN

    def exec_clip(self, w, A, fin, floor=UNSET):
        """rule 2 of MaximumExecutionTimeSeconds: (finish column, expires first) of a row of record w Admitted at A
        whose own next event is fin"""
        if self.exec_max[w] <= 0:
            return fin, False
        dl = max(exec_deadline(A, int(self.exec_max[w]), int(self.acc[w])), A, floor)
        return (dl, True) if dl < fin else (fin, False)

    def admitted(self, row, w, t):
        """row of record w is Admitted at t: the run clock or the PodsReady attempt starts, and the
        MaximumExecutionTimeSeconds deadline with it (rule 1 of each; the reservation without a check delay, or a Ready
        verdict)"""
        rows = self.rows
        if self.checks:
            self.ready_ns[w] = t
        if self.pr:
            rows.finish[row], rows.phase[row] = self.pr_attempt(w, t)
        else:
            rows.finish[row] = finish_time(t, int(self.run_ns[w])) if self.run_ns is not None else NEVER
        if self.rc:  # rule 1 of reclaim steps: the run starts at Admitted, or at PodsReady of a ready attempt
            if not self.pr or rows.phase[row] == RUN:
                self.rc_begin(row, w, int(self.pr_at[w]) if self.pr else t)
            else:
                rows.rc_next[row] = NEVER
        if self.mx:
            rows.since[row] = t
            rows.finish[row], e = self.exec_clip(w, t, int(rows.finish[row]))
            if e:
                rows.phase[row] = EXPIRE

    def exec_deactivate(self, w):
        """rule 3 of MaximumExecutionTimeSeconds: deactivated, acc nil, RequeueState cleared"""
        self.deactivated[w] = MAX_EXEC
        self.acc[w] = -1
        self.clear_requeue(w)
        self.log("max_exec_deactivated", [w])

    def exec_release(self, row, w, t_rel):
        """rule 4: the release at t_rel of a row with an Admitted time adds its seconds to acc, after deactivating a
        record whose deadline has passed; returns whether it deactivated the record"""
        A = int(self.rows.since[row])
        if A == UNSET:
            return False
        acc, lim = self.acc, self.exec_max
        deact = lim[w] > 0 and self.deactivated[w] == 0 and exec_deadline(A, int(lim[w]), int(acc[w])) <= t_rel
        if deact:
            self.exec_deactivate(w)
        d = exec_seconds(t_rel - A)
        total = d if acc[w] < 0 else int(acc[w]) + d
        if total > _I32_MAX:
            raise ExecOverflow(total)
        acc[w] = total
        self.res.exec_spans.append((int(w), A, int(t_rel), d))
        return deact

    # ---- reclaim steps
    def rc_begin(self, row, w, S):
        """rule 1: the run of row (record w) starts at S; its steps replay from the first"""
        i = int(self.rc_start[w])
        self.rows.rc_cur[row] = i
        self.rows.rc_next[row] = min(S + int(self.rc_after[i]), NEVER) if i < self.rc_start[w + 1] else NEVER

    def rc_live(self):
        """rule 2: the rows that can take a step (their run started, not checking, not evicting, RUN or EXPIRE)"""
        rows = self.rows
        live = rows.rc_next < NEVER
        if rows.checking is not None:
            live &= ~rows.checking
        if rows.evicting is not None:
            live &= ~rows.evicting
        if rows.phase is not None:
            live &= (rows.phase == RUN) | (rows.phase == EXPIRE)
        return live

    def reclaim_row(self, row, lim, notified):
        """rules 2 and 4: the steps of a running row due at or before lim, in time order; a record's steps at one instant
        are one update"""
        rows, R, a = self.rows, self.R, self.a
        t, i, w = int(rows.rc_next[row]), int(rows.rc_cur[row]), int(rows.wl[row])
        if t > lim:
            return
        i1, S = int(self.rc_start[w + 1]), t - int(self.rc_after[i])
        cq = int(rows.adm["adm_cq"][row])
        us = rows.adm["adm_use_start"]
        while i < i1 and t <= lim:
            lowered = False
            while i < i1 and min(S + int(self.rc_after[i]), NEVER) == t:
                p, rem = int(self.rc_ps[i]), int(self.rc_rem[i])
                c = int(self.ps_cnt[p])
                if rem < c:
                    self.ps_req[p] = self.ps_req[p] // c * rem
                    n = int(self.adm_cnt[p])
                    for r in range(R):
                        f = int(self.adm_fl[p, r])
                        if f < 0 or n <= 0:
                            continue
                        u = int(self.adm_use[p, r]) // n
                        d = u * min(rem, n) - u * min(c, n)
                        if d == 0:
                            continue
                        fr = f * R + r
                        for k in range(int(us[row]), int(us[row + 1])):
                            if int(rows.adm["adm_use_fr"][k]) == fr:
                                rows.adm["adm_use_qty"][k] += d
                                break
                        self.usage[cq, fr] += d
                        if self.decay and rows.lq[row] >= 0 and self.afs_cq[cq]:
                            self.ladm[rows.lq[row], r] += d
                    self.ps_cnt[p] = rem
                    if self.shash is not None:
                        self.shash[w] = int(self.rc_hash[i]) if self.rc_hash is not None else 0
                    lowered = True
                    self.log("reclaims", [i])
                i += 1
            if lowered:  # AllocatableResourceGeneration + 1, the root tree requeued
                self.gen[cq] += 1
                self.static["cq_generation"] = self.gen.copy()
                notified.add(cq)
                self.qc_rowed += 1
                self.static_gen = static_generation_after(int(self.snap.static_generation), self.qc_rowed, self.n_gen_edits)
            t = min(S + int(self.rc_after[i]), NEVER) if i < i1 else NEVER
        rows.rc_cur[row], rows.rc_next[row] = i, t

    def apply_reclaims(self, t_next, notified):
        """rule 3: the steps due by t_next of every running row, strictly before its finish column"""
        rows = self.rows
        for row in np.flatnonzero(self.rc_live() & (rows.rc_next <= t_next)):
            self.reclaim_row(row, min(int(t_next), int(rows.finish[row]) - 1), notified)

    # ---- the boundary: steps 5-8
    def next_event(self):
        """earliest pending event after the evictions: a live row's finish or an ABSENT workload's creation (None = none)"""
        fin = self.rows.finish
        e = int(fin.min()) if len(fin) else NEVER
        if self.quota and self.qc_next < len(self.qc_ns):
            e = min(e, int(self.qc_ns[self.qc_next]))
        if self.act and self.ac_next < len(self.ac_ns):
            e = min(e, int(self.ac_ns[self.ac_next]))
        if self.arr_next < len(self.arr_order):
            e = min(e, int(self.create[self.arr_order[self.arr_next]]))
        if self.backoff and (self.state == BACKOFF).any():
            e = min(e, int(self.requeue_at[self.state == BACKOFF].min()))
        if self.rc and len(fin):
            e = min(e, int(np.where(self.rc_live(), self.rows.rc_next, NEVER).min()))
        return None if e >= NEVER else e

    def sample(self, t_to):
        """rule 3 of decay: every sample due at or before t_to (nothing is due at or before the previous boundary)"""
        consumed, cscale, lq_last, samp, R = self.consumed, self.cscale, self.lq_last, self.samp, self.R
        for l in np.flatnonzero(self.lq_afs & (lq_last <= t_to - samp)):
            k = (int(t_to) - int(lq_last[l])) // samp
            self.n_samples += k
            moved = False
            for _ in range(k):
                if self.hl == 0:
                    vals, sc = [0] * R, 0
                    changed = any(int(v) != 0 for v in consumed[l]) or bool((cscale[l] != 0).any())
                else:
                    (vals, changed), sc = decay_quantities(consumed[l], cscale[l], self.ladm[l], self.a["afs_milli_mul"],
                                                           self.snap.afs_alpha), -3
                consumed[l, :] = vals
                cscale[l, :] = sc
                if not changed:
                    break
                moved = True
            lq_last[l] += k * samp
            if moved:
                self.lqu[int(l)] = self.usage_of(l)

    def apply_quota_changes(self, t_next, notified):
        """rules 2-4 of quota changes: the edits due by t_next, in table order, before the verdicts"""
        static, keys = self.static, ("nominal", "borrow_limit", "lend_limit")
        while self.qc_next < len(self.qc_ns) and int(self.qc_ns[self.qc_next]) <= t_next:
            i, n = self.qc_next, int(self.qc_node[self.qc_next])
            self.qc_next += 1
            self.log("quota_changes", [i])
            if all(np.array_equal(static[k][n], new[i]) for k, new in zip(keys, self.qc_rows)):
                continue  # no-op: specUpdated is false
            for k, new in zip(keys, self.qc_rows):
                static[k] = static[k].copy()
                static[k][n] = new[i]
            self.gen[self.root[:self.Q] == self.root[n]] += 1
            static["cq_generation"] = self.gen.copy()
            notified.add(n)  # its root tree is requeued (requeue_inadmissible maps a node to its root)
            self.qc_rowed += 1
            self.static_gen = static_generation_after(int(self.snap.static_generation), self.qc_rowed, self.n_gen_edits)

    def apply_active_edit(self, j, w, held, notified):
        """rules 2, 4 and 5 of deactivation on record w; held: it holds a row at the edit's time (nothing changes)"""
        state, deactivated = self.state, self.deactivated
        if held:
            return
        if self.ac_on[j] == 0:
            if deactivated[w] == 0 and state[w] in (QUEUED, SET_ASIDE, BACKOFF):  # rule 2
                state[w] = DEACTIVATED
                deactivated[w] = USER
                self.clear_requeue(w)
                q = int(self.a["wl_cq"][w])
                if self.sticky is not None and self.sticky[q] == w:
                    self.sticky[q] = -1
                notified.add(q)
                self.forget(w)
                self.log("stopped", [w])
        elif state[w] == DEACTIVATED:  # rule 5: LastAssignment nil, Count 0 since the deactivation
            deactivated[w] = 0
            self.forget(w)
            self.enqueue(w)
            self.log("resumed", [w])

    def apply_active_first(self, t_next, notified):
        """rule 1: the edits due by t_next, in table order per record, before the row events.  A record that is ABSENT
        or holds a row meets its own events first: its edits from there wait for apply_active_rest; the first stop of an
        active row-holding record sets its stop time (apply_row_stops)"""
        state, deactivated, ac_ns = self.state, self.deactivated, self.ac_ns
        hi = self.ac_next
        while hi < len(ac_ns) and int(ac_ns[hi]) <= t_next:
            hi += 1
        by_w = {}
        for j in range(self.ac_next, hi):
            by_w.setdefault(int(self.ac_wl[j]), []).append(j)
        self.log("active_changes", range(self.ac_next, hi))
        self.ac_next = hi
        for w, js in by_w.items():
            for k, j in enumerate(js):
                if state[w] == ABSENT or (state[w] == HELD and (deactivated[w] != 0 or self.ac_on[j] == 0)):
                    if state[w] == HELD and deactivated[w] == 0:
                        self.stop_at[w] = int(ac_ns[j])
                    self.deferred[w] = js[k:]
                    break
                self.apply_active_edit(j, w, state[w] == HELD, notified)

    def apply_row_stops(self, notified):
        """rule 3: every row of an active record whose stop time comes before the row's next own event"""
        rows, stop_at, deactivated = self.rows, self.stop_at, self.deactivated
        if not stop_at:
            return
        gone = [row for row in range(len(rows.wl)) if int(rows.wl[row]) in stop_at and deactivated[rows.wl[row]] == 0
                and stop_at[int(rows.wl[row])] < rows.finish[row]]
        if self.rc:  # a step at or before the stop goes first
            live = self.rc_live()
            for row in gone:
                if live[row]:
                    self.reclaim_row(row, stop_at[int(rows.wl[row])], notified)
        for row in gone:
            w = int(rows.wl[row]); d = stop_at[w]
            deactivated[w] = USER
            self.clear_requeue(w)
            self.drop_attempt(w, d)
            if self.mx:  # QuotaReserved unset once the pods are gone
                rel = rows.evicting is not None and rows.evicting[row]
                t_rel = int(rows.finish[row]) if rel else min(d + int(self.lat[w]), NEVER) if self.lat is not None else d
                self.exec_release(row, w, t_rel)
            notified.add(int(rows.adm["adm_cq"][row]))
            self.lq_release(row)
            self.state[w] = DEACTIVATED
            self.forget(w)
            self.row_gone[w] = d
            self.log("stopped", [w])
        if gone:
            rows.remove(gone)

    def apply_active_rest(self, notified):
        """rule 1: the deferred edits after the row events and arrivals; a record whose row went at a time after an
        edit held it then"""
        for w, js in self.deferred.items():
            for j in js:
                self.apply_active_edit(j, w, self.state[w] == HELD or self.row_gone.get(w, UNSET) > int(self.ac_ns[j]), notified)
        self.deferred.clear(); self.stop_at.clear(); self.row_gone.clear()

    def apply_verdicts(self, t_next, notified):
        """rule 2 of the checks: the verdicts due by t_next, before the completions"""
        rows, chk_fail, state = self.rows, self.chk_fail, self.state
        gone = []
        for row in np.flatnonzero(rows.checking & (rows.finish <= t_next)):
            w, tv = int(rows.wl[row]), int(rows.finish[row])
            rows.checking[row] = False
            if chk_fail[w] == 0:  # Ready: Admitted, the run clock (or the PodsReady attempt) starts
                self.admitted(row, w, tv)
                self.res.n_check_ready += 1
                continue
            if chk_fail[w] != ALL_FAIL:
                chk_fail[w] -= 1
            k = int(self.retries[w]) + 1
            gone.append(row)
            notified.add(int(rows.adm["adm_cq"][row]))
            self.forget(w)
            if k <= self.snap.check_backoff_limit:  # Retry: backoff, then requeued with the eviction time as its queue-order timestamp
                self.retries[w] = k
                state[w] = BACKOFF
                wait_s = check_wait_s(k, self.snap.check_backoff_base_s, self.snap.check_backoff_max_s)
                self.requeue_at[w] = min(tv + wait_s * 1_000_000_000, NEVER)
                self.qts[w] = tv
                self.log("check_retry", [w])
            else:  # Rejected: deactivated
                state[w] = DEACTIVATED
                self.deactivated[w] = REJECTED
                self.log("check_rejected", [w])
        if gone:
            rows.remove(gone)

    def apply_timeouts(self, t_next):
        """rules 3-4 of WaitForPodsReady: the timeouts due by t_next, after the verdicts and before the completions"""
        rows, snap, pr_count = self.rows, self.snap, self.pr_count
        limit = int(snap.pods_ready_backoff_limit)
        for row in np.flatnonzero((rows.phase == WAIT) & (rows.finish <= t_next)):
            w, T = int(rows.wl[row]), int(rows.finish[row])
            if 0 < self.pr_fail[w] != ALL_FAIL:
                self.pr_fail[w] -= 1
            if limit >= 0 and pr_count[w] + 1 > limit:  # RequeuingLimitExceeded: deactivated, RequeueState cleared
                pr_count[w] = 0
                self.deactivated[w] = REQUEUING_LIMIT
                self.log("pods_ready_deactivated", [w])
            else:
                pr_count[w] = min(int(pr_count[w]) + 1, ALL_FAIL)
                self.requeue_at[w] = min(T + pods_ready_wait_ns(int(pr_count[w]), snap.pods_ready_backoff_base_s,
                                                                snap.pods_ready_backoff_max_s), NEVER)
                if not snap.pods_ready_requeue_creation:
                    self.qts[w] = T
                self.log("pods_ready_timeout", [w])
                self.log("pods_ready_timeout_at", [(T, int(self.requeue_at[w]))])
            rows.phase[row] = TIMED_OUT
            if self.lat is not None:  # the pods terminate: an evicting row until T + latency
                self.evict_row(row, w, T)

    def apply_expiries(self, t_next):
        """rules 2-3 of MaximumExecutionTimeSeconds: the expiries due by t_next, after the timeouts, before the completions"""
        rows = self.rows
        for row in np.flatnonzero((rows.phase == EXPIRE) & (rows.finish <= t_next)):
            w, dl = int(rows.wl[row]), int(rows.finish[row])
            self.exec_deactivate(w)
            self.drop_attempt(w, dl)
            rows.phase[row] = TIMED_OUT
            if self.lat is not None:  # evicted at the deadline: an evicting row until deadline + latency
                self.evict_row(row, w, dl)

    def apply_events(self, t_next, notified):
        """steps 5 and 6 at t_next: the row events, the completions and the arrivals"""
        rows, state = self.rows, self.state
        if self.quota:
            self.apply_quota_changes(t_next, notified)
        if self.act:
            self.apply_active_first(t_next, notified)
            self.apply_row_stops(notified)
        if self.checks:
            self.apply_verdicts(t_next, notified)
            if self.act:
                self.apply_row_stops(notified)
        if self.rc:
            self.apply_reclaims(t_next, notified)
        if self.pr:
            self.apply_timeouts(t_next)
            if self.act:
                self.apply_row_stops(notified)
        if self.mx:
            self.apply_expiries(t_next)
        done = np.flatnonzero(rows.finish <= t_next)
        gone = rows.evicting[done] if rows.evicting is not None else np.zeros(len(done), bool)
        to = rows.phase[done] == TIMED_OUT if rows.phase is not None else np.zeros(len(done), bool)
        self.log("finished", rows.wl[done[~gone & ~to]].copy())
        self.log("evict_done", rows.wl[done[gone & ~to]].copy())
        for row in done:
            notified.add(int(rows.adm["adm_cq"][row]))
            self.lq_release(row)
            w = int(rows.wl[row])
            if self.act:
                self.row_gone[w] = int(rows.finish[row])
            timed_out = rows.phase is not None and rows.phase[row] == TIMED_OUT
            rel = rows.evicting is not None and rows.evicting[row]
            expired = self.mx and (timed_out or rel) and self.exec_release(row, w, int(rows.finish[row]))  # rule 4 (max exec)
            if timed_out or expired:  # rule 4 (PodsReady): the record waits for RequeueAt, or is deactivated
                state[w] = DEACTIVATED if self.deactivated[w] else BACKOFF
                self.forget(w)
            elif rel:
                self.release(w)
            elif w >= 0:
                state[w] = FINISHED
                self.admit_cycle[w] = -1
                self.finish_ns[w] = int(rows.finish[row])
        if len(done):
            rows.remove(done)
        arr = []
        while self.arr_next < len(self.arr_order) and int(self.create[self.arr_order[self.arr_next]]) <= t_next:
            w = int(self.arr_order[self.arr_next]); self.arr_next += 1
            self.enqueue(w)
            arr.append(w)
        self.log("arrived", arr)
        if self.act:  # before the requeue after a backoff: a BACKOFF record's stop and its requeue give the same state
            self.apply_active_rest(notified)
        if self.backoff:  # rule 3 of the checks: the records whose RequeueAt has come
            for w in np.flatnonzero((state == BACKOFF) & (self.requeue_at <= t_next)):
                self.requeue_at[w] = UNSET
                self.enqueue(int(w))

    def boundary(self, t_next, notified):
        """the clock moves to t_next: samples, steps 5-7, and the cursors and the order of step 8; `notified`: the
        ClusterQueues whose root trees the cycle's evictions marked"""
        if self.decay:
            self.sample(t_next)
        self.t = t_next
        self.apply_events(t_next, notified)
        if notified:
            self.requeue(notified)
        if self.act:  # a deactivated record may sit at a cursor or at first_aside: every cursor to its first QUEUED
            for s in range(len(self.qlen)):
                self.advance(s)
        self.resort()

    # ---- the loop
    def run(self, run_cycle, max_cycles):
        res, qlen, cursor, first_seg = self.res, self.qlen, self.cursor, self.first_seg
        if self.decay and len(qlen) and self.snap.n_wl and max_cycles > 0:
            self.sample(self.t)
        while len(qlen) and res.cycles < max_cycles:
            hseg = np.where(cursor[np.minimum(first_seg, len(qlen) - 1)] < qlen[np.minimum(first_seg, len(qlen) - 1)], first_seg, -1)
            for q in np.flatnonzero(self.afs_cq):
                hseg[q] = self.afs_head_seg(q)
            live = np.flatnonzero(hseg >= 0)
            if len(live) == 0:
                if not self.events:
                    break
                e = self.next_event()  # step 1: the clock jumps to the next event
                if e is None:
                    break
                self.boundary(e, set())
                continue
            if not self.cycle(run_cycle, live, hseg[live]):
                break
        return self.result()

    def cycle(self, run_cycle, live, segs):
        """steps 2-4 at t for the ClusterQueues `live` with heads in segments `segs`, then the boundary; False when the
        drain ends"""
        a, snap, res, rows, R, t = self.a, self.snap, self.res, self.rows, self.R, self.t
        state, sticky, strict, seg_start, ps_start = self.state, self.sticky, self.strict, self.seg_start, self.ps_start
        c = res.cycles
        heads = self.order[self.qstart[segs] + self.cursor[segs]]  # global pending indices, one per ClusterQueue with work left
        chosen = []
        if sticky is not None:  # a queued sticky workload is its ClusterQueue's head
            for e, q in enumerate(live):
                w = int(sticky[q])
                if w >= 0 and state[w] == QUEUED and w != heads[e]:
                    heads[e] = w
                    chosen.append(w)
        cs = abi.FlatSnapshot(n_cq=self.Q, n_cohort=snap.n_cohort, n_flavor=snap.n_flavor, n_resource=R,
                              pods_resource=snap.pods_resource, flags=snap.flags, now_ns=t, static_generation=self.static_gen)
        cs.arrays.update(self.static)
        cs.set("cq_usage", self.usage)
        for k, v in rows.adm.items():
            cs.set(k, v)
        for nm in ("wl_cq", "wl_priority", "wl_uid"):
            cs.set(nm, a[nm][heads])
        cs.set("wl_ts", self.qts[heads])  # the queue-order timestamp (rule 6)
        cs.set("wl_last_gen", self.last_gen[heads])
        if self.has_qr is not None:
            cs.set("wl_has_quota_reservation", self.has_qr[heads])
        st, psr = _csr_take(ps_start, heads)
        cs.set("wl_ps_start", st)
        cs.set("ps_req", self.ps_req[psr]); cs.set("ps_last_tried", self.last_tried[psr])
        cs.set("ps_count", self.ps_cnt[psr])  # the counts after reclaim
        for nm in ("ps_req_mask", "ps_min_count", "ps_flavor_ok"):
            cs.set(nm, a[nm][psr])
        if "ps_group" in a:  # optional tables (kb_snapshot: NULL when absent)
            cs.set("ps_group", a["ps_group"][psr])
        cs.set("heads", np.arange(len(heads)))
        cs.finalize()
        out = run_cycle(cs)
        dec = np.asarray(out.decision).copy()
        res.cycles += 1
        res.heads.append(heads); res.decisions.append(dec)
        res.sticky_heads.append(np.asarray(chosen, np.int64))
        res.cycle_start_ns.append(t)
        for k in _EVENT_LISTS:
            getattr(res, k).append(np.zeros((0, 2) if k == "pods_ready_timeout_at" else 0, np.int64))
        res.static_generations.append(self.static_gen)
        ok = dec == abi.DEC_ASSUMED
        res.admitted.append(heads[ok])
        # ---- apply the admissions: Assignment.Usage (flavorassigner.go:198-218) with the admitted counts
        new_cells = []
        for e in np.flatnonzero(ok):
            cqi = int(cs.arrays["wl_cq"][e])
            cells = {}
            for row in range(int(st[e]), int(st[e + 1])):
                full, cnt = int(cs.arrays["ps_count"][row]), int(out.ps_count[row])
                if self.rc:  # the admission's PodSetAssignment (rule 4 of reclaim steps)
                    g_row = int(ps_start[heads[e]]) + row - int(st[e])
                    self.adm_fl[g_row], self.adm_cnt[g_row], self.adm_use[g_row] = -1, cnt, 0
                for r in range(R):
                    f = int(out.ps_flavor[row, r])
                    if f < 0:
                        continue
                    if self.covers_pods[cqi] and r == snap.pods_resource:
                        q = cnt
                    else:
                        q = int(cs.arrays["ps_req"].reshape(-1, R)[row, r])
                        if full != 0 and full != cnt:
                            q = q // full * cnt  # ScaledTo workload.go:258-275
                    cells[f * R + r] = cells.get(f * R + r, 0) + q
                    if self.rc:
                        self.adm_fl[g_row, r], self.adm_use[g_row, r] = f, q
            new_cells.append(cells)
            if self.afs_cq[cqi]:  # AfsEntryPenalties.Push of the entry penalty, then the LocalQueue's usage again
                w, lq = int(heads[e]), int(a["wl_lq"][heads[e]])
                wrows = slice(int(ps_start[w]), int(ps_start[w + 1]))
                pen = entry_penalty(self.ps_req[wrows], a["ps_req_mask"][wrows], a["afs_milli_mul"], snap.afs_alpha)
                if self.decay:  # rule 4: admitted usage, decay to t, LastUpdate = t, the penalty into consumed
                    consumed, cscale, ladm = self.consumed, self.cscale, self.ladm
                    for fr, q in cells.items():
                        ladm[lq, fr % R] += q
                    alpha = alpha_of(t - int(self.lq_last[lq]), self.hl)
                    vals, _ = decay_quantities(consumed[lq], cscale[lq], ladm[lq], a["afs_milli_mul"], alpha)
                    consumed[lq, :] = vals
                    cscale[lq, :] = -3
                    self.lq_last[lq] = t
                    for r, d in enumerate(pen):
                        consumed[lq, r], cscale[lq, r] = quantity_add((int(consumed[lq, r]), int(cscale[lq, r])), (d, -3))
                else:
                    for r, d in enumerate(pen):
                        self.penalty[lq, r] = _int64(int(self.penalty[lq, r]) + d)
                self.lqu[lq] = self.usage_of(lq)
        g = heads[ok]
        n_new = len(g)
        if n_new:
            self.admit(g, new_cells, c)
        # ---- LastAssignment of the entries that stay pending (scheduler.go:345,494)
        tried = np.asarray(out.ps_tried_idx).reshape(-1, R)
        cqs = live
        last_gen, last_tried = self.last_gen, self.last_tried
        for e in range(len(heads)):
            if ok[e]:
                continue
            w = int(heads[e])
            r0, r1 = int(st[e]), int(st[e + 1])
            if dec[e] == abi.DEC_PREEMPTING:
                last_gen[w] = -1
                last = None
            else:
                last_gen[w] = int(self.gen[int(a["wl_cq"][w])])  # the current generation (rule 6 of quota changes)
                last_tried[int(ps_start[w]):int(ps_start[w + 1])] = tried[r0:r1]
                last = tried[r0:r1]
            # ---- queue movement (cluster_queue.go:362-425,609-633); a StrictFIFO queue keeps its head either way
            if requeue_goes_inadmissible(False, requeue_reason(int(dec[e])), last) and not strict[cqs[e]]:
                self.set_aside(w)
        if sticky is not None:  # admission deletes the sticky workload, a BestEffortFIFO preemptor becomes it
            for e in range(len(heads)):
                q, w = int(cqs[e]), int(heads[e])
                if ok[e] and sticky[q] == w:
                    sticky[q] = -1
                elif dec[e] == abi.DEC_PREEMPTING and not strict[q]:
                    sticky[q] = w
        if self.shash is not None:
            order, qstart, cursor, shash = self.order, self.qstart, self.cursor, self.shash
            for e in np.flatnonzero((dec == abi.DEC_NOFIT) & ~strict[cqs]):
                hsh = int(shash[heads[e]])
                if hsh == 0:
                    continue
                q = int(cqs[e])
                self.nofit.insert(q, hsh)
                for s in range(int(seg_start[q]), int(seg_start[q + 1])):  # every queued workload of the class but the head
                    rest = order[qstart[s] + cursor[s]:qstart[s + 1]]
                    for w in rest[(shash[rest] == hsh) & (state[rest] == QUEUED) & (rest != heads[e])]:
                        self.set_aside(int(w))
        advance = self.advance
        for q in cqs:  # the next head is the first queued workload
            for s in range(int(seg_start[q]), int(seg_start[q + 1])):
                advance(s)
        # ---- evictions (replay): every target of every Preempting entry, as rows of the tables the cycle saw
        victims = []
        if self.replay:
            for e in np.flatnonzero(dec == abi.DEC_PREEMPTING):
                victims.extend(int(out.tgt_adm[k]) for k in range(int(out.tgt_start[e]), int(out.tgt_start[e + 1])))
            victims = sorted(set(victims))
        if rows.evicting is not None:  # latency: issue the evictions not under way yet; the rows stay until their end time
            victims = [row for row in victims if not rows.evicting[row]]
        res.evicted.append(np.sort(rows.wl[victims]) if victims else np.zeros(0, np.int64))
        notified = set()
        for row in victims:
            w = int(rows.wl[row])
            if rows.evicting is not None:
                self.evict_row(row, w, t)
                if rows.checking is not None and rows.checking[row]:  # rule 5 of the checks: no pods, released at the next boundary
                    rows.checking[row] = False
                    rows.finish[row] = t
                if rows.phase is not None:  # an ordinary evicting row (rule 5 of PodsReady: a waiting attempt is dropped)
                    rows.phase[row] = RUN
            else:
                if self.mx and self.exec_release(row, w, t):  # rule 4 of max exec: past its deadline, deactivated
                    state[w] = DEACTIVATED
                    self.forget(w)
                else:
                    self.release(w)
                notified.add(int(rows.adm["adm_cq"][row]))
            self.drop_attempt(w, t)  # rule 5 of PodsReady: dropped before PodsReady
            self.evictions[w] += 1
        if victims and rows.evicting is None:
            rows.remove(victims)
        if not self.events:
            if notified:  # ---- inadmissible requeue in the root cohort trees of the victims
                self.requeue(notified)
            if n_new == 0 and not victims:
                return False
            self.t += 1
            return True
        # ---- the next time, then the completions and arrivals up to it
        if n_new or victims:
            t_next = min(t + self.step, NEVER)
        else:
            e = self.next_event()
            if e is None:
                return False  # quiet, and nothing will ever happen again
            t_next = max(min(t + self.step, NEVER), e)
        self.boundary(t_next, notified)
        return True

    def admit(self, g, cells, c):
        """the workloads g admitted in cycle c at t join the tables with their cells: HELD, a reservation with a check
        delay starts an attempt (rule 1 of the checks), every other one is Admitted at once"""
        a, t, rows = self.a, self.t, self.rows
        self.admit_cycle[g] = c
        self.admit_ns[g] = t
        self.state[g] = HELD
        if self.backoff:  # rule 4 of the checks, 6 of PodsReady: the reservation resets Evicted
            self.qts[g] = a["wl_ts"][g]
        n = len(g)
        chk = self.chk_ns[g] > 0 if self.checks else np.zeros(n, bool)
        fin = [min(t + int(self.chk_ns[w]), NEVER) if k else NEVER for w, k in zip(g, chk)]  # a verdict comes at t + delay
        first = len(rows.adm["adm_cq"])
        rows.append(cells, adm_cq=a["wl_cq"][g], adm_priority=a["wl_priority"][g], adm_ts=a["wl_ts"][g],
                    adm_qr_ts=np.full(n, t, np.int64), adm_uid=a["wl_uid"][g], adm_evicted=np.zeros(n, np.uint8), wl=g,
                    finish=np.asarray(fin, np.int64), evicting=np.zeros(n, bool), since=np.full(n, UNSET, np.int64),
                    checking=chk, phase=np.full(n, RUN, np.int64),
                    lq=a["wl_lq"][g].astype(np.int64) if self.decay else None,
                    rc_next=np.full(n, NEVER, np.int64), rc_cur=np.zeros(n, np.int64))
        if self.events:
            for i in np.flatnonzero(~chk):
                self.admitted(first + int(i), int(g[i]), t)

    def result(self):
        res = self.res
        res.cq_usage = self.usage
        res.wl_evictions = self.evictions
        res.wl_admit_cycle = self.admit_cycle
        res.state = self.state
        res.adm = self.rows.export(hide=[c for c, on in (("wl", self.replay), ("phase", self.pr)) if not on])
        res.wl_admit_ns = self.admit_ns
        res.wl_finish_ns = self.finish_ns
        res.end_ns = self.t
        res.cq_sticky = self.sticky
        if self.quota or self.rc:
            res.cq_generation = self.gen
        if self.rc:
            res.ps_remaining = self.ps_cnt
        if self.backoff:
            res.wl_queue_ts = self.qts
        if self.backoff or self.mx or self.blk:
            res.wl_deactivated, res.wl_deactivation_reason = (self.deactivated != 0).astype(np.uint8), self.deactivated
        if self.mx:
            res.wl_exec_acc_s = self.acc
        if self.checks:
            res.wl_ready_ns, res.wl_check_retries = self.ready_ns, self.retries
        if self.pr:
            res.wl_pods_ready_at, res.wl_pods_ready_count = self.pr_at, self.pr_count
        if self.decay:
            res.lq_consumed = self.consumed.astype(np.int64)
            res.lq_consumed_scale = self.cscale.astype(np.int32)
            res.lq_last_update_ns = self.lq_last
            res.n_afs_samples = self.n_samples
        return res
