"""limiters — CPU restatement of the concurrency limiters that consume findReadySteps' list.

TEST INFRASTRUCTURE ONLY (see oracle/README.md): only tests/, __graft_entry__.smoke() and
bench.py's CPU legs may import this module, and only as the checker.

Two layers, as for the frontier pass itself:

* object level (reference-shaped): enforce_story_concurrency / enforce_scheduling_limits /
  enforce_priority_ordering / effective_priority ... follow
  internal/controller/runs/dag.go:1780-1999 and scheduling.go function by function, over
  objects that stand in for the cluster LISTs the reference issues (StepRunList, StoryRunList).
  Pinned by the reference's own tests dag_test.go:528 (BlocksLowerPriority), :579
  (AllowsAgedRun) and :744 (EnforcesConcurrency) in tests/test_limiters_oracle.py.
* packed level: schedule_packed() states the batch contract of include/bobrafrontier.h
  (bf_schedule): ONE consistent snapshot per tick, counts are reductions over the batch's
  own state records plus host-supplied base counts.  Differential against the object level
  on random clusters.

Snapshot contract.  The reference evaluates one StoryRun per reconcile and reads the counts
(running StepRuns per story / queue / cluster, other runs' priorities) from the informer cache at
that moment.  StepRuns created in the same reconcile start without a phase, so they do not count as
Running until the StepRun controller has picked them up (steprun phase "Running" is what
countRunningStepRuns compares, dag.go:1883-1888): within one snapshot every run sees the same
counts.  The batch contract is exactly that: counts first, then every run is limited
independently against them.
"""
from __future__ import annotations

from dataclasses import dataclass, field
from typing import Dict, List, Optional, Tuple

import numpy as np

from oracle.pyoracle import StepState, is_terminal

# dag.go:103-108
STORY_PREFIX = "Queued due to story concurrency limit"
QUEUE_PREFIX = "Queued due to queue concurrency limit"
GLOBAL_PREFIX = "Queued due to global concurrency limit"
PRIORITY_PREFIX = "Queued due to higher-priority work"
QUEUED_PREFIXES = (STORY_PREFIX, QUEUE_PREFIX, GLOBAL_PREFIX, PRIORITY_PREFIX)
DEFAULT_QUEUE = "default"  # scheduling.go:14


# ------------------------------------------------------------------------------------------
# object level
# ------------------------------------------------------------------------------------------
@dataclass
class QueueConfig:
    """config.QueueConfig, internal/config/controller_config.go:533-545."""
    concurrency: int = 0
    default_priority: int = 0
    priority_aging_seconds: int = 0


@dataclass
class SchedulingConfig:
    """config.SchedulingConfig :523-531; default (:731-739): no global limit, queue "default" ages every 60 s."""
    global_concurrency: int = 0
    queues: Dict[str, QueueConfig] = field(default_factory=lambda: {DEFAULT_QUEUE: QueueConfig(0, 0, 60)})


@dataclass
class ClusterStepRun:
    namespace: str
    story_name: str     # contracts.StoryNameLabelKey
    queue_label: str    # contracts.QueueLabelKey
    phase: str = ""


@dataclass
class ClusterStoryRun:
    name: str
    namespace: str
    queue_label: str
    priority_label: Optional[str]   # contracts.QueuePriorityLabelKey (a decimal string) or None
    phase: str = ""
    step_states: Dict[str, StepState] = field(default_factory=dict)


def normalize_queue_name(name: str) -> str:
    """scheduling.go:21-27."""
    return name.strip().lower()


def queue_label_value(queue: str) -> str:
    """scheduling.go:29-35 (coreidentity.SafeLabelValue is the identity on the plain names used here)."""
    n = normalize_queue_name(queue)
    return n if n else DEFAULT_QUEUE


def queue_config_for(cfg: SchedulingConfig, queue: str) -> QueueConfig:
    """scheduling.go:101-112."""
    name = normalize_queue_name(queue) or DEFAULT_QUEUE
    return cfg.queues.get(name, QueueConfig())


def resolve_scheduling_decision(policy_queue: Optional[str], policy_priority: Optional[int], cfg: SchedulingConfig) -> Tuple[str, int]:
    """resolveSchedulingDecision with a nil fallback (the call of dag.go:1805), scheduling.go:130-163."""
    queue, priority = DEFAULT_QUEUE, 0
    story_queue = normalize_queue_name(policy_queue) if policy_queue is not None else ""
    if story_queue != "":
        queue = story_queue
    if policy_priority is not None:
        priority = policy_priority
    else:   # `storyQueue != ""` and the default case both read the decided queue's default priority
        priority = queue_config_for(cfg, queue).default_priority
    if queue.strip() == "":
        queue = DEFAULT_QUEUE
    return queue, priority


def priority_from_labels(label: Optional[str]) -> int:
    """scheduling.go:165-178."""
    if label is None:
        return 0
    raw = label.strip()
    if raw == "":
        return 0
    try:
        v = int(raw, 10)
    except ValueError:
        return 0
    return v if -(1 << 31) <= v < (1 << 31) else 0


def is_concurrency_queued(state: StepState) -> bool:
    """dag.go:2035-2051."""
    return state.phase == "Pending" and state.message.startswith(QUEUED_PREFIXES)


def wrap_int32(v: int) -> int:
    """Go int32 arithmetic: the result modulo 2^32, read as signed."""
    return ((int(v) + (1 << 31)) & 0xFFFFFFFF) - (1 << 31)


def effective_priority(base: int, queued_since: Optional[float], aging_seconds: int, now: float) -> int:
    """dag.go:1948-1961.  int32(elapsed.Seconds()) / agingSeconds, Go integer division; `base + steps` is an int32 sum and
    wraps as in Go (a priority near INT32_MAX that ages becomes a very low one).

    One departure from Go: an elapsed time past INT32_MAX seconds (68 years) is read as INT32_MAX, the clamp of the
    bf_sched_run contract (include/bobrafrontier.h: the host fills queued_elapsed_s so, and the kernel clamps).  Go's
    int32(elapsed.Seconds()) is implementation-defined there (INT32_MIN on amd64, which makes effectivePriority return base)."""
    if queued_since is None or aging_seconds <= 0:
        return base
    elapsed = now - queued_since
    if elapsed <= 0:
        return base
    steps = min(int(elapsed), 0x7FFFFFFF) // aging_seconds
    if steps <= 0:
        return base
    return wrap_int32(base + steps)


def story_run_queued_since(srun: ClusterStoryRun) -> Optional[float]:
    """dag.go:1963-1979: the earliest StartedAt among the queued step states."""
    earliest = None
    for st in srun.step_states.values():
        if not is_concurrency_queued(st) or st.started_at is None:
            continue
        if earliest is None or st.started_at < earliest:
            earliest = st.started_at
    return earliest


def story_run_has_demand(srun: ClusterStoryRun) -> bool:
    """dag.go:1981-1999."""
    if srun.phase in ("Running", "Pending"):
        return True
    for st in srun.step_states.values():
        if st.phase == "Running" or is_concurrency_queued(st):
            return True
    return False


def enforce_priority_ordering(cluster_runs: List[ClusterStoryRun], srun: ClusterStoryRun, queue_name: str,
                              queue_label: str, priority: int, cfg: SchedulingConfig, now: float) -> Tuple[bool, str]:
    """dag.go:1910-1946."""
    if queue_label.strip() == "":
        return False, ""
    if queue_name.strip() == "":
        queue_name = DEFAULT_QUEUE
    aging = queue_config_for(cfg, queue_name).priority_aging_seconds
    current = effective_priority(priority, story_run_queued_since(srun), aging, now)
    for other in cluster_runs:
        if other.queue_label != queue_label:          # client.MatchingLabels{QueueLabelKey: queueLabel}
            continue
        if other.name == srun.name and other.namespace == srun.namespace:
            continue
        if is_terminal(other.phase):
            continue
        if not story_run_has_demand(other):
            continue
        other_eff = effective_priority(priority_from_labels(other.priority_label), story_run_queued_since(other), aging, now)
        if other_eff <= current:
            continue
        return True, PRIORITY_PREFIX
    return False, ""


def count_running_step_runs(step_runs: List[ClusterStepRun], namespace: str, story_name: str) -> int:
    """dag.go:1870-1888."""
    if story_name.strip() == "":
        return 0
    return sum(1 for s in step_runs if s.namespace == namespace and s.story_name == story_name and s.phase == "Running")


def enforce_story_concurrency(step_runs: List[ClusterStepRun], namespace: str, story_name: str, limit: int,
                              ready: List[str]) -> Tuple[List[str], List[str], str]:
    """dag.go:1780-1799."""
    if not ready or limit <= 0:
        return ready, [], ""
    running = count_running_step_runs(step_runs, namespace, story_name)
    slots = max(limit - running, 0)
    if slots >= len(ready):
        return ready, [], ""
    return ready[:slots], ready[slots:], "%s (%d running, limit %d)" % (STORY_PREFIX, running, limit)


def enforce_scheduling_limits(step_runs: List[ClusterStepRun], cluster_runs: List[ClusterStoryRun],
                              srun: ClusterStoryRun, queue: str, priority: int, cfg: SchedulingConfig,
                              ready: List[str], now: float) -> Tuple[List[str], List[str], str]:
    """dag.go:1801-1861."""
    if not ready:
        return ready, [], ""
    qlabel = queue_label_value(queue)
    blocked, reason = enforce_priority_ordering(cluster_runs, srun, queue, qlabel, priority, cfg, now)
    if blocked:
        return [], ready, reason
    glimit = cfg.global_concurrency
    qlimit = queue_config_for(cfg, queue).concurrency
    rg = rq = 0
    gslots = len(ready)
    if glimit > 0:
        rg = sum(1 for s in step_runs if s.phase == "Running")               # :1890-1896
        gslots = max(glimit - rg, 0)
    qslots = len(ready)
    if qlimit > 0:
        rq = sum(1 for s in step_runs if s.queue_label == qlabel and s.phase == "Running")   # :1898-1915
        qslots = max(qlimit - rq, 0)
    slots = min(len(ready), gslots, qslots)
    if slots >= len(ready):
        return ready, [], ""
    if glimit > 0 and (qlimit <= 0 or gslots <= qslots):
        reason = "%s (%d running, limit %d)" % (GLOBAL_PREFIX, rg, glimit)
    elif qlimit > 0:
        reason = "%s (%d running, limit %d)" % (QUEUE_PREFIX, rq, qlimit)
    else:
        reason = "Queued due to scheduling limits"
    return ready[:slots], ready[slots:], reason


@dataclass
class LimitResult:
    launch: List[str]
    queued_story: List[str]
    queued_sched: List[str]
    msg_story: str = ""
    msg_sched: str = ""


def apply_limiters(step_runs: List[ClusterStepRun], cluster_runs: List[ClusterStoryRun], srun: ClusterStoryRun,
                   story_name: str, story_limit: int, queue: str, priority: int, cfg: SchedulingConfig,
                   ready: List[str], now: float) -> LimitResult:
    """The limiter section of findAndLaunchReadySteps, dag.go:1709-1728."""
    ready, q1, m1 = enforce_story_concurrency(step_runs, srun.namespace, story_name, story_limit, list(ready))
    ready, q2, m2 = enforce_scheduling_limits(step_runs, cluster_runs, srun, queue, priority, cfg, ready, now)
    return LimitResult(ready, q1, q2, m1, m2)


# ------------------------------------------------------------------------------------------
# packed level: the bf_schedule contract (include/bobrafrontier.h)
# ------------------------------------------------------------------------------------------
NONE_U32 = 0xFFFFFFFF
REASON_NONE, REASON_PRIORITY, REASON_GLOBAL, REASON_QUEUE, REASON_OTHER = 0, 1, 2, 3, 4
INT32_MIN = -(1 << 31)

SCHED_RUN_DTYPE = np.dtype([("story_key", "<u4"), ("queue_key", "<u4"), ("priority", "<i4"), ("queued_elapsed_s", "<u4"),
                            ("run_phase", "<u4"), ("reserved", "<u4", (3,))])
assert SCHED_RUN_DTYPE.itemsize == 32


def effective_priority_packed(priority: int, elapsed_s: int, aging: int) -> int:
    """effective_priority over the bf_sched_run fields: elapsed_s above INT32_MAX reads as INT32_MAX (the host's
    int32(elapsed.Seconds())), and the sum wraps to int32 as in Go."""
    if elapsed_s == NONE_U32 or aging <= 0 or elapsed_s == 0:
        return priority
    steps = min(elapsed_s, 0x7FFFFFFF) // aging
    return wrap_int32(priority + steps) if steps > 0 else priority


def truncate_mask(words: np.ndarray, keep: int) -> np.ndarray:
    """first `keep` set bits of a little-endian bit mask (step order = list order, dag.go:1796-1798)."""
    out = np.zeros_like(words)
    left = keep
    for w in range(len(words)):
        v = int(words[w])
        o = 0
        while v and left > 0:
            low = v & -v
            o |= low
            v ^= low
            left -= 1
        out[w] = o
    return out


TERMINAL_PHASES = (3, 4, 5, 6, 7, 11, 12, 13)   # BF_LUT_TERMINAL


def schedule_packed(run_running: np.ndarray, run_demand: np.ndarray, sched: np.ndarray, ready_masks: np.ndarray,
                    story_limit: np.ndarray, story_base: np.ndarray, queue_limit: np.ndarray, queue_aging: np.ndarray,
                    queue_base: np.ndarray, global_limit: int, global_base: int, queue_maxprio_base=None):
    """run_running[r]: Running StepRuns the batch attributes to run r (engram steps in phase Running + Running
    children of registered parallel steps); run_demand[r]: some step Running or queued (the run-phase part of
    storyRunHasDemand is added here from sched.run_phase).  Returns (launch, queued_story, queued_sched, info,
    story_running, queue_running, global_running, queue_maxprio); info[r] = (n_launch, n_queued_story,
    n_queued_sched, reason).

    The edges include/bobrafrontier.h pins in its limiter block: a story_key >= n_stories / queue_key >= n_queues is
    counted in no story / queue total and gets no story limit, no queue limit, no aging and no priority ordering (its
    steps still count globally and the global limit still applies); only the low 4 bits of run_phase are read; effective
    priorities and the queue maxima are int32, the aging sum wrapping as in Go."""
    n, W = ready_masks.shape
    ns, nq = len(story_limit), len(queue_limit)
    story_running = story_base.astype(np.int64).copy()
    queue_running = queue_base.astype(np.int64).copy()
    for r in range(n):
        k, q = int(sched["story_key"][r]), int(sched["queue_key"][r])
        if k < ns:
            story_running[k] += int(run_running[r])
        if q < nq:
            queue_running[q] += int(run_running[r])
    global_running = int(global_base) + int(run_running.astype(np.int64).sum())
    eff = np.array([effective_priority_packed(int(sched["priority"][r]), int(sched["queued_elapsed_s"][r]),
                                              int(queue_aging[sched["queue_key"][r]]) if sched["queue_key"][r] < nq else 0)
                    for r in range(n)], dtype=np.int32)
    phase = sched["run_phase"] & 0xF
    term = np.isin(phase, TERMINAL_PHASES)
    demand = np.isin(phase, [1, 2]) | (run_demand != 0)
    maxprio = (np.full(nq, INT32_MIN, dtype=np.int32) if queue_maxprio_base is None
               else np.asarray(queue_maxprio_base, dtype=np.int32).copy())
    for r in range(n):
        q = int(sched["queue_key"][r])
        if not term[r] and demand[r] and q < nq:
            maxprio[q] = max(maxprio[q], eff[r])
    launch = np.zeros_like(ready_masks)
    q_story = np.zeros_like(ready_masks)
    q_sched = np.zeros_like(ready_masks)
    info = np.zeros((n, 4), dtype=np.uint32)
    for r in range(n):
        cur = ready_masks[r].copy()
        cnt = int(sum(bin(int(x)).count("1") for x in cur))
        k, q = int(sched["story_key"][r]), int(sched["queue_key"][r])
        lim = int(story_limit[k]) if k < ns else 0
        if cnt and lim > 0:
            slots = max(lim - int(story_running[k]), 0)
            if slots < cnt:
                kept = truncate_mask(cur, slots)
                q_story[r] = cur & ~kept
                cur = kept
                cnt = slots
        reason = REASON_NONE
        if cnt:
            if q < nq and maxprio[q] > eff[r]:
                q_sched[r] = cur
                cur = np.zeros_like(cur)
                reason = REASON_PRIORITY
            else:
                gl, ql = int(global_limit), int(queue_limit[q]) if q < nq else 0
                gslots = cnt if gl <= 0 else max(gl - global_running, 0)
                qslots = cnt if ql <= 0 else max(ql - int(queue_running[q]), 0)
                slots = min(cnt, gslots, qslots)
                if slots < cnt:
                    kept = truncate_mask(cur, slots)
                    q_sched[r] = cur & ~kept
                    cur = kept
                    if gl > 0 and (ql <= 0 or gslots <= qslots):
                        reason = REASON_GLOBAL
                    elif ql > 0:
                        reason = REASON_QUEUE
                    else:
                        reason = REASON_OTHER
        launch[r] = cur
        pc = lambda m: int(sum(bin(int(x)).count("1") for x in m))
        info[r] = (pc(launch[r]), pc(q_story[r]), pc(q_sched[r]), reason)
    return launch, q_story, q_sched, info, story_running, queue_running, global_running, maxprio
