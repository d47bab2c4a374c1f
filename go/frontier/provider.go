package frontier

import (
	bubuv1alpha1 "github.com/bubustack/bobrapet/api/v1alpha1"
)

// FrontierProvider is the seam DAGReconciler gets (SOURCE ONLY, see frontier.go).
//
// internal/controller/runs/dag.go:1708 today:
//
//	readySteps, skippedSteps, skippedReasons, unskipped := r.findReadySteps(ctx, srun, story, steps,
//	    srun.Status.StepStates, completedSteps, runningSteps, dependencies, vars, depPolicy)
//
// becomes
//
//	if row, ok := r.Frontier.Lookup(string(srun.UID), srun.ResourceVersion); ok {
//	    readySteps, skippedSteps, skippedReasons = row.Steps(allStorySteps(story))
//	} else {
//	    ... the Go path above (first sight of a run, packer miss, or a bf_eval error)
//	}
//
// Ready bits are LSB-first in list order, so the concurrency limiters' readySteps[:slots] (dag.go:1796-1798)
// keep working on the slice returned by Row.Steps.
type FrontierProvider interface {
	// Lookup returns the result row computed for this StoryRun at exactly this resourceVersion, if any.
	Lookup(uid string, resourceVersion string) (Row, bool)
}

// Row is one StoryRun's result of the last tick that listed it, decoded from the compact lists.
type Row struct {
	Summary uint32   // low 15 bits of BF_SUM_*: group evaluated, mainDone / mainFailed flags, "some phase changed"
	Events  []uint16 // this run's slice of the tick's event list: step | kind << 10
	// FailedDep names, per skipped step, the dependency that failed — "Skipped due to failed dependency: <d>"
	// (dag.go:2735-2739): the lowest index among the step's needs whose phase is terminal and not Succeeded/Skipped
	// (the packer fills it from the host copy of the phases; the kernel reports only WHICH steps were skipped for it).
	FailedDep map[uint16]string
}

const (
	evtReady   = 0x1 // BF_EVT_READY
	evtSkip    = 0x2 // BF_EVT_SKIP
	evtSkipDep = 0x10
)

// Rows walks one tick's lists: run r's events are the next head[r]>>16 entries; only listed runs are handed to `set`
// (with BF_EVAL_CHANGED_ONLY the cache keeps the previous Row of every other run).
func Rows(head []uint32, events []uint16, set func(run uint32, row Row)) {
	pos := 0
	for r, h := range head {
		n := int(h >> HeadCountShift)
		if h&HeadListed != 0 {
			set(uint32(r), Row{Summary: h & HeadSummaryMask, Events: events[pos : pos+n]})
		}
		pos += n
	}
}

// RowsTouched walks the lists of a touched tick (Resident.TickTouched): runs[i] is listed with head word head[i], and its
// events are the next head[i]>>16 entries.  Every other run keeps its previous Row.  The caller passes runs[:k] and head[:k],
// k = min(t.NListed, len(runs), len(head)), never the whole buffers (entries past NListed are stale).  Only rows whose events
// arrived whole are handed to `set`; RowsTouched returns false when the event list was cut short, and the caller then resyncs
// (a Tick with EvalChangedOnly, or larger buffers) — as it must when t.NListed exceeded its buffers.
func RowsTouched(runs, head []uint32, events []uint16, set func(run uint32, row Row)) bool {
	pos := 0
	for i, h := range head {
		n := int(h >> HeadCountShift)
		if i >= len(runs) || pos+n > len(events) {
			return false
		}
		set(runs[i], Row{Summary: h & HeadSummaryMask, Events: events[pos : pos+n]})
		pos += n
	}
	return true
}

// SchedRow is one run's schedule from ScheduleResident: its header and the steps of its three masks, ascending.
type SchedRow struct {
	Header                         SchedHeader
	Launch, QueuedStory, QueuedSched []uint16
}

// RowsScheduled decodes the listed runs of a ScheduleResident part: runs[:k], heads[:k] and events with k = min(NListed, buffer
// length), set called once per listed run.  False when the events do not cover the heads (NEvents past the buffer): resync.
// The launch steps go to StepExecutor.Execute, the queued ones to markQueuedSteps.
func RowsScheduled(runs []uint32, heads []SchedHeader, events []uint16, set func(run uint32, row SchedRow)) bool {
	pos := 0
	for i, h := range heads {
		n := int(h.NLaunch + h.NQueuedStory + h.NQueuedSched)
		if i >= len(runs) || pos+n > len(events) {
			return false
		}
		row := SchedRow{Header: h}
		for _, e := range events[pos : pos+n] {
			step := e & 0x3FF
			switch e >> 10 {
			case SevtLaunch:
				row.Launch = append(row.Launch, step)
			case SevtQueuedStory:
				row.QueuedStory = append(row.QueuedStory, step)
			default:
				row.QueuedSched = append(row.QueuedSched, step)
			}
		}
		set(runs[i], row)
		pos += n
	}
	return true
}

// Steps turns the row back into the three results of findReadySteps (dag.go:2631-2641) over `steps` =
// allStorySteps(story) — index i of the packed topology is &steps[i].
func (r Row) Steps(steps []bubuv1alpha1.Step) (ready, skipped []*bubuv1alpha1.Step, reasons map[string]string) {
	reasons = map[string]string{}
	for _, e := range r.Events {
		step, kind := e&0x3FF, e>>10
		if int(step) >= len(steps) {
			continue
		}
		st := &steps[step]
		switch {
		case kind&evtReady != 0:
			ready = append(ready, st)
		case kind&evtSkip != 0:
			skipped = append(skipped, st)
			if kind&evtSkipDep != 0 || r.FailedDep[step] != "" {
				reasons[st.Name] = "Skipped due to failed dependency: " + r.FailedDep[step] // dag.go:2736
			} else {
				reasons[st.Name] = "Skipped due to 'if' condition" // dag.go:2831
			}
		}
	}
	return ready, skipped, reasons
}
