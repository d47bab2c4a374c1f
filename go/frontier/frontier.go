// Package frontier is the cgo binding of include/bobrafrontier.h: the per-reconcile "which steps are ready now?"
// computation of internal/controller/runs/dag.go evaluated for a whole batch of StoryRuns on H100 GPUs.
//
// SOURCE ONLY in this repository: the build image has no Go toolchain.  What keeps it honest without one:
//   - every C call goes through go/frontier/shim.h — flat arguments, structs built on the C stack — and
//     tests/c_abi_harness.c compiles that same header with gcc and performs this file's call sequence on a GPU;
//   - no call passes a pointer to Go memory that holds Go pointers (the cgo rule the previous draft broke): Go only
//     hands over &slice[0] of pointer-free slices, or C / pinned memory it got from the library.
//
// Build (on a box with Go + the built library):
//
//	CGO_CFLAGS="-I${REPO}/include -I${REPO}/go/frontier" CGO_LDFLAGS="-L${REPO}/bobrapet_b200/lib -lbobrafrontier" go build ./...
package frontier

/*
#include <stdlib.h>
#include "shim.h"
*/
import "C"

import (
	"fmt"
	"unsafe"
)

// Ctx owns one GPU.  bf_ctx is thread-safe (internal mutex); the recommended shape is one batcher goroutine
// per Ctx (INTEGRATION.md).
type Ctx struct{ p *C.bf_ctx }

// Error carries a negative bf_status and the library's text.
type Error struct {
	Status int
	Msg    string
}

func (e *Error) Error() string {
	return fmt.Sprintf("bobrafrontier: %s (%d): %s", C.GoString(C.bf_strerror(C.int(e.Status))), e.Status, e.Msg)
}

func (c *Ctx) err(rc C.int) error {
	if rc == C.BF_OK {
		return nil
	}
	return &Error{Status: int(rc), Msg: C.GoString(C.bf_last_error(c.p))}
}

// New creates the context of one device.
func New(device int) (*Ctx, error) {
	var p *C.bf_ctx
	if rc := C.bfgo_create(C.int32_t(device), &p); rc != C.BF_OK {
		return nil, &Error{Status: int(rc), Msg: "bf_create"}
	}
	return &Ctx{p: p}, nil
}

func (c *Ctx) Close() { C.bf_destroy(c.p); c.p = nil }

func u32p(s []uint32) *C.uint32_t {
	if len(s) == 0 {
		return nil
	}
	return (*C.uint32_t)(unsafe.Pointer(&s[0]))
}
func i32p(s []int32) *C.int32_t {
	if len(s) == 0 {
		return nil
	}
	return (*C.int32_t)(unsafe.Pointer(&s[0]))
}
func u8p(s []uint8) *C.uint8_t {
	if len(s) == 0 {
		return nil
	}
	return (*C.uint8_t)(unsafe.Pointer(&s[0]))
}

// ParallelDesc mirrors bf_parallel_desc (8 bytes, no pointers).
type ParallelDesc struct {
	Step       uint16
	Branches   uint16
	AllowFirst uint32
}

// Topology is one Story generation packed by PackStory: CSR over allStorySteps (dag.go:3270) + step flags.
type Topology struct {
	RowPtr    []uint32 // len S+1
	ColIdx    []uint16 // len E
	StepFlags []uint8  // len S, BF_SF_*
	Parallel  []ParallelDesc
	AllowBits []uint8
}

// PutTopology uploads one topology and returns its slot.  BF_ETOPO means what validateRuntimeDependencyGraph
// (dag.go:3076-3146) reports: an unknown dependency or a cycle.
func (c *Ctx) PutTopology(t *Topology) (uint32, error) {
	var col *C.uint16_t
	if len(t.ColIdx) > 0 {
		col = (*C.uint16_t)(unsafe.Pointer(&t.ColIdx[0]))
	}
	var par *C.bf_parallel_desc
	if len(t.Parallel) > 0 {
		par = (*C.bf_parallel_desc)(unsafe.Pointer(&t.Parallel[0]))
	}
	var slot C.uint32_t
	rc := C.bfgo_topology_put(c.p, C.uint32_t(len(t.StepFlags)), C.uint32_t(len(t.ColIdx)), u32p(t.RowPtr), col, u8p(t.StepFlags),
		par, C.uint32_t(len(t.Parallel)), u8p(t.AllowBits), C.uint32_t(8*len(t.AllowBits)), &slot)
	return uint32(slot), c.err(rc)
}

func (c *Ctx) DropTopology(slot uint32) error { return c.err(C.bf_topology_drop(c.p, C.uint32_t(slot))) }

// StepTiming is one step's timer (bf_step_timing, 8 bytes, no pointers): Code is the BF_DEC_* code the armed timer writes
// when it fires, Delay its clock units after the now of the commit that arms it.  PackStory emits them.
type StepTiming struct {
	Step  uint16
	Code  uint8
	_     uint8
	Delay uint32
}

// PutTimings replaces the step timings of a live slot (bf_topology_timings); none clears them.  CommitTimed arms the
// launched sleep, gate and wait steps that have one.  A drop discards them.
func (c *Ctx) PutTimings(slot uint32, timings []StepTiming) error {
	var tp *C.bf_step_timing
	if len(timings) > 0 {
		tp = (*C.bf_step_timing)(unsafe.Pointer(&timings[0]))
	}
	return c.err(C.bfgo_topology_timings(c.p, C.uint32_t(slot), tp, C.uint32_t(len(timings))))
}

// Batch is a pair of pinned C buffers (bf_alloc_pinned) laid out by bf_layout_init; the packer writes state
// records into State, the library writes result records into Result.  Both are C memory: no cgo pointer rule applies.
type Batch struct {
	Layout C.bf_layout
	N      uint32
	Cap    uint32
	State  unsafe.Pointer
	Result unsafe.Pointer
}

func (c *Ctx) NewBatch(stepsMax, childNibbles, fields, capRuns uint32) (*Batch, error) {
	b := &Batch{Cap: capRuns}
	if rc := C.bf_layout_init(&b.Layout, C.uint32_t(stepsMax), C.uint32_t(childNibbles), C.uint32_t(fields)); rc != C.BF_OK {
		return nil, &Error{Status: int(rc), Msg: "bf_layout_init"}
	}
	if err := c.err(C.bf_alloc_pinned(c.p, C.size_t(capRuns)*C.size_t(b.Layout.state_stride), &b.State)); err != nil {
		return nil, err
	}
	if err := c.err(C.bf_alloc_pinned(c.p, C.size_t(capRuns)*C.size_t(b.Layout.result_stride), &b.Result)); err != nil {
		return nil, err
	}
	return b, nil
}

// StateRecord returns run r's state record as a byte slice over the pinned buffer.
func (b *Batch) StateRecord(r uint32) []byte {
	return unsafe.Slice((*byte)(unsafe.Add(b.State, uintptr(r)*uintptr(b.Layout.state_stride))), int(b.Layout.state_stride))
}

// ResultRecord returns run r's result record.
func (b *Batch) ResultRecord(r uint32) []byte {
	return unsafe.Slice((*byte)(unsafe.Add(b.Result, uintptr(r)*uintptr(b.Layout.result_stride))), int(b.Layout.result_stride))
}

// Counts mirrors bf_counts.
type Counts struct{ Ready, Skip, Expansion, Evals uint64 }

// Eval runs one frontier pass over the batch (H2D state -> kernels -> D2H results), synchronously and
// bounded; a non-nil error makes the reconciler requeue with backoff or fall back to the Go path.
func (c *Ctx) Eval(b *Batch, flags uint32) (Counts, error) {
	var k Counts
	rc := C.bfgo_eval(c.p, &b.Layout, C.uint32_t(b.N), C.uint32_t(flags), 0, b.State, b.Result, (*C.bf_counts)(unsafe.Pointer(&k)))
	return k, c.err(rc)
}

// Compact results: head[r] = low 15 summary bits | listed << 15 | event count << 16 (BF_HEAD_*), events = one uint16 per
// ready / skipped / failed step, step | kind << 10 (BF_EVT_*), run-major in batch order and step-ascending inside a run —
// the order of findReadySteps' lists.  Run r's events are the next head[r]>>16 entries.
const (
	HeadSummaryMask = 0x7FFF
	HeadListed      = 0x8000
	HeadCountShift  = 16
	EvalChangedOnly = 0x10 // BF_EVAL_CHANGED_ONLY: list only the runs whose result differs from the previous tick's
	// bf_eval_device only (a co-located GPU pipeline submitting passes over device buffers; the host-buffer calls ignore them):
	EvalCountsSet = 0x20 // BF_EVAL_COUNTS_SET: the pass overwrites the counts block, nobody zeroes it
	EvalPipelined = 0x40 // BF_EVAL_PIPELINED: the pass is independent of the preceding kernel of its stream and may start in its tail
)

// EvalCompact is Eval with the results as lists.
func (c *Ctx) EvalCompact(b *Batch, flags uint32, head []uint32, events []uint16) (nEvents uint64, nListed uint32, k Counts, err error) {
	var ev *C.uint16_t
	if len(events) > 0 {
		ev = (*C.uint16_t)(unsafe.Pointer(&events[0]))
	}
	var ne C.uint64_t
	var nl C.uint32_t
	rc := C.bfgo_eval_compact(c.p, &b.Layout, C.uint32_t(b.N), C.uint32_t(flags), 0, b.State, u32p(head), ev, C.uint64_t(len(events)),
		&ne, &nl, (*C.bf_counts)(unsafe.Pointer(&k)))
	return uint64(ne), uint32(nl), k, c.err(rc)
}

// SchedRun mirrors bf_sched_run (32 bytes, no pointers).
type SchedRun struct {
	StoryKey, QueueKey uint32
	Priority           int32
	QueuedElapsedS     uint32 // BF_SCHED_NONE when nothing is queued with a StartedAt
	RunPhase           uint32
	_                  [3]uint32
}

// SchedTables are the limits and what the batch does not hold (dag.go:1780-1961).
type SchedTables struct {
	StoryLimit           []int32  // Story.spec.policy.concurrency per story key
	StoryRunningBase     []uint32 // nil = zeros
	QueueLimit           []int32  // scheduling.queues[q].concurrency per queue key
	QueueAgingS          []int32  // scheduling.queues[q].priorityAgingSeconds
	QueueRunningBase     []uint32 // nil = zeros
	QueueMaxPriorityBase []int32  // highest effective priority among runs with demand outside the batch; nil = none
	GlobalLimit          int32    // scheduling.globalConcurrency
	GlobalBase           uint32
}

// SchedResult holds the schedule records (BF_SCHED_STRIDE(words) bytes per run: bf_sched_header, launch,
// queued_story, queued_sched masks) and the totals the "(%d running, limit %d)" messages are formatted from.
type SchedResult struct {
	Records       []byte
	StoryRunning  []uint32
	QueueRunning  []uint32
	QueueMaxPrio  []int32
	GlobalRunning uint32
}

// Schedule applies enforceStoryConcurrency / enforceSchedulingLimits to the ready sets of the batch Eval just
// evaluated: it replaces the three cluster-wide LISTs per reconcile (dag.go:1863-1920) by one reduction per tick.
func (c *Ctx) Schedule(b *Batch, runs []SchedRun, t *SchedTables) (*SchedResult, error) {
	words := uint32(b.Layout.words)
	stride := (16 + 12*words + 15) &^ 15
	res := &SchedResult{
		Records:      make([]byte, int(b.N)*int(stride)),
		StoryRunning: make([]uint32, len(t.StoryLimit)),
		QueueRunning: make([]uint32, len(t.QueueLimit)),
		QueueMaxPrio: make([]int32, len(t.QueueLimit)),
	}
	var rp *C.bf_sched_run
	if len(runs) > 0 {
		rp = (*C.bf_sched_run)(unsafe.Pointer(&runs[0]))
	}
	var rec unsafe.Pointer
	if len(res.Records) > 0 {
		rec = unsafe.Pointer(&res.Records[0])
	}
	rc := C.bfgo_schedule(c.p, &b.Layout, C.uint32_t(b.N), rp, C.uint32_t(len(t.StoryLimit)), C.uint32_t(len(t.QueueLimit)),
		C.int32_t(t.GlobalLimit), C.uint32_t(t.GlobalBase), i32p(t.StoryLimit), u32p(t.StoryRunningBase), i32p(t.QueueLimit),
		i32p(t.QueueAgingS), u32p(t.QueueRunningBase), i32p(t.QueueMaxPriorityBase), rec, u32p(res.StoryRunning),
		u32p(res.QueueRunning), i32p(res.QueueMaxPrio), (*C.uint32_t)(unsafe.Pointer(&res.GlobalRunning)))
	return res, c.err(rc)
}

// RedriveClosure returns, for each (slot, step), the bit mask of the steps a redrive from that step resets
// (resolveRedriveFromStepSet, storyrun_controller.go:535-558).
func (c *Ctx) RedriveClosure(slots, steps []uint32, words uint32) ([]uint32, error) {
	masks := make([]uint32, len(slots)*int(words))
	if len(slots) == 0 {
		return masks, nil
	}
	return masks, c.err(C.bf_topology_closure(c.p, u32p(slots), u32p(steps), C.uint32_t(len(slots)), C.uint32_t(words), u32p(masks)))
}

// Delta mirrors bf_delta: one changed code of one state record.
type Delta struct {
	Run   uint32
	Index uint16
	Field uint8
	Code  uint8
}

// Resident is a device-resident batch (row f2): full records travel once, afterwards only deltas.
type Resident struct {
	c      *Ctx
	handle C.uint32_t
	layout C.bf_layout
	timerK uint32 // slots per run of the timer area (EnableTimers), 0 without one
}

func (c *Ctx) NewResident(layout C.bf_layout, capacity uint32) (*Resident, error) {
	r := &Resident{c: c, layout: layout}
	return r, c.err(C.bf_resident_create(c.p, &r.layout, C.uint32_t(capacity), &r.handle))
}

func (r *Resident) Close() error { return r.c.err(C.bf_resident_destroy(r.c.p, r.handle)) }

// Upload sends full state records for runs [first, first+n) (new StoryRuns, or a resync).
func (r *Resident) Upload(first, n uint32, records unsafe.Pointer) error {
	return r.c.err(C.bf_resident_upload(r.c.p, r.handle, C.uint32_t(first), C.uint32_t(n), records))
}

// Tick is the steady-state reconcile tick: the deltas syncStateFromStepRuns (dag.go:965-1009) produced go up, the
// pass runs over the resident state, and the ready / skipped steps come back as lists; with EvalChangedOnly only the
// runs whose result changed since the previous tick are listed (the batcher keeps every run's last Row).
func (r *Resident) Tick(deltas []Delta, n, flags uint32, head []uint32, events []uint16) (nEvents uint64, nListed uint32, k Counts, err error) {
	var dp *C.bf_delta
	if len(deltas) > 0 {
		dp = (*C.bf_delta)(unsafe.Pointer(&deltas[0]))
	}
	var ev *C.uint16_t
	if len(events) > 0 {
		ev = (*C.uint16_t)(unsafe.Pointer(&events[0]))
	}
	var ne C.uint64_t
	var nl C.uint32_t
	rc := C.bfgo_resident_tick_compact(r.c.p, r.handle, dp, C.uint32_t(len(deltas)), C.uint32_t(n), C.uint32_t(flags), 0, u32p(head), ev,
		C.uint64_t(len(events)), &ne, &nl, (*C.bf_counts)(unsafe.Pointer(&k)))
	return uint64(ne), uint32(nl), k, r.c.err(rc)
}

// Touched describes a TickTouched call: Full when every run in [0, n) was evaluated and listed (first tick, topology drop,
// changed fixpoint flag or iteration cap, n beyond the last full tick), else only the runs touched since they were last
// evaluated were; runs / head / events then hold what a changed-only Tick would list for them.
type Touched struct {
	Full       bool
	NListed    uint32 // listed runs; runs / head hold the first min(NListed, len) of them
	NEvaluated uint32
	NEvents    uint64
}

// TickTouched is the steady-state tick of a batcher that ticks often: the deltas go up, and only the runs that received a
// delta or an upload since they were last evaluated are evaluated; of those, the ones whose result changed (or that were
// uploaded) come back in runs (ascending) with their head words and events.  Counts cover the evaluated runs.  Use Tick with
// EvalChangedOnly as the resync check.
func (r *Resident) TickTouched(deltas []Delta, n, flags uint32, runs, head []uint32, events []uint16) (t Touched, k Counts, err error) {
	var dp *C.bf_delta
	if len(deltas) > 0 {
		dp = (*C.bf_delta)(unsafe.Pointer(&deltas[0]))
	}
	var ev *C.uint16_t
	if len(events) > 0 {
		ev = (*C.uint16_t)(unsafe.Pointer(&events[0]))
	}
	capRuns := len(runs)
	if len(head) < capRuns {
		capRuns = len(head)
	}
	var full, nl, ne C.uint32_t
	var nev C.uint64_t
	rc := C.bfgo_resident_tick_touched(r.c.p, r.handle, dp, C.uint32_t(len(deltas)), C.uint32_t(n), C.uint32_t(flags), 0, u32p(runs),
		u32p(head), C.uint32_t(capRuns), ev, C.uint64_t(len(events)), &full, &nl, &ne, &nev, (*C.bf_counts)(unsafe.Pointer(&k)))
	return Touched{Full: full != 0, NListed: uint32(nl), NEvaluated: uint32(ne), NEvents: uint64(nev)}, k, r.c.err(rc)
}

// TickPart is one batch of Ctx.TickTouched, with the arguments Resident.TickTouched takes for it.
type TickPart struct {
	R      *Resident
	Deltas []Delta
	N      uint32
	Runs   []uint32
	Head   []uint32
	Events []uint16
}

// TickTouched runs the touched ticks of several batches of this ctx, e.g. one per width class, in one call and one
// synchronisation (bf_resident_tick_touched_many).  Part i gets what parts[i].R.TickTouched would give, called in order; its
// lists land in parts[i].Runs / Head / Events as there.  badPart names the first refused part, or the first part with a
// rejected delta (the call still ticked every part then), or is CommitNone.  Pass the same batches to ScheduleResident next.
func (c *Ctx) TickTouched(flags uint32, parts ...TickPart) (ts []Touched, ks []Counts, badPart uint32, err error) {
	n := len(parts)
	handles, nRuns := make([]uint32, n), make([]uint32, n)
	deltaFirst, runsFirst, eventsFirst := make([]uint32, n+1), make([]uint32, n+1), make([]uint64, n+1)
	var deltas []Delta
	for i, p := range parts {
		handles[i], nRuns[i] = p.R.handle, p.N
		deltas = append(deltas, p.Deltas...)
		capRuns := len(p.Runs)
		if len(p.Head) < capRuns {
			capRuns = len(p.Head)
		}
		deltaFirst[i+1] = deltaFirst[i] + uint32(len(p.Deltas))
		runsFirst[i+1] = runsFirst[i] + uint32(capRuns)
		eventsFirst[i+1] = eventsFirst[i] + uint64(len(p.Events))
	}
	// one flat buffer per list (Go memory without Go pointers), copied back into each part's slices
	runs, head, events := make([]uint32, runsFirst[n]+1), make([]uint32, runsFirst[n]+1), make([]uint16, eventsFirst[n]+1)
	var dp *C.bf_delta
	if len(deltas) > 0 {
		dp = (*C.bf_delta)(unsafe.Pointer(&deltas[0]))
	}
	full, nl, ne := make([]uint32, n+1), make([]uint32, n+1), make([]uint32, n+1)
	nev := make([]uint64, n+1)
	ks = make([]Counts, n+1)
	var bad C.uint32_t
	rc := C.bfgo_resident_tick_touched_many(c.p, C.uint32_t(flags), 0, C.uint32_t(n), u32p(handles), u32p(nRuns), dp, u32p(deltaFirst),
		u32p(runs), u32p(head), u32p(runsFirst), (*C.uint16_t)(unsafe.Pointer(&events[0])),
		(*C.uint64_t)(unsafe.Pointer(&eventsFirst[0])), u32p(full), u32p(nl), u32p(ne), (*C.uint64_t)(unsafe.Pointer(&nev[0])),
		(*C.bf_counts)(unsafe.Pointer(&ks[0])), &bad)
	ts = make([]Touched, n)
	for i, p := range parts {
		ts[i] = Touched{Full: full[i] != 0, NListed: nl[i], NEvaluated: ne[i], NEvents: nev[i]}
		copy(p.Runs, runs[runsFirst[i]:runsFirst[i+1]])
		copy(p.Head, head[runsFirst[i]:runsFirst[i+1]])
		copy(p.Events, events[eventsFirst[i]:eventsFirst[i+1]])
	}
	return ts, ks[:n], uint32(bad), c.err(rc)
}

// MigrateGone marks an old step that has no step of the new Story generation (BF_MIGRATE_GONE).
const MigrateGone = 0xFFFF

// Migrate moves the live runs in [0, n) of an edited Story from its old topology slot to the new one, re-indexing their step
// state on the device by name (stepMap from MigrationMap).  Afterwards the old slot may be dropped; the next TickTouched lists
// every migrated run.  A kept parallel step whose branch count changed is rejected: re-pack and Upload those runs instead.
func (r *Resident) Migrate(oldSlot, newSlot uint32, stepMap []uint16, n uint32) (migrated uint32, err error) {
	var mp *C.uint16_t
	if len(stepMap) > 0 {
		mp = (*C.uint16_t)(unsafe.Pointer(&stepMap[0]))
	}
	var m C.uint32_t
	rc := C.bfgo_resident_migrate(r.c.p, r.handle, C.uint32_t(oldSlot), C.uint32_t(newSlot), mp, C.uint32_t(len(stepMap)), C.uint32_t(n), &m)
	return uint32(m), r.c.err(rc)
}

// RedriveAll is the Redrive.Step of a redrive of the whole run (BF_REDRIVE_ALL, resetStoryRunForRedrive).
const RedriveAll = 0xFFFFFFFF

// Redrive is one request of Resident.Redrive (bf_redrive, 16 bytes): reset run Run, held on topology slot Slot, from step
// Step (an allStorySteps index: the step and everything downstream of it in its group) or, with RedriveAll, entirely.
type Redrive struct {
	Run      uint32
	Slot     uint32
	Step     uint32
	Reserved uint32 // 0
}

// Redrive applies operator redrives to live runs on the device: the reset steps lose their phase, gate decision and
// primitive children, their cond codes become HOLD (steps with an `if`) or PASS, and the TopologyTerminated flag is cleared.
// Call it once the reference's cleanup of the StepRuns and child StoryRuns has finished, then patch the observed annotation.
// status (nil, or at least len(reqs) long) receives 1 per applied request and 0 for a run that no longer holds the slot.
// The next TickTouched evaluates the reset runs and lists the ones whose result changed.
func (r *Resident) Redrive(reqs []Redrive, status []uint8) (applied uint32, err error) {
	if status != nil && len(status) < len(reqs) {
		return 0, fmt.Errorf("frontier: status holds %d entries for %d requests", len(status), len(reqs))
	}
	var rp *C.bf_redrive
	if len(reqs) > 0 {
		rp = (*C.bf_redrive)(unsafe.Pointer(&reqs[0]))
	}
	var sp *C.uint8_t
	if len(status) > 0 {
		sp = (*C.uint8_t)(unsafe.Pointer(&status[0]))
	}
	var a C.uint32_t
	rc := C.bfgo_resident_redrive(r.c.p, r.handle, rp, C.uint32_t(len(reqs)), sp, &a)
	return uint32(a), r.c.err(rc)
}

// Reshape grows the batch in place to the layout bf_layout_init(stepsMax, childNibbles, fields) and capacity runs, keeping
// every run's state, the current results and the touched-tick bookkeeping (bf_resident_reshape).  Growth only: a smaller
// capacity, steps_max or child area, or a dropped field, is an error and changes nothing.  Call it when a Story or the run
// count does not fit, then upload or migrate.  With an output field added, the next TickTouched is a full one.
func (r *Resident) Reshape(stepsMax, childNibbles, fields, capacity uint32) error {
	var L C.bf_layout
	rc := C.bfgo_resident_reshape(r.c.p, r.handle, C.uint32_t(stepsMax), C.uint32_t(childNibbles), C.uint32_t(fields),
		C.uint32_t(capacity), &L)
	if rc == C.BF_OK {
		r.layout = L
	}
	return r.c.err(rc)
}

// Retire takes runs (distinct indices below nRuns) out of the batch, typically terminal StoryRuns the batcher no longer
// needs rows for, at the latest on the informer's delete (bf_resident_retire).  The last live runs move into the freed
// indices: run from[i] now lives at to[i], ascending by target, and the batch's runs become [0, newN).  Re-key the rows by the
// moves; the next TickTouched lists every moved run under its new index.  capacity 0 keeps the capacity, else it becomes
// capacity (newN <= capacity <= current) and the memory above it is released.  A bad argument changes nothing.
func (r *Resident) Retire(nRuns uint32, runs []uint32, capacity uint32) (newN uint32, from, to []uint32, err error) {
	from = make([]uint32, len(runs)+1)
	to = make([]uint32, len(runs)+1)
	var rp *C.uint32_t
	if len(runs) > 0 {
		rp = (*C.uint32_t)(unsafe.Pointer(&runs[0]))
	}
	var nOut, nMoves C.uint32_t
	rc := C.bfgo_resident_retire(r.c.p, r.handle, C.uint32_t(nRuns), rp, C.uint32_t(len(runs)), C.uint32_t(capacity),
		(*C.uint32_t)(unsafe.Pointer(&from[0])), (*C.uint32_t)(unsafe.Pointer(&to[0])), &nOut, &nMoves)
	return uint32(nOut), from[:nMoves], to[:nMoves], r.c.err(rc)
}

// Extent is the smallest layout a batch's contents allow (bf_extent): a Narrow to StepsMax, ChildNibbles and a superset of
// Fields succeeds.  WidestRun is the lowest run that needs StepsMax, or 0xFFFFFFFF when none does.
type Extent struct {
	StepsMax, ChildNibbles, Fields, WidestRun uint32
}

// Extent reports the smallest layout the runs [0, nRuns) and every record of the batch allow (bf_resident_extent).  Query it
// after a Retire: when it is well below the layout, Narrow; when one straggler holds the width, WidestRun names it.
func (r *Resident) Extent(nRuns uint32) (Extent, error) {
	var out [4]C.uint32_t
	rc := C.bfgo_resident_extent(r.c.p, r.handle, C.uint32_t(nRuns), &out[0])
	return Extent{uint32(out[0]), uint32(out[1]), uint32(out[2]), uint32(out[3])}, r.c.err(rc)
}

// Narrow re-lays the batch in place at the smaller layout bf_layout_init(stepsMax, childNibbles, fields), keeping every run's
// state, the current results and, unless decision planes, the child area or an output field are dropped, the touched-tick
// bookkeeping (bf_resident_narrow).  A layout below the extent of the runs [0, nRuns) and the batch's records is an error that
// changes nothing; the returned Extent says why.
func (r *Resident) Narrow(stepsMax, childNibbles, fields, nRuns uint32) (Extent, error) {
	var out [4]C.uint32_t
	var L C.bf_layout
	rc := C.bfgo_resident_narrow(r.c.p, r.handle, C.uint32_t(stepsMax), C.uint32_t(childNibbles), C.uint32_t(fields),
		C.uint32_t(nRuns), &out[0], &L)
	if rc == C.BF_OK {
		r.layout = L
	}
	return Extent{uint32(out[0]), uint32(out[1]), uint32(out[2]), uint32(out[3])}, r.c.err(rc)
}

// Transfer is what TransferTo reports.  SrcN and DstN are the batches' run counts afterwards; the source's run From[i] moved to
// To[i] (bf_resident_retire's moves).  On a refusal because a run does not fit the destination layout, Unfit is its position
// in runs and Why its own extent; otherwise Unfit is 0xFFFFFFFF.
type Transfer struct {
	SrcN, DstN uint32
	From, To   []uint32
	Unfit      uint32
	Why        Extent
}

// TransferTo moves runs (distinct indices below srcN) of this batch to dst, a batch of the same Frontier, where runs[i] becomes
// run dstN + i, re-laid to dst's layout with its state, its current result and a must-list mark (bf_resident_transfer).  This
// batch compacts as by Retire: re-key its rows by From / To and the moved ones to dstN + i.  Use it for width classes: after
// (or instead of) Migrate when a Story edit changes a run's class, and for a live straggler that holds a batch's width.  Grow
// dst with Reshape first when it is full.  A refusal changes neither batch.
func (r *Resident) TransferTo(dst *Resident, srcN, dstN uint32, runs []uint32) (Transfer, error) {
	from := make([]uint32, len(runs)+1)
	to := make([]uint32, len(runs)+1)
	var rp *C.uint32_t
	if len(runs) > 0 {
		rp = (*C.uint32_t)(unsafe.Pointer(&runs[0]))
	}
	var counts, why [4]C.uint32_t
	rc := C.bfgo_resident_transfer(r.c.p, r.handle, dst.handle, C.uint32_t(srcN), C.uint32_t(dstN), rp, C.uint32_t(len(runs)),
		(*C.uint32_t)(unsafe.Pointer(&from[0])), (*C.uint32_t)(unsafe.Pointer(&to[0])), &counts[0], &why[0])
	t := Transfer{SrcN: uint32(counts[0]), DstN: uint32(counts[1]), From: from[:counts[2]], To: to[:counts[2]], Unfit: uint32(counts[3]),
		Why: Extent{uint32(why[0]), uint32(why[1]), uint32(why[2]), uint32(why[3])}}
	return t, r.c.err(rc)
}

// SlotNone is a SlotMap entry of TransferToCtx that maps no slot (BF_SLOT_NONE).
const SlotNone = 0xFFFFFFFF

// Why TransferToCtx found a run unfit (BF_UNFIT_*).
const (
	UnfitNone         = 0 // every run fits
	UnfitLayout       = 1 // the destination layout or its areas cannot hold the run, as for TransferTo
	UnfitSlotUnmapped = 2 // SlotMap maps the run's slot to SlotNone
	UnfitSlotPastMap  = 3 // the run's slot is at or past len(SlotMap)
	UnfitSlotDead     = 4 // the run's slot is not live in the source Frontier
)

// CtxTransfer is what TransferToCtx reports: Transfer's fields, and on a refusal of a run UnfitReason (Unfit*).
type CtxTransfer struct {
	Transfer
	UnfitReason uint32
}

// TransferToCtx moves runs of this batch to dst, a batch of another Frontier (another GPU, or another ctx of the same one), as
// TransferTo does within one (bf_resident_transfer_ctx): both batches end as TransferTo leaves them, with each arrival's
// topology slot taken through slotMap (this Frontier's slot s -> dst's slot slotMap[s], SlotNone where unmapped).  Put the same
// Story generations into both Frontiers first; map the slots the moved runs hold, since the call compares the topology record
// of every mapped slot with its image.  A refusal changes neither batch; Unfit and UnfitReason name the run.
func (r *Resident) TransferToCtx(dst *Resident, srcN, dstN uint32, runs, slotMap []uint32) (CtxTransfer, error) {
	from := make([]uint32, len(runs)+1)
	to := make([]uint32, len(runs)+1)
	var rp, mp *C.uint32_t
	if len(runs) > 0 {
		rp = (*C.uint32_t)(unsafe.Pointer(&runs[0]))
	}
	if len(slotMap) > 0 {
		mp = (*C.uint32_t)(unsafe.Pointer(&slotMap[0]))
	}
	var counts [5]C.uint32_t
	var why [4]C.uint32_t
	rc := C.bfgo_resident_transfer_ctx(r.c.p, r.handle, dst.c.p, dst.handle, C.uint32_t(srcN), C.uint32_t(dstN), rp,
		C.uint32_t(len(runs)), mp, C.uint32_t(len(slotMap)), (*C.uint32_t)(unsafe.Pointer(&from[0])),
		(*C.uint32_t)(unsafe.Pointer(&to[0])), &counts[0], &why[0])
	t := CtxTransfer{Transfer: Transfer{SrcN: uint32(counts[0]), DstN: uint32(counts[1]), From: from[:counts[2]], To: to[:counts[2]],
		Unfit: uint32(counts[3]), Why: Extent{uint32(why[0]), uint32(why[1]), uint32(why[2]), uint32(why[3])}},
		UnfitReason: uint32(counts[4])}
	return t, r.c.err(rc)
}

// Timer is one arm request of ArmTimers (bf_timer): firing at Deadline writes Code (a DecSucceed for a sleep, a timed-out code
// for a gate or wait) as the step's decision code; Code 0 (pending) is wake-only; Deadline TimerNone cancels.
type Timer struct {
	Run      uint32
	Step     uint16
	Code     uint8
	_        uint8
	Deadline uint32
	_        uint32
}

// Fired is one due timer of Fire (bf_fired): Written is 1 when its code was written and the run touched.
type Fired struct {
	Run     uint32
	Step    uint16
	Code    uint8
	Written uint8
}

// TimerNone is an empty slot's deadline, a cancel's deadline, and NextDeadline when nothing is armed.
const TimerNone = 0xFFFFFFFF

// FireResult is what Fire reports.  NextDeadline is the batcher's next wake-up: sleep until min(NextDeadline, the next event).
type FireResult struct {
	NFired, NWritten, NPruned, NextDeadline uint32
	Fired                                   []Fired
}

// EnableTimers gives the batch slotsPerRun timer slots per run (1..64), or grows them keeping every armed timer
// (bf_resident_timers).  Retire, TransferTo, Migrate and Redrive re-key the timers with the runs from then on.
func (r *Resident) EnableTimers(slotsPerRun uint32) error {
	err := r.c.err(C.bf_resident_timers(r.c.p, r.handle, C.uint32_t(slotsPerRun)))
	if err == nil {
		r.timerK = slotsPerRun
	}
	return err
}

// ArmTimers arms, replaces or cancels the timers of (run, step) pairs (bf_resident_timers_arm): the sleepUntil, gateTimeoutAt,
// waitTimeoutAt and pollInterval entries of a run's step-timers annotation.  A refusal changes nothing.
func (r *Resident) ArmTimers(timers []Timer) error {
	var tp *C.bf_timer
	if len(timers) > 0 {
		tp = (*C.bf_timer)(unsafe.Pointer(&timers[0]))
	}
	return r.c.err(C.bf_resident_timers_arm(r.c.p, r.handle, tp, C.uint32_t(len(timers))))
}

// Fire fires the timers of runs [0, n) due at now (bf_resident_fire), before TickTouched: the written codes touch their runs
// as deltas do.  fired receives the first len(fired) due timers, ascending by run and step.
func (r *Resident) Fire(n, now uint32, fired []Fired) (FireResult, error) {
	var fp *C.bf_fired
	if len(fired) > 0 {
		fp = (*C.bf_fired)(unsafe.Pointer(&fired[0]))
	}
	var counts [5]C.uint32_t
	rc := C.bfgo_resident_fire(r.c.p, r.handle, C.uint32_t(n), C.uint32_t(now), fp, C.uint32_t(len(fired)), &counts[0])
	return FireResult{NFired: uint32(counts[0]), NWritten: uint32(counts[1]), NPruned: uint32(counts[2]),
		NextDeadline: uint32(counts[3]), Fired: fired[:counts[4]]}, r.c.err(rc)
}

// Run-level entries of a Fire: Step holds one of these instead of a step index.
const (
	FiredDrain = 0xFFFE // the graceful-cancel drain deadline is due: force-delete the run's StepRuns (wake-only)
	FiredStory = 0xFFFF // the story timeout fired: the run is stopped; patch the StoryRun to Timeout and retire it when done
)

// IsStoryTimeout reports a story timeout (enforceStoryTimeout): the device stopped the run.
func (f Fired) IsStoryTimeout() bool { return f.Step == FiredStory }

// IsDrain reports a due graceful-cancel drain deadline (handleGracefulCancel's force-delete time); it wrote nothing.
func (f Fired) IsDrain() bool { return f.Step == FiredDrain }

// Why a run is stopped (BF_STOP_*).
const (
	StopNone    = 0
	StopTimeout = 1 // policy.timeouts.story elapsed
	StopCancel  = 2 // spec.cancelRequested
	StopHost    = 3 // any other reason the host stops DAG evaluation
)

// RunCtl is one run-control request of PutRunCtl (bf_run_ctl_put, 16 bytes, no pointers): both deadlines on Fire's clock
// (TimerNone: none) and a stop (StopNone: deadlines only).
type RunCtl struct {
	Run, StoryDeadline, DrainDeadline uint32
	Stop                              uint8
	reserved                          [3]uint8
}

// EnableRunCtl gives the batch its run-control area (bf_resident_runctl): stops and story / drain deadlines kept on the device.
func (r *Resident) EnableRunCtl() error { return r.c.err(C.bf_resident_runctl(r.c.p, r.handle)) }

// PutRunCtl writes the deadlines of chosen runs and stops those with a Stop (bf_resident_runctl_put): StartedAt +
// timeouts.story when a run is first packed or its StartedAt is set; StopCancel with observedAt + gracefulShutdownTimeout on
// cancelRequested.  A stopped run lists no ready step and no launch until a redrive.  At most one request per run; a refusal
// changes nothing.  One request goes through the flat shim wrapper, several through one call.
func (r *Resident) PutRunCtl(reqs []RunCtl) error {
	if len(reqs) == 1 {
		q := reqs[0]
		return r.c.err(C.bfgo_resident_runctl_put1(r.c.p, r.handle, C.uint32_t(q.Run), C.uint32_t(q.StoryDeadline),
			C.uint32_t(q.DrainDeadline), C.uint8_t(q.Stop)))
	}
	var rp *C.bf_run_ctl_put
	if len(reqs) > 0 {
		rp = (*C.bf_run_ctl_put)(unsafe.Pointer(&reqs[0]))
	}
	return r.c.err(C.bf_resident_runctl_put(r.c.p, r.handle, rp, C.uint32_t(len(reqs))))
}

// Kinds of a CommitEntry (BF_COMMIT_*): what the host's StepExecutor.Execute did with a launched step other than launch it.
const (
	CommitHold  = 1          // Execute was blocked on template evaluation: the step gets no launch write
	CommitError = 2          // Execute failed: the whole run gets no write (nothing of the reconcile is persisted)
	CommitPhase = 3          // Code is the with.phase of a launched stop step (executeStopStep)
	CommitNone  = 0xFFFFFFFF // BadRun / BadStep of a refusal of the whole call
)

// CommitEntry is one exception of Commit (bf_commit_entry, 8 bytes, no pointers), at most one per (run, step).
type CommitEntry struct {
	Run        uint32
	Step       uint16
	Kind, Code uint8
}

// CommitResult is what Commit wrote (steps whose code changed) and, on a refusal, the first offending (run, step).
type CommitResult struct {
	RunsWritten, Skipped, Launched, Queued, Failed uint32
	BadRun, BadStep                                uint32
}

// Commit writes the decisions of the last tick and schedule of runs [0, n) into the batch's records (bf_resident_commit):
// skipped steps Skipped, cond-FAIL steps Failed, launched steps what Execute writes for their type, queued steps Pending
// queued.  Call it after Execute has run the launches of ScheduleResident (or of TickTouched without limiter inputs); entries
// report the held steps, the runs whose Execute failed and the phase of every launched stop step.  The batcher then sends no
// echo deltas for these writes.  A refusal changes nothing and names the offender in BadRun / BadStep.
func (r *Resident) Commit(n uint32, entries []CommitEntry) (CommitResult, error) {
	var ep *C.bf_commit_entry
	if len(entries) > 0 {
		ep = (*C.bf_commit_entry)(unsafe.Pointer(&entries[0]))
	}
	var k [7]C.uint32_t
	rc := C.bfgo_resident_commit(r.c.p, r.handle, C.uint32_t(n), ep, C.uint32_t(len(entries)), &k[0])
	res := CommitResult{uint32(k[0]), uint32(k[1]), uint32(k[2]), uint32(k[3]), uint32(k[4]), uint32(k[5]), uint32(k[6])}
	return res, r.c.err(rc)
}

// CommitTimed is Commit that also arms the step timers of the launched sleep, gate and wait steps with a timing (PutTimings)
// at now + Delay (bf_resident_commit_timed); a step whose timer is already armed keeps it.  Armed is the number of slots it
// armed and NextDeadline the earliest of them (TimerNone: none): sleep until the smaller of it and Fire's NextDeadline.  A
// run that would hold more than the batch's slots per run is refused with ENOMEM: grow them with EnableTimers and repeat.
func (r *Resident) CommitTimed(n, now uint32, entries []CommitEntry) (res CommitResult, armed, nextDeadline uint32, err error) {
	var ep *C.bf_commit_entry
	if len(entries) > 0 {
		ep = (*C.bf_commit_entry)(unsafe.Pointer(&entries[0]))
	}
	var k [9]C.uint32_t
	rc := C.bfgo_resident_commit_timed(r.c.p, r.handle, C.uint32_t(n), ep, C.uint32_t(len(entries)), C.uint32_t(now), &k[0])
	res = CommitResult{uint32(k[0]), uint32(k[1]), uint32(k[2]), uint32(k[3]), uint32(k[4]), uint32(k[5]), uint32(k[6])}
	return res, uint32(k[7]), uint32(k[8]), r.c.err(rc)
}

// Fields of a CommitWrite: a step's phase code (BF_DELTA_PHASE), a parallel desc's children_registered bit
// (BF_DELTA_REGISTERED) or a newly armed step timer (BF_COMMIT_WRITE_TIMER).
const (
	CommitWritePhase      = 0
	CommitWriteRegistered = 5
	CommitWriteTimer      = 0x10
)

// CommitWriteRewrite is the Code of a phase item of CommitRewrites whose code comes from the stages G / H / I of a single pass
// (BF_COMMIT_WRITE_REWRITE), not from the tick's masks.
const CommitWriteRewrite = 0x1

// CommitWrite is one item of a commit's journal (bf_commit_write, 16 bytes, no pointers): a step whose stored phase code changed
// (Before: the stored nibble, 15 as stored; After: the code written), a desc whose registered bit was set (0 -> 1), or a timer
// slot armed for step Index (Code: the armed decision code; Before: TimerNone; After: the deadline).
type CommitWrite struct {
	Run         uint32
	Index       uint16
	Field, Code uint8
	Before      uint32
	After       uint32
}

// Journal is what CommitJournal wrote.  Items and Runs are the prefixes of the caller's buffers that were filled; NItems and
// NRuns are the true counts (larger than the buffers when they were too small: the commit itself was applied in full).
type Journal struct {
	Items               []CommitWrite
	NItems              uint64
	Runs                []uint32 // ascending runs whose record changed: the runs the commit wrote
	NRuns               uint32
	Armed, NextDeadline uint32
}

// CommitJournal is Commit (now == TimerNone) or CommitTimed (any other now) that also lists every write it made, in
// bf_resident_commit_journal's order (run, then phase, registered and timer items, then index), into items and runs.  The
// batcher persists these writes to StoryRun.status instead of re-deriving them (GroupWrites builds the per-run PATCH), and
// takes the runs whose status to read (Status) from Journal.Runs.  A refusal changes nothing and lists nothing.
func (r *Resident) CommitJournal(n, now uint32, entries []CommitEntry, items []CommitWrite, runs []uint32) (CommitResult, Journal, error) {
	var ep *C.bf_commit_entry
	if len(entries) > 0 {
		ep = (*C.bf_commit_entry)(unsafe.Pointer(&entries[0]))
	}
	var ip *C.bf_commit_write
	if len(items) > 0 {
		ip = (*C.bf_commit_write)(unsafe.Pointer(&items[0]))
	}
	var rp *C.uint32_t
	if len(runs) > 0 {
		rp = (*C.uint32_t)(unsafe.Pointer(&runs[0]))
	}
	var k [10]C.uint32_t
	var nItems C.uint64_t
	rc := C.bfgo_resident_commit_journal(r.c.p, r.handle, C.uint32_t(n), ep, C.uint32_t(len(entries)), C.uint32_t(now), ip,
		C.uint64_t(len(items)), rp, C.uint32_t(len(runs)), &k[0], &nItems)
	res := CommitResult{uint32(k[0]), uint32(k[1]), uint32(k[2]), uint32(k[3]), uint32(k[4]), uint32(k[5]), uint32(k[6])}
	j := Journal{NItems: uint64(nItems), NRuns: uint32(k[9]), Armed: uint32(k[7]), NextDeadline: uint32(k[8])}
	j.Items = items[:minU64(j.NItems, uint64(len(items)))]
	j.Runs = runs[:minU64(uint64(j.NRuns), uint64(len(runs)))]
	return res, j, r.c.err(rc)
}

// CommitRewrites is CommitJournal through bf_resident_commit_rewrites: the commit also stores the phases a single pass's stages
// G, H and I rewrote (fired sleeps, decided or timed-out gates and waits, joined parallel steps, fail-fast and compensation
// skips, a terminated topology's Failed codes), and lists each as a phase item with Code CommitWriteRewrite.  The batcher persists
// them in the same status PATCH (GroupWrites: a rewrite whose After is terminal finishes its step).  -> also the number of steps
// written from the stages.
func (r *Resident) CommitRewrites(n, now uint32, entries []CommitEntry, items []CommitWrite, runs []uint32) (CommitResult, Journal, uint32, error) {
	var ep *C.bf_commit_entry
	if len(entries) > 0 {
		ep = (*C.bf_commit_entry)(unsafe.Pointer(&entries[0]))
	}
	var ip *C.bf_commit_write
	if len(items) > 0 {
		ip = (*C.bf_commit_write)(unsafe.Pointer(&items[0]))
	}
	var rp *C.uint32_t
	if len(runs) > 0 {
		rp = (*C.uint32_t)(unsafe.Pointer(&runs[0]))
	}
	var k [11]C.uint32_t
	var nItems C.uint64_t
	rc := C.bfgo_resident_commit_rewrites(r.c.p, r.handle, C.uint32_t(n), ep, C.uint32_t(len(entries)), C.uint32_t(now), ip,
		C.uint64_t(len(items)), rp, C.uint32_t(len(runs)), &k[0], &nItems)
	res := CommitResult{uint32(k[0]), uint32(k[1]), uint32(k[2]), uint32(k[3]), uint32(k[4]), uint32(k[5]), uint32(k[6])}
	j := Journal{NItems: uint64(nItems), NRuns: uint32(k[9]), Armed: uint32(k[7]), NextDeadline: uint32(k[8])}
	j.Items = items[:minU64(j.NItems, uint64(len(items)))]
	j.Runs = runs[:minU64(uint64(j.NRuns), uint64(len(runs)))]
	return res, j, uint32(k[10]), r.c.err(rc)
}

// EnableCommitMarks gives the batch its commit-due bits (bf_resident_commit_marks), which CommitTouched needs: one bit per run,
// every run due.  Calling it again makes every run due again.
func (r *Resident) EnableCommitMarks() error {
	return r.c.err(C.bf_resident_commit_marks(r.c.p, r.handle))
}

// CommitScope says what a touched commit considered: Full when it took every run of [0, n), else the runs whose writes could
// not be in place (those the touched ticks evaluated, the schedule changed or the entries named since their last touched
// commit); NConsidered counts them.
type CommitScope struct {
	Full        bool
	NConsidered uint32
}

// CommitTouched is the commit the arguments pick, through bf_resident_commit_touched: CommitTimed when now != TimerNone, else
// Commit; CommitJournal into items and runs when journal is set; CommitRewrites when rewrites is set too.  Its results are
// exactly that form's, at the cost of the runs it considers instead of all n: use it in the steady-state loop, after
// EnableCommitMarks.  -> also the steps written from the stages (rewrites) and the scope.
func (r *Resident) CommitTouched(n, now uint32, entries []CommitEntry, journal, rewrites bool, items []CommitWrite,
	runs []uint32) (CommitResult, Journal, uint32, CommitScope, error) {
	var ep *C.bf_commit_entry
	if len(entries) > 0 {
		ep = (*C.bf_commit_entry)(unsafe.Pointer(&entries[0]))
	}
	var ip *C.bf_commit_write
	if len(items) > 0 {
		ip = (*C.bf_commit_write)(unsafe.Pointer(&items[0]))
	}
	var rp *C.uint32_t
	if len(runs) > 0 {
		rp = (*C.uint32_t)(unsafe.Pointer(&runs[0]))
	}
	var flags, jn C.uint32_t
	if rewrites {
		flags = C.BF_COMMIT_SCOPE_REWRITES
	}
	if journal {
		jn = 1
	}
	var k [13]C.uint32_t
	var nItems C.uint64_t
	rc := C.bfgo_resident_commit_touched(r.c.p, r.handle, C.uint32_t(n), ep, C.uint32_t(len(entries)), C.uint32_t(now), flags, jn,
		ip, C.uint64_t(len(items)), rp, C.uint32_t(len(runs)), &k[0], &nItems)
	res := CommitResult{uint32(k[0]), uint32(k[1]), uint32(k[2]), uint32(k[3]), uint32(k[4]), uint32(k[5]), uint32(k[6])}
	j := Journal{NItems: uint64(nItems), NRuns: uint32(k[9]), Armed: uint32(k[7]), NextDeadline: uint32(k[8])}
	j.Items = items[:minU64(j.NItems, uint64(len(items)))]
	j.Runs = runs[:minU64(uint64(j.NRuns), uint64(len(runs)))]
	return res, j, uint32(k[10]), CommitScope{Full: k[11] != 0, NConsidered: uint32(k[12])}, r.c.err(rc)
}

func minU64(a, b uint64) uint64 {
	if a < b {
		return a
	}
	return b
}

// RunWrites are one run's items of a journal, split by field, each ascending by index: what one StoryRun status PATCH carries.
// A Phases item whose Before is 0 or 15 (no phase yet) and whose After is not is a step that starts now, and one whose After is
// terminal a step that finishes now: the StartedAt / FinishedAt that ensureStepStateTimes (step_state.go:25) sets.
type RunWrites struct {
	Run        uint32
	Phases     []CommitWrite
	Registered []uint16 // parallel descs whose children_registered bit was set
	Timers     []CommitWrite
}

// GroupWrites splits a journal's items (ordered by run) into one RunWrites per run, in run order.  The slices share items.
func GroupWrites(items []CommitWrite) []RunWrites {
	var out []RunWrites
	for i := 0; i < len(items); {
		j := i
		for j < len(items) && items[j].Run == items[i].Run {
			j++
		}
		w := RunWrites{Run: items[i].Run}
		for _, it := range items[i:j] {
			switch it.Field {
			case CommitWritePhase:
				w.Phases = append(w.Phases, it)
			case CommitWriteRegistered:
				w.Registered = append(w.Registered, it.Index)
			case CommitWriteTimer:
				w.Timers = append(w.Timers, it)
			}
		}
		out = append(out, w)
		i = j
	}
	return out
}

// Outcomes of a StatusRecord (BF_OUTCOME_*) and the kinds of its events (BF_STATUS_EVT_*).
const (
	OutcomeNone               = 0 // the run's group is not done
	OutcomeSucceeded          = 1 // no group failed: evaluate the Story's output template (finalizeSuccessfulRun) before Succeeded
	OutcomeDependencyFailed   = 2 // Failed, reason DependencyFailed
	OutcomeCompensated        = 3 // Compensated, reason Compensated
	OutcomeCompensationFailed = 4 // Failed, reason CompensationFailed
	OutcomeCleanupFailed      = 5 // Failed, reason CleanupFailed
	OutcomeTimedOut           = 6 // stopped at its story deadline: Timeout
	OutcomeCanceled           = 7 // stopped by a cancel: Finished once the drain ends
	OutcomeStopped            = 8 // stopped by the host
	OutcomeDead               = 9 // the run's topology slot is dead or wider than the layout
	StatusEvtFailed           = 1 // a step of the deciding failed set (status.error's failedSteps)
	StatusEvtAllowed          = 2 // an allowed failure (status.allowedFailures)
	StatusNoStep              = 0xFFFF
)

// StatusRecord is one run's report of Status (bf_status_rec, 32 bytes, no pointers).  Its events are
// events[FirstEvent : FirstEvent+NEvents]; Active / Completed / Failed / Skipped are the step counters of the status.
type StatusRecord struct {
	Run, FirstEvent                    uint32
	NEvents, FirstFailed, Summary      uint16
	Group, Outcome, StoryPhase         uint8
	_                                  [7]uint8
	Active, Completed, Failed, Skipped uint16
}

// StatusEvent splits an event of Status: step | phase << 10 | kind << 14.
func StatusEvent(e uint16) (step uint16, phase, kind uint8) {
	return e & 0x3FF, uint8(e>>10) & 0xF, uint8(e >> 14)
}

// Status reports the listed runs' status after the gate, sleep, wait and join syncs and the fail-fast and compensation marking
// a single tick would apply now (bf_resident_status), changing nothing on the device.  runs must ascend strictly below n; nil
// lists every run of [0, n).  statuses receives one record per listed run; events the first len(events) of nEvents events.
func (r *Resident) Status(n uint32, runs []uint32, statuses []StatusRecord, events []uint16) (nEvents uint64, err error) {
	count := int(n)
	var rp *C.uint32_t
	if runs != nil {
		count = len(runs)
		if count > 0 {
			rp = (*C.uint32_t)(unsafe.Pointer(&runs[0]))
		}
	}
	if len(statuses) < count {
		return 0, fmt.Errorf("frontier: statuses holds %d records for %d runs", len(statuses), count)
	}
	var sp *C.bf_status_rec
	if count > 0 {
		sp = (*C.bf_status_rec)(unsafe.Pointer(&statuses[0]))
	}
	var ep *C.uint16_t
	if len(events) > 0 {
		ep = (*C.uint16_t)(unsafe.Pointer(&events[0]))
	}
	var ne C.uint64_t
	rc := C.bfgo_resident_status(r.c.p, r.handle, C.uint32_t(n), rp, C.uint32_t(count), sp, ep, C.uint64_t(len(events)), &ne)
	return uint64(ne), r.c.err(rc)
}

// Drift is one difference Resync found (bf_drift, 16 bytes, no pointers): Field is a Delta* field, Index the step, child nibble or
// parallel desc it names, Device and Record the compared values, the device's and the caller's.
type Drift struct {
	Run            uint32
	Index          uint16
	Field          uint8
	Reserved       uint8
	Device, Record uint32
}

// Resync flags and fields (BF_RESYNC_*): ResyncCheck compares and lists only; ResyncField(f) selects a Delta* field.
const (
	ResyncCheck     = 0x1
	ResyncAllFields = 0x3F
)

// ResyncField is BF_RESYNC_FIELD(f) for a Delta* field.
func ResyncField(f uint8) uint32 { return 1 << f }

// Resync compares the device's records of the listed runs (runs: strictly ascending, below n; nil: every run of [0, n)) with
// records packed from the cluster (one state record per listed run, in list order), lists every difference into drifted and
// items, and without ResyncCheck repairs the runs that drifted (bf_resident_resync).  The counts are the true ones; only the first
// len(drifted) / len(items) entries are written.  On a refusal that names a run (a record holding a slot no put has returned),
// badRun is that run, else SchedNone.
func (r *Resident) Resync(n uint32, runs []uint32, records []byte, fields uint32, check bool, drifted []uint32,
	items []Drift) (nDrifted, nWritten uint32, nItems uint64, badRun uint32, err error) {
	count := int(n)
	var rp *C.uint32_t
	if runs != nil {
		count = len(runs)
		if count > 0 {
			rp = (*C.uint32_t)(unsafe.Pointer(&runs[0]))
		}
	}
	if need := count * int(r.layout.state_stride); len(records) < need {
		return 0, 0, 0, SchedNone, fmt.Errorf("frontier: records holds %d bytes for %d runs of %d", len(records), count,
			int(r.layout.state_stride))
	}
	var recp unsafe.Pointer
	if len(records) > 0 {
		recp = unsafe.Pointer(&records[0])
	}
	var dp *C.uint32_t
	if len(drifted) > 0 {
		dp = (*C.uint32_t)(unsafe.Pointer(&drifted[0]))
	}
	var ip *C.bf_drift
	if len(items) > 0 {
		ip = (*C.bf_drift)(unsafe.Pointer(&items[0]))
	}
	var flags C.uint32_t
	if check {
		flags = ResyncCheck
	}
	var nd, nw, bad C.uint32_t
	var ni C.uint64_t
	rc := C.bfgo_resident_resync(r.c.p, r.handle, C.uint32_t(n), rp, C.uint32_t(count), recp, C.uint32_t(fields), flags, dp,
		C.uint32_t(len(drifted)), ip, C.uint64_t(len(items)), &nd, &nw, &ni, &bad)
	return uint32(nd), uint32(nw), uint64(ni), uint32(bad), r.c.err(rc)
}

// TimerSlot is one step-timer slot of a run as the batch keeps it (bf_timer_slot, 8 bytes, no pointers): Deadline TimerNone is an
// empty slot, whose other bytes are 0.  A run's armed slots come first, ascending by step.
type TimerSlot struct {
	Deadline uint32
	Step     uint16
	Code     uint8
	_        uint8
}

// RunCtlRecord is a run's run control as the batch keeps it (bf_run_ctl, 16 bytes, no pointers); ResyncAreas takes SavedFlags 0.
type RunCtlRecord struct {
	StoryDeadline, DrainDeadline uint32
	Stop, SavedFlags             uint8
	_                            [6]uint8
}

// Areas of ResyncAreas (BF_RESYNC_AREA_*) and the Drift fields it lists (BF_DRIFT_*, clear of the Delta* fields).
const (
	ResyncAreaTimers = 0x1
	ResyncAreaSched  = 0x2
	ResyncAreaRunCtl = 0x4

	DriftTimer            = 8  // Index = step; the deadlines, TimerNone for a side without a slot at the step
	DriftTimerCode        = 9  // Index = step; the codes of the two slots at the step
	DriftSchedStoryKey    = 10 // the five limiter inputs, in SchedPut order
	DriftSchedQueueKey    = 11
	DriftSchedPriority    = 12
	DriftSchedQueuedSince = 13
	DriftSchedRunPhase    = 14
	DriftStoryDeadline    = 15
	DriftDrainDeadline    = 16
	DriftStop             = 17 // the Stop* reasons
)

// ResyncAreas compares the device's step timers, limiter inputs and run control of the listed runs (runs: strictly ascending,
// below n; nil: every run of [0, n)) with the areas packed from the cluster, one row per listed run in list order (timers: the
// slots-per-run slots of each run, canonical, from the step-timers annotation; sched: SchedPut with Run the listed run; runctl:
// the deadlines and the stop), lists every difference into drifted and items, and without ResyncCheck repairs the runs that
// drifted (bf_resident_resync_areas).  A nil slice leaves its area out.  firedNow is the now of the last Fire (TimerNone: none): a
// slot the annotation still holds after a fire disarmed it is taken as fired.  Resync the records first.  The counts are the true
// ones; only the first len(drifted) / len(items) entries are written.  On a refusal that names a run, badRun is that run, else
// SchedNone.
func (r *Resident) ResyncAreas(n uint32, runs []uint32, timers []TimerSlot, sched []SchedPut, runctl []RunCtlRecord,
	firedNow uint32, check bool, drifted []uint32, items []Drift) (nDrifted, nWritten uint32, nItems uint64, badRun uint32, err error) {
	count := int(n)
	var rp *C.uint32_t
	if runs != nil {
		count = len(runs)
		if count > 0 {
			rp = (*C.uint32_t)(unsafe.Pointer(&runs[0]))
		}
	}
	var areas C.uint32_t
	var tp *C.bf_timer_slot
	var sp *C.bf_sched_put
	var cp *C.bf_run_ctl
	if timers != nil {
		areas |= ResyncAreaTimers
		if len(timers) != count*int(r.timerK) {
			return 0, 0, 0, SchedNone, fmt.Errorf("frontier: timers holds %d slots for %d runs of %d", len(timers), count, r.timerK)
		}
		if len(timers) > 0 {
			tp = (*C.bf_timer_slot)(unsafe.Pointer(&timers[0]))
		}
	}
	if sched != nil {
		areas |= ResyncAreaSched
		if len(sched) != count {
			return 0, 0, 0, SchedNone, fmt.Errorf("frontier: sched holds %d rows for %d runs", len(sched), count)
		}
		if count > 0 {
			sp = (*C.bf_sched_put)(unsafe.Pointer(&sched[0]))
		}
	}
	if runctl != nil {
		areas |= ResyncAreaRunCtl
		if len(runctl) != count {
			return 0, 0, 0, SchedNone, fmt.Errorf("frontier: runctl holds %d rows for %d runs", len(runctl), count)
		}
		if count > 0 {
			cp = (*C.bf_run_ctl)(unsafe.Pointer(&runctl[0]))
		}
	}
	var dp *C.uint32_t
	if len(drifted) > 0 {
		dp = (*C.uint32_t)(unsafe.Pointer(&drifted[0]))
	}
	var ip *C.bf_drift
	if len(items) > 0 {
		ip = (*C.bf_drift)(unsafe.Pointer(&items[0]))
	}
	var flags C.uint32_t
	if check {
		flags = ResyncCheck
	}
	var nd, nw, bad C.uint32_t
	var ni C.uint64_t
	rc := C.bfgo_resident_resync_areas(r.c.p, r.handle, C.uint32_t(n), rp, C.uint32_t(count), areas, tp, sp, cp,
		C.uint32_t(firedNow), flags, dp, C.uint32_t(len(drifted)), ip, C.uint64_t(len(items)), &nd, &nw, &ni, &bad)
	return uint32(nd), uint32(nw), uint64(ni), uint32(bad), r.c.err(rc)
}

// SchedPut is one limiter-input request of PutSched (bf_sched_put, 32 bytes, no pointers).  QueuedSince is the StartedAt of the
// run's earliest queued step on the clock of ScheduleResident's now (SchedNone: nothing queued); the device ages from it.
type SchedPut struct {
	Run, StoryKey, QueueKey uint32
	Priority                int32
	QueuedSince, RunPhase   uint32
	_                       [2]uint32
}

// SchedNone is a key, a queue origin or an elapsed time that is absent (BF_SCHED_NONE).
const SchedNone = 0xFFFFFFFF

// SchedHeader mirrors bf_sched_header: the steps to launch, queued by the Story's limit and queued by the scheduling limits,
// and why the latter were queued (BF_QUEUED_*).
type SchedHeader struct {
	NLaunch, NQueuedStory, NQueuedSched, Reason uint32
}

// Event kinds of ScheduleResident (BF_SEVT_*).
const (
	SevtLaunch      = 0x1
	SevtQueuedStory = 0x2
	SevtQueuedSched = 0x4
)

// EnableSched gives the batch its limiter-inputs area, every run at the defaults (no keys, priority 0, nothing queued)
// (bf_resident_sched).  Retire and TransferTo move the inputs with the runs from then on.
func (r *Resident) EnableSched() error { return r.c.err(C.bf_resident_sched(r.c.p, r.handle)) }

// PutSched writes the limiter inputs of chosen runs (bf_resident_sched_put): when the batcher first packs a run, and again when
// its keys, priority, StoryRun phase or queue origin change.  At most one request per run; a refusal changes nothing.
func (r *Resident) PutSched(reqs []SchedPut) error {
	var rp *C.bf_sched_put
	if len(reqs) > 0 {
		rp = (*C.bf_sched_put)(unsafe.Pointer(&reqs[0]))
	}
	return r.c.err(C.bf_resident_sched_put(r.c.p, r.handle, rp, C.uint32_t(len(reqs))))
}

// SchedBuffers are the list buffers of one ScheduleResident part, in pinned C memory so that the kernels write them in place.
type SchedBuffers struct {
	Runs   []uint32
	Heads  []SchedHeader
	Events []uint16
	mem    [3]unsafe.Pointer
}

// NewSchedBuffers allocates the lists of one part: runsCap runs and heads, eventsCap events.
func (c *Ctx) NewSchedBuffers(runsCap, eventsCap uint32) (*SchedBuffers, error) {
	b := &SchedBuffers{}
	sizes := [3]C.size_t{C.size_t(runsCap) * 4, C.size_t(runsCap) * 16, C.size_t(eventsCap) * 2}
	for i, n := range sizes {
		if n == 0 {
			n = 16
		}
		if err := c.err(C.bf_alloc_pinned(c.p, n, &b.mem[i])); err != nil {
			c.FreeSchedBuffers(b)
			return nil, err
		}
	}
	b.Runs = unsafe.Slice((*uint32)(b.mem[0]), runsCap)
	b.Heads = unsafe.Slice((*SchedHeader)(b.mem[1]), runsCap)
	b.Events = unsafe.Slice((*uint16)(b.mem[2]), eventsCap)
	return b, nil
}

// FreeSchedBuffers returns the buffers' pinned memory.
func (c *Ctx) FreeSchedBuffers(b *SchedBuffers) {
	for i, p := range b.mem {
		if p != nil {
			C.bf_free_pinned(c.p, p)
			b.mem[i] = nil
		}
	}
}

// SchedPart is one batch of ScheduleResident: its runs [0, N) are counted and limited, and the listed ones land in Buf.
type SchedPart struct {
	R   *Resident
	N   uint32
	Buf *SchedBuffers
}

// SchedListed is what ScheduleResident reports per part: Buf holds the first min(NListed, len(Buf.Runs)) listed runs and the
// first min(NEvents, len(Buf.Events)) events; Full when every run of [0, N) was listed.
type SchedListed struct {
	NListed uint32
	Full    bool
	NEvents uint64
}

// ScheduleResident limits the runs of every part against one set of totals (bf_resident_schedule): the tables' bases plus
// the Running StepRuns and queue priority maxima of all parts, so the limits and the priority ordering hold across width
// classes.  Call it once per tick after TickTouched of every batch; only the runs whose schedule changed are listed.
func (c *Ctx) ScheduleResident(now uint32, t *SchedTables, parts ...SchedPart) ([]SchedListed, *SchedResult, error) {
	res := &SchedResult{
		StoryRunning: make([]uint32, len(t.StoryLimit)),
		QueueRunning: make([]uint32, len(t.QueueLimit)),
		QueueMaxPrio: make([]int32, len(t.QueueLimit)),
	}
	ps := make([]C.bf_resident_sched_part, len(parts))   // Go memory holding only C pointers
	for i, p := range parts {
		capRuns := len(p.Buf.Runs)
		if len(p.Buf.Heads) < capRuns {
			capRuns = len(p.Buf.Heads)
		}
		var rp *C.uint32_t
		var hp *C.bf_sched_header
		var ep *C.uint16_t
		if capRuns > 0 {
			rp, hp = (*C.uint32_t)(unsafe.Pointer(&p.Buf.Runs[0])), (*C.bf_sched_header)(unsafe.Pointer(&p.Buf.Heads[0]))
		}
		if len(p.Buf.Events) > 0 {
			ep = (*C.uint16_t)(unsafe.Pointer(&p.Buf.Events[0]))
		}
		C.bfgo_sched_part(&ps[i], p.R.handle, C.uint32_t(p.N), rp, hp, C.uint32_t(capRuns), ep, C.uint64_t(len(p.Buf.Events)))
	}
	var pp *C.bf_resident_sched_part
	if len(ps) > 0 {
		pp = &ps[0]
	}
	rc := C.bfgo_resident_schedule(c.p, C.uint32_t(now), C.uint32_t(len(t.StoryLimit)), C.uint32_t(len(t.QueueLimit)),
		C.int32_t(t.GlobalLimit), C.uint32_t(t.GlobalBase), i32p(t.StoryLimit), u32p(t.StoryRunningBase), i32p(t.QueueLimit),
		i32p(t.QueueAgingS), u32p(t.QueueRunningBase), i32p(t.QueueMaxPriorityBase), pp, C.uint32_t(len(ps)),
		u32p(res.StoryRunning), u32p(res.QueueRunning), i32p(res.QueueMaxPrio), (*C.uint32_t)(unsafe.Pointer(&res.GlobalRunning)))
	out := make([]SchedListed, len(parts))
	for i := range ps {
		out[i] = SchedListed{NListed: uint32(ps[i].n_listed), Full: ps[i].full != 0, NEvents: uint64(ps[i].n_events)}
	}
	return out, res, c.err(rc)
}

// ScheduleResidentCtxs is ScheduleResident over batches of several Frontiers, e.g. one per GPU (bf_resident_schedule_ctxs):
// each part's lists and the totals are those of one ScheduleResident over the same batches held in one Frontier, so the
// Story, queue and global limits and the priority ordering count the Running steps of every GPU.  Call it once per tick after
// TickTouched of every Frontier.  A refusal changes nothing, and its text names the refused part whichever Frontier holds it.
func ScheduleResidentCtxs(now uint32, t *SchedTables, parts ...SchedPart) ([]SchedListed, *SchedResult, error) {
	if len(parts) == 0 {
		return nil, nil, &Error{Status: int(C.BF_EINVAL), Msg: "ScheduleResidentCtxs: no parts"}
	}
	res := &SchedResult{
		StoryRunning: make([]uint32, len(t.StoryLimit)),
		QueueRunning: make([]uint32, len(t.QueueLimit)),
		QueueMaxPrio: make([]int32, len(t.QueueLimit)),
	}
	ps := make([]C.bf_resident_sched_part, len(parts)) // Go memory holding only C pointers
	ctxs := make([]*C.bf_ctx, len(parts))
	for i, p := range parts {
		capRuns := len(p.Buf.Runs)
		if len(p.Buf.Heads) < capRuns {
			capRuns = len(p.Buf.Heads)
		}
		var rp *C.uint32_t
		var hp *C.bf_sched_header
		var ep *C.uint16_t
		if capRuns > 0 {
			rp, hp = (*C.uint32_t)(unsafe.Pointer(&p.Buf.Runs[0])), (*C.bf_sched_header)(unsafe.Pointer(&p.Buf.Heads[0]))
		}
		if len(p.Buf.Events) > 0 {
			ep = (*C.uint16_t)(unsafe.Pointer(&p.Buf.Events[0]))
		}
		C.bfgo_sched_part(&ps[i], p.R.handle, C.uint32_t(p.N), rp, hp, C.uint32_t(capRuns), ep, C.uint64_t(len(p.Buf.Events)))
		ctxs[i] = p.R.c.p
	}
	rc := C.bfgo_resident_schedule_ctxs(C.uint32_t(now), C.uint32_t(len(t.StoryLimit)), C.uint32_t(len(t.QueueLimit)),
		C.int32_t(t.GlobalLimit), C.uint32_t(t.GlobalBase), i32p(t.StoryLimit), u32p(t.StoryRunningBase), i32p(t.QueueLimit),
		i32p(t.QueueAgingS), u32p(t.QueueRunningBase), i32p(t.QueueMaxPriorityBase), &ctxs[0], &ps[0], C.uint32_t(len(ps)),
		u32p(res.StoryRunning), u32p(res.QueueRunning), i32p(res.QueueMaxPrio), (*C.uint32_t)(unsafe.Pointer(&res.GlobalRunning)))
	out := make([]SchedListed, len(parts))
	for i := range ps {
		out[i] = SchedListed{NListed: uint32(ps[i].n_listed), Full: ps[i].full != 0, NEvents: uint64(ps[i].n_events)}
	}
	return out, res, parts[0].R.c.err(rc)
}

// Group is one operator process driving several GPUs (bf_group_*): contiguous blocks of runs per device, one NCCL
// all-gather of the per-shard counts per pass, limiter totals all-reduced across the shards.
type Group struct{ p *C.bf_group }

func NewGroup(devices []int32) (*Group, error) {
	var p *C.bf_group
	rc := C.bf_group_create(&p, i32p(devices), C.uint32_t(len(devices)), nil)
	if rc != C.BF_OK {
		return nil, &Error{Status: int(rc), Msg: "bf_group_create"}
	}
	return &Group{p: p}, nil
}

func (g *Group) Close()               { C.bf_group_destroy(g.p); g.p = nil }
func (g *Group) Size() uint32         { return uint32(C.bf_group_size(g.p)) }
func (g *Group) Shard(k uint32) *Ctx  { return &Ctx{p: C.bf_group_ctx(g.p, C.uint32_t(k))} }
func (g *Group) err(rc C.int) error {
	if rc == C.BF_OK {
		return nil
	}
	return &Error{Status: int(rc), Msg: C.GoString(C.bf_group_last_error(g.p))}
}

// ShardRange says which runs of an n-run batch live on shard k (so that the packer writes the shard's own slot ids).
func (g *Group) ShardRange(n, k uint32) (first, count uint32) {
	var f, cnt C.uint32_t
	C.bf_group_shard_range(g.p, C.uint32_t(n), C.uint32_t(k), &f, &cnt)
	return uint32(f), uint32(cnt)
}

// Eval runs the pass on every shard concurrently and returns the per-shard and the global counts.
func (g *Group) Eval(b *Batch, flags uint32) (perShard []Counts, global Counts, err error) {
	perShard = make([]Counts, g.Size())
	rc := C.bfgo_group_eval(g.p, &b.Layout, C.uint32_t(b.N), C.uint32_t(flags), 0, b.State, b.Result,
		(*C.bf_counts)(unsafe.Pointer(&perShard[0])), (*C.bf_counts)(unsafe.Pointer(&global)))
	return perShard, global, g.err(rc)
}
