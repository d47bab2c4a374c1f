package frontier

// packer.go — the step BEFORE the kernel (SURVEY.md rows a10 / f2): CRD objects -> packed records.
//
// Everything here is host work the reference already does per reconcile, done once per Story generation (topology)
// and once per changed code (state): names -> indices, `needs` + template references -> CSR, StepState.Phase -> 4-bit
// code (with the "Queued due to ..." message folded in), gate / sleep / wait status -> decision code.  SOURCE ONLY
// (no Go toolchain in the build image); the C++ twin that IS compiled and tested against the same rules is
// bobrapet_b200/csrc/host_mirror.cc (tests/test_host_mirror.py), and tests/packing.py is the test-side statement.

import (
	"encoding/json"
	"regexp"
	"strings"
	"time"

	runsv1alpha1 "github.com/bubustack/bobrapet/api/runs/v1alpha1"
	bubuv1alpha1 "github.com/bubustack/bobrapet/api/v1alpha1"
	"github.com/bubustack/bobrapet/pkg/enums"
)

// step flag bits (include/bobrafrontier.h BF_SF_*)
const (
	sfAllowFailure  = 0x08
	sfOnTimeoutSkip = 0x10
	sfHasIf         = 0x20
	sfGroupShift    = 6
)

// phaseCode: declaration order of enums.Phase (pkg/enums/enums.go:44-97); 0 = no StepState entry.
var phaseCode = map[enums.Phase]uint8{
	"": 0, enums.PhasePending: 1, enums.PhaseRunning: 2, enums.PhaseSucceeded: 3, enums.PhaseFailed: 4,
	enums.PhaseFinished: 5, enums.PhaseCanceled: 6, enums.PhaseCompensated: 7, enums.PhasePaused: 8,
	enums.PhaseBlocked: 9, enums.PhaseScheduling: 10, enums.PhaseTimeout: 11, enums.PhaseAborted: 12, enums.PhaseSkipped: 13,
}

// the four prefixes of isConcurrencyQueued (dag.go:103-108, 2035-2051)
var queuedPrefixes = []string{
	"Queued due to story concurrency limit", "Queued due to queue concurrency limit",
	"Queued due to global concurrency limit", "Queued due to higher-priority work",
}

// PhaseCode is the 4-bit code of one StepState: 14 = Pending whose message says the limiter queued it, so that
// clearConcurrencyQueuedSteps (dag.go:2020-2033) needs no second input.
func PhaseCode(st runsv1alpha1.StepState, present bool) uint8 {
	if !present {
		return 0
	}
	if st.Phase == enums.PhasePending {
		for _, p := range queuedPrefixes {
			if strings.HasPrefix(st.Message, p) {
				return 14
			}
		}
	}
	return phaseCode[st.Phase]
}

// step type codes (BF_STEP_*): a step with Ref set is an engram whatever its Type says (step_executor.go:150-166)
func typeCode(s *bubuv1alpha1.Step) uint8 {
	if s.Ref != nil {
		return 0
	}
	switch s.Type {
	case enums.StepTypeCondition:
		return 1
	case enums.StepTypeParallel:
		return 2
	case enums.StepTypeSleep:
		return 3
	case enums.StepTypeStop:
		return 4
	case enums.StepTypeWait:
		return 5
	case enums.StepTypeExecuteStory:
		return 6
	case enums.StepTypeGate:
		return 7
	}
	return 0
}

// the three template-reference forms buildDependencyGraphs scans for (dag.go:3028-3030)
var stepRef = regexp.MustCompile(
	`steps\.([a-zA-Z0-9_\-]+)\.|steps\s*\[\s*['"]([a-zA-Z0-9_\-]+)['"]\s*\]|\(index\s+\.steps\s+["']([a-zA-Z0-9_\-]+)["']\)`)

// alias of a step name inside templates: every rune outside [A-Za-z0-9_] becomes '_' (sanitizeStepIdentifier,
// step_executor.go:1652-1670)
func alias(name string) string {
	b := []byte(name)
	for i, ch := range b {
		ok := ch >= 'a' && ch <= 'z' || ch >= 'A' && ch <= 'Z' || ch >= '0' && ch <= '9' || ch == '_'
		if !ok {
			b[i] = '_'
		}
	}
	return string(b)
}

// PackedStory is a Story generation ready for Ctx.PutTopology, plus the name tables the decode side needs.
type PackedStory struct {
	Topology Topology
	Names    []string          // index -> step name, allStorySteps order (dag.go:3270-3280)
	Index    map[string]uint16 // step name -> index
	Branches [][]string        // per parallel desc: branch names in with.steps order
	Unknown  []string          // dependency names that match no step ("unknown step dependencies", dag.go:3087-3098)
	Timings  []StepTiming      // for Ctx.PutTimings: the sleep, gate and wait steps' timers, ascending by step (stepTiming)
}

// PackStory builds the CSR of buildDependencyGraphs (dag.go:3024-3073) over allStorySteps.  The reference builds the
// graph from the CURRENT group's step list, so alias -> name resolution sees only that group's names, while a
// dependency may name a step of any group: both rules are kept (per-group alias maps, global index space).
// parallelBranches(step) returns the branch names and allowFailure flags of a `parallel` step's with.steps
// (parseParallelBranches, dag.go:1202-1214) — JSON decoding stays with the caller.  unit is the step timers' clock unit
// (Resident.Fire's now): each sleep, gate and wait step gets its timing in Timings (0: none are packed).
func PackStory(story *bubuv1alpha1.Story, parallelBranches func(*bubuv1alpha1.Step) ([]string, []bool), onTimeoutSkip func(*bubuv1alpha1.Step) bool,
	unit time.Duration) *PackedStory {
	groups := [][]bubuv1alpha1.Step{story.Spec.Steps, story.Spec.Compensations, story.Spec.Finally}
	ps := &PackedStory{Index: map[string]uint16{}}
	for _, g := range groups {
		for i := range g {
			ps.Index[g[i].Name] = uint16(len(ps.Names))
			ps.Names = append(ps.Names, g[i].Name)
		}
	}
	t := &ps.Topology
	t.RowPtr = append(t.RowPtr, 0)
	for gi, g := range groups {
		aliasToReal := map[string]string{}
		for i := range g {
			if a := alias(g[i].Name); a != g[i].Name {
				aliasToReal[a] = g[i].Name
			}
		}
		for i := range g {
			s := &g[i]
			seen := map[uint16]bool{}
			var row []uint16
			add := func(dep string) {
				idx, ok := ps.Index[dep]
				if !ok {
					ps.Unknown = append(ps.Unknown, dep)
					return
				}
				if !seen[idx] { // the reference's adjacency is a set
					seen[idx] = true
					row = append(row, idx)
				}
			}
			scan := func(expr string) {
				for _, m := range stepRef.FindAllStringSubmatch(expr, -1) {
					dep := m[3]
					if dep == "" {
						dep = m[2]
					}
					if dep == "" {
						dep = m[1]
					}
					if dep == "" {
						continue
					}
					if real, ok := aliasToReal[dep]; ok {
						dep = real
					}
					add(dep)
				}
			}
			for _, d := range s.Needs {
				add(d)
			}
			if s.If != nil {
				scan(*s.If)
			}
			if s.With != nil && (s.Ref != nil || s.Type == enums.StepTypeExecuteStory) {
				scan(string(s.With.Raw))
			}
			t.ColIdx = append(t.ColIdx, row...)
			t.RowPtr = append(t.RowPtr, uint32(len(t.ColIdx)))

			f := typeCode(s) | uint8(gi)<<sfGroupShift
			if s.AllowFailure != nil && *s.AllowFailure {
				f |= sfAllowFailure
			}
			if s.If != nil && *s.If != "" {
				f |= sfHasIf
			}
			if onTimeoutSkip != nil && onTimeoutSkip(s) {
				f |= sfOnTimeoutSkip
			}
			t.StepFlags = append(t.StepFlags, f)
			if unit > 0 {
				if code, delay, ok := stepTiming(s, typeCode(s), unit); ok {
					ps.Timings = append(ps.Timings, StepTiming{Step: ps.Index[s.Name], Code: code, Delay: delay})
				}
			}
			if typeCode(s) == 2 && parallelBranches != nil {
				names, allow := parallelBranches(s)
				first := uint32(8 * len(t.AllowBits))
				bits := make([]uint8, (len(names)+7)/8)
				for b, a := range allow {
					if a {
						bits[b/8] |= 1 << (b % 8)
					}
				}
				t.AllowBits = append(t.AllowBits, bits...)
				t.Parallel = append(t.Parallel, ParallelDesc{Step: ps.Index[s.Name], Branches: uint16(len(names)), AllowFirst: first})
				ps.Branches = append(ps.Branches, names)
			}
		}
	}
	return ps
}

// decision codes a timer writes (BF_DEC_*)
const (
	decPending  = 0
	decSucceed  = 1
	decFail     = 2
	decTimedOut = 3
)

// positive is parsePositiveDuration (steprun_controller.go:1364)
func positive(raw string) (time.Duration, bool) {
	d, err := time.ParseDuration(raw)
	return d, err == nil && d > 0
}

// units rounds d up to whole clock units, so that no armed timer fires before the reference's deadline
func units(d, unit time.Duration) uint32 {
	n := (d + unit - 1) / unit
	if d > 0 && n <= 0 || n > 0xFFFFFFFF {
		return 0xFFFFFFFF
	}
	return uint32(n)
}

// stepTiming is what parseSleepConfig / parseGateConfig / parseWaitConfig (dag.go:1549-1653) make of a step's `with`: the
// code its timer writes and its delay in clock units, or ok = false (no timer: a gate without a timeout takes its decision
// as a delta).  A `with` the reference refuses fails the step at once (FAIL, 0: :1239-1249, :1331-1341, :1477-1487); a sleep
// without a duration completes on its next sync (SUCCEED, 0: :1252-1254).  tests/step_timings.py states the same rules.
func stepTiming(s *bubuv1alpha1.Step, ty uint8, unit time.Duration) (code uint8, delay uint32, ok bool) {
	onTimeout := func(raw string) bool {
		v := strings.ToLower(strings.TrimSpace(raw))
		return v == "" || v == "fail" || v == "skip"
	}
	switch ty {
	case 3: // sleep
		if s.With == nil || len(s.With.Raw) == 0 {
			return decSucceed, 0, true
		}
		var raw struct {
			Duration string `json:"duration"`
		}
		if json.Unmarshal(s.With.Raw, &raw) != nil {
			return decFail, 0, true
		}
		if strings.TrimSpace(raw.Duration) == "" {
			return decSucceed, 0, true
		}
		d, good := positive(raw.Duration)
		if !good {
			return decFail, 0, true
		}
		return decSucceed, units(d, unit), true
	case 7, 5: // gate, wait
		if s.With == nil {
			if ty == 5 {
				return decFail, 0, true
			}
			return 0, 0, false
		}
		var raw struct {
			Until        string `json:"until"`
			Timeout      string `json:"timeout,omitempty"`
			PollInterval string `json:"pollInterval,omitempty"`
			OnTimeout    string `json:"onTimeout,omitempty"`
		}
		if json.Unmarshal(s.With.Raw, &raw) != nil || !onTimeout(raw.OnTimeout) || (ty == 5 && strings.TrimSpace(raw.Until) == "") {
			return decFail, 0, true
		}
		var timeout, poll time.Duration
		if raw.Timeout != "" {
			d, good := positive(raw.Timeout)
			if !good {
				return decFail, 0, true
			}
			timeout = d
		}
		if raw.PollInterval != "" {
			d, good := positive(raw.PollInterval)
			if !good {
				return decFail, 0, true
			}
			poll = d
		}
		switch {
		case timeout > 0:
			return decTimedOut, units(timeout, unit), true
		case ty == 5 && poll > 0:
			return decPending, units(poll, unit), true // wake-only: the host re-evaluates until
		}
	}
	return 0, 0, false
}

// run flag bits (BF_RF_*)
const (
	rfFailFast           = 0x01
	rfRealtime           = 0x02
	rfTopologyTerminated = 0x04
)

// MigrationMap is the step map of Resident.Migrate for an edited Story: stepMap[i] is the index in newer of the step named
// older.Names[i], or MigrateGone.  The reference keys StepStates, Gates and PrimitiveChildren by name and walks the current
// Story's allStorySteps on every reconcile (getStoryForRun, storyrun_controller.go:1297-1313), so state follows the name.
// added lists the names of newer that older lacks: a name that existed in an earlier generation may still have a StepState
// in the StoryRun, which the migrated record does not carry; send deltas for it.
func MigrationMap(older, newer *PackedStory) (stepMap []uint16, added []string) {
	stepMap = make([]uint16, len(older.Names))
	for i, n := range older.Names {
		stepMap[i] = MigrateGone
		if j, ok := newer.Index[n]; ok {
			stepMap[i] = j
		}
	}
	for _, n := range newer.Names {
		if _, ok := older.Index[n]; !ok {
			added = append(added, n)
		}
	}
	return stepMap, added
}

// RunFlags: shouldFailFast (dag.go:3504-3511), Pattern.IsRealtime (enums.go:335), and the Degraded /
// TopologyTerminated condition the caller read from the StoryRun (dag.go:436-464).
func RunFlags(story *bubuv1alpha1.Story, topologyTerminated bool) uint8 {
	f := uint8(rfFailFast)
	if p := story.Spec.Policy; p != nil && p.Retries != nil && p.Retries.ContinueOnStepFailure != nil && *p.Retries.ContinueOnStepFailure {
		f = 0
	}
	if story.Spec.Pattern.IsRealtime() {
		f |= rfRealtime
	}
	if topologyTerminated {
		f |= rfTopologyTerminated
	}
	return f
}

// decision codes (BF_DEC_*)
const (
	DecPending  = 0
	DecSucceed  = 1
	DecFail     = 2
	DecTimedOut = 3
)

// GateDecision maps status.gates[name].state to the decision code of a gate step (dag.go:1489-1533): Approved and
// Rejected win over an elapsed timeout; the time comparison itself (parseGateConfig, :1519-1531) is the caller's.
func GateDecision(gs runsv1alpha1.GateStatus, present, timedOut bool) uint8 {
	if present {
		switch gs.State {
		case runsv1alpha1.GateDecisionApproved:
			return DecSucceed
		case runsv1alpha1.GateDecisionRejected:
			return DecFail
		}
	}
	if timedOut {
		return DecTimedOut
	}
	return DecPending
}

// setCode writes a k-bit code of step i into a bit-sliced field (k planes of `words` u32, include/bobrafrontier.h
// "record layout"): the O(1) in-place update a StepRun watch event turns into.
func setCode(field []byte, words uint32, nbits int, i uint32, code uint8) {
	w, bit := i>>5, byte(1)<<(i&7)
	byteIn := (i & 31) >> 3
	for b := 0; b < nbits; b++ {
		p := (uint32(b)*words+w)*4 + byteIn
		if code>>uint(b)&1 != 0 {
			field[p] |= bit
		} else {
			field[p] &^= bit
		}
	}
}

// PackRun writes one StoryRun's state record (bf_run_header + phase planes [+ decision planes]) into rec
// (Batch.StateRecord(r)); slot is the topology slot of the run's Story ON THE SHARD THAT OWNS THE RUN.
// Cond codes and child phases are written by the caller the same way (setCode on off_cond; nibbles at off_child).
func PackRun(rec []byte, L BatchLayout, ps *PackedStory, slot uint32, flags uint8, srun *runsv1alpha1.StoryRun, timedOut func(step string) bool) {
	for i := range rec {
		rec[i] = 0
	}
	rec[0], rec[1], rec[2], rec[3] = byte(slot), byte(slot>>8), byte(slot>>16), byte(slot>>24)
	rec[4] = flags
	var registered uint64
	for q := range ps.Topology.Parallel {
		if len(srun.Status.PrimitiveChildren[ps.Names[ps.Topology.Parallel[q].Step]]) > 0 { // dag.go:1140
			registered |= 1 << uint(q)
		}
	}
	for b := 0; b < 8; b++ {
		rec[8+b] = byte(registered >> (8 * uint(b)))
	}
	for i, name := range ps.Names {
		st, ok := srun.Status.StepStates[name]
		setCode(rec[L.OffPhase:], L.Words, 4, uint32(i), PhaseCode(st, ok))
		if L.OffDecision != offNone && ps.Topology.StepFlags[i]&7 == 7 { // gate
			gs, present := srun.Status.Gates[name]
			setCode(rec[L.OffDecision:], L.Words, 2, uint32(i), GateDecision(gs, present, timedOut != nil && timedOut(name)))
		}
	}
}

const offNone = 0xFFFFFFFF

// BatchLayout is the Go view of bf_layout (filled from Batch.Layout).
type BatchLayout struct {
	Words, OffPhase, OffCond, OffDecision, OffChild uint32
}
