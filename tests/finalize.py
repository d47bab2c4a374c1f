"""finalizeStoryRun (dag.go:693-754) and summarizeStepProgress (:928-942) restated over pyoracle's objects, beside the restatement
of the loop body in oracle/pyoracle.py: what a batcher writes into a StoryRun's status once group selection finds nothing left
to run, and the step counters it writes on every persist."""
from typing import Dict, Tuple

from oracle import pyoracle as O


def failed_sets(story: O.Story, states: Dict[str, O.StepState]):
    """the failed sets of buildStateMaps (dag.go:3358-3391) of the main, compensation and finally groups, as group selection reads
    them after stage I (dag.go:428-473) when `states` are the step states a pass left"""
    return tuple(O.build_state_maps(steps, states)[2] for steps in (story.steps, story.compensations, story.finally_))


def first_failed_step_name(story: O.Story, failed: Dict[str, bool]) -> str:
    """dag.go:3344 takes any key of the map; the contract fixes the lowest step index (allStorySteps order, SURVEY.md 8.0-F)"""
    for st in O.all_story_steps(story):
        if failed.get(st.name):
            return st.name
    return ""


def finalize_story_run(story: O.Story, states: Dict[str, O.StepState], main_failed: Dict[str, bool],
                       comp_failed: Dict[str, bool], final_failed: Dict[str, bool]):
    """-> (StoryRun phase, condition reason, message, failedSteps of status.error as {name: phase}).  A run without failures gets
    ("Succeeded", "", "", {}): finalizeSuccessfulRun (the Story's output template) stays with the caller."""
    def listed(failed):   # BuildStoryRunError, pkg/runs/status/storyrun.go:165-189
        return {n: states[n].phase if n in states else "" for n in failed}
    if final_failed:
        return "Failed", "CleanupFailed", "Finally step %s failed." % first_failed_step_name(story, final_failed), listed(final_failed)
    if comp_failed:
        return ("Failed", "CompensationFailed", "Compensation step %s failed." % first_failed_step_name(story, comp_failed),
                listed(comp_failed))
    if main_failed:
        if story.compensations:
            return "Compensated", "Compensated", "Story failed; compensations completed.", listed(main_failed)
        return ("Failed", "DependencyFailed", "Story completed with failed step: %s." % first_failed_step_name(story, main_failed),
                listed(main_failed))
    return "Succeeded", "", "", {}


def summarize_step_progress(states: Dict[str, O.StepState]) -> Tuple[int, int, int, int]:
    """-> (active, completed, failed, skipped): Running or Paused / Succeeded / Failed / Skipped; every other phase counts in none"""
    active = completed = failed = skipped = 0
    for st in states.values():
        if st.phase in ("Running", "Paused"):
            active += 1
        elif st.phase == "Succeeded":
            completed += 1
        elif st.phase == "Failed":
            failed += 1
        elif st.phase == "Skipped":
            skipped += 1
    return active, completed, failed, skipped
