"""The daemon's gate in front of NodeSelect, restated from the reference's text.

TEST INFRASTRUCTURE ONLY (nothing under cranesched_b200/ may import it).

Before NodeSelect, ScheduleThread_ drops from the pending vector every job that is
held, whose begin time is ahead, or whose dependencies are not met
(JobScheduler.cpp:1090-1113); the dependency state is updated by the events queued
since the last tick (:1073-1088). `Deps` is DependenciesInJob (CtldPublicDefs.h:413-428,
update at CtldPublicDefs.cpp:144-159, SetDependency at :1600-1611); `Daemon` models the
call sites that queue the events, keyed by job id:

    submit      JobScheduler.cpp:4215-4248, AddDependent (CtldPublicDefs.cpp:1617-1626):
                a pending dependee registers the dependent, a running one too except that
                AFTER fires at once at its start time; a missing or ended one rejects
    start       :1549                AFTER at the start time
    cancel      :4067-4073           AFTER, AFTER_ANY at the cancel time; AFTER_OK,
                                     AFTER_NOT_OK at InfiniteFuture
    end         :4531-4538           AFTER_ANY at the end time; AFTER_OK at the end time if
                                     the exit code is 0 else InfiniteFuture; AFTER_NOT_OK
                                     the other way round
    recover     Init, :552-594       events of dependees that ended before the restart

The queued events are applied here as they happen rather than at the next tick: `update`
is a min or a max and an erase, which commute, and the state is only read at a tick.
"""
from __future__ import annotations

from dataclasses import dataclass, field

PAST = -(2 ** 63)     # absl::InfinitePast()
FUTURE = 2 ** 63 - 1  # absl::InfiniteFuture()
AFTER, AFTER_ANY, AFTER_OK, AFTER_NOT_OK = 0, 1, 2, 3  # PublicDefs.proto:136-141

# reason codes of include/crane_sched.h
NONE, HELD, BEGIN_TIME, DEPENDENCY, DEPENDENCY_NEVER = 0, 7, 8, 9, 10


def time_plus(t: int, delay: int) -> int:
    """absl::Time + absl::Seconds(delay): an infinite time stays infinite, and a sum
    beyond the int64 seconds range saturates to InfiniteFuture (delay >= 0)."""
    return t if t in (PAST, FUTURE) else min(t + delay, FUTURE)


class Deps:
    """DependenciesInJob: deps (dependee id -> (type, delay)), is_or, ready_time."""

    def __init__(self, is_or: bool = False, deps: dict | None = None):
        # SetDependency (CtldPublicDefs.cpp:1600-1611); a job without dependencies keeps
        # the defaults (is_or false, ready_time InfinitePast, CtldPublicDefs.h:415-417)
        self.is_or = bool(is_or)
        self.deps = dict(deps or {})
        self.ready = FUTURE if self.is_or else PAST

    def update(self, job_id, t: int) -> bool:
        """CtldPublicDefs.cpp:144-159; an id not in deps is logged and ignored (False)."""
        if job_id not in self.deps:
            return False
        _, delay = self.deps.pop(job_id)
        r = time_plus(t, delay)
        self.ready = min(self.ready, r) if self.is_or else max(self.ready, r)
        return True

    def is_met(self, now: int) -> bool:
        return (self.is_or or not self.deps) and self.ready <= now

    def is_failed(self) -> bool:
        return self.ready >= FUTURE and (not self.is_or or not self.deps)


class MissingDependency(Exception):
    """ERR_MISSING_DEPENDENCY (JobScheduler.cpp:4215-4248)."""


@dataclass
class Job:
    state: str = "pending"  # pending / running / ended
    held: bool = False
    begin: int = PAST       # begin_time default (CtldPublicDefs.h:779)
    deps: Deps = field(default_factory=Deps)
    dependents: dict = field(default_factory=lambda: {AFTER: [], AFTER_ANY: [], AFTER_OK: [], AFTER_NOT_OK: []})
    start_time: int = 0


class Daemon:
    """The daemon's job bookkeeping over a trajectory, as far as the gate reads it."""

    def __init__(self):
        self.jobs: dict = {}

    def _event(self, dependent, dependee, t):
        self.jobs[dependent].deps.update(dependee, t)

    def _trigger(self, job_id, dep_type, t):
        # JobInCtld::TriggerDependencyEvents
        for d in self.jobs[job_id].dependents[dep_type]:
            self._event(d, job_id, t)

    def running(self, job_id, start_time: int):
        """A job known to be running (recovered, or started outside this model)."""
        self.jobs[job_id] = Job(state="running", start_time=start_time)

    def submit(self, job_id, deps=(), is_or=False, held=False, begin=PAST, resolved=None):
        """deps: (dependee id, type, delay) triples. `resolved` (recovery): dependee id ->
        event time of dependees that ended before, taken from the DB (Init, :552-594)."""
        resolved = resolved or {}
        for dep, _, _ in deps:
            if dep not in resolved and (dep not in self.jobs or self.jobs[dep].state == "ended"):
                raise MissingDependency(dep)
        job = Job(held=held, begin=begin, deps=Deps(is_or, {d: (ty, dl) for d, ty, dl in deps}))
        self.jobs[job_id] = job
        for dep, ty, _ in deps:
            if dep in resolved:
                self._event(job_id, dep, resolved[dep])
            elif ty == AFTER and self.jobs[dep].state != "pending":  # AddDependent
                self._event(job_id, dep, self.jobs[dep].start_time)
            else:
                self.jobs[dep].dependents[ty].append(job_id)

    def set_held(self, job_id, held: bool):
        self.jobs[job_id].held = bool(held)

    def set_begin(self, job_id, begin: int):
        self.jobs[job_id].begin = int(begin)

    def start(self, job_id, t: int):
        j = self.jobs[job_id]
        j.state, j.start_time = "running", t
        self._trigger(job_id, AFTER, t)

    def cancel(self, job_id, t: int):
        """A pending job is cancelled."""
        self.jobs[job_id].state = "ended"
        self._trigger(job_id, AFTER, t)
        self._trigger(job_id, AFTER_ANY, t)
        self._trigger(job_id, AFTER_OK, FUTURE)
        self._trigger(job_id, AFTER_NOT_OK, FUTURE)

    def end(self, job_id, t: int, exit_code: int):
        """A running job ends at t (the time the daemon records)."""
        self.jobs[job_id].state = "ended"
        self._trigger(job_id, AFTER_ANY, t)
        self._trigger(job_id, AFTER_OK, t if exit_code == 0 else FUTURE)
        self._trigger(job_id, AFTER_NOT_OK, t if exit_code != 0 else FUTURE)

    def reason(self, job_id, now: int) -> int:
        """The filter of JobScheduler.cpp:1090-1113: NONE if the job enters NodeSelect."""
        j = self.jobs[job_id]
        if j.held:
            return HELD
        if j.begin > now:
            return BEGIN_TIME
        if not j.deps.is_met(now):
            return DEPENDENCY_NEVER if j.deps.is_failed() else DEPENDENCY
        return NONE
