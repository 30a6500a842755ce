// gate_kernels.cuh — sm_90a kernels of the gate of the resident pending table.
//
// The daemon leaves held jobs, jobs whose begin time is ahead and jobs whose
// dependencies are not met out of the pending vector before NodeSelect
// (JobScheduler.cpp:1090-1113). Here those rows stay resident and carry:
//   per row    held, begin, is_or, open (entries not yet resolved), ready (int64)
//   per entry  the dependent row, the dependee (a pending or a running row), type,
//              delay and a live flag
// which is DependenciesInJob (CtldPublicDefs.h:413-428) with `deps` kept as the live
// entries and their count. Two kernels:
//   k_gate      thread per row, once per run: the run's exclusion code of every row
//               (0, ERASED or a gate reason), passed where the run passes the
//               tombstones, so the priority bounds, the sort and the queue leave gated
//               rows out as they leave erased rows out.
//   k_dep_fire  thread per entry: the events of one call (depend, start, cancel, end).
//               DependenciesInJob::update (CtldPublicDefs.cpp:144-159) is a min or max
//               of ready_time and an erase of the entry; both commute, so applying them
//               with atomicMin/atomicMax and an atomic decrement of `open` gives the same
//               state in any thread order. The state is read only by the next k_gate.
#pragma once

#include "sched_kernels.cuh"

namespace crane {

constexpr long long kTimePast = INT64_MIN;   // absl::InfinitePast
constexpr long long kTimeFuture = INT64_MAX;  // absl::InfiniteFuture

enum : uint8_t { kDepPending = 0, kDepRunning = 1, kDepEvent = 2 };
enum : uint8_t { kAfter = 0, kAfterAny = 1, kAfterOk = 2, kAfterNotOk = 3 };
enum : uint32_t { kFireDepend = 0, kFireStart = 1, kFireCancel = 2, kFireEnd = 3 };

struct GateDev {
  uint32_t n;              // pending rows with gate state
  const uint8_t* dead;     // tombstones of the pending table, or null
  uint8_t* held;
  int64_t* begin;
  uint8_t* is_or;
  uint32_t* open;          // entries of the row not yet resolved
  long long* ready;        // ready_time
  uint32_t n_ent;
  uint32_t* dependent;     // [n_ent] pending row waiting on the entry
  uint32_t* dependee;      // pending or running row
  uint8_t* kind;           // kDepPending / kDepRunning
  uint8_t* type;
  uint8_t* live;
  uint64_t* delay;
};

// The events of one call. `rows` are the call's rows sorted ascending, `pos[k]` the
// place of rows[k] in the call's own list.
struct DepEvents {
  uint32_t mode;
  uint32_t n;
  const uint32_t* rows;
  const uint32_t* pos;
  long long t;                  // cancel time
  const int64_t* time;          // start: placement start per pending row; end: end time per call row
  const uint32_t* code;         // end: exit code per call row
  uint32_t base;                // start: running row of the call's first row
  const int64_t* run_start;     // depend: start time per running row
  const int64_t* event_time;    // depend: event time per new entry (from e0), or null
  uint32_t e0;                  // depend: first new entry
};

// absl::Time + absl::Seconds(delay): an infinite time stays infinite, and a finite sum
// past the int64 range saturates to InfiniteFuture as Abseil's does (0 <= delay < 2^62)
__device__ __forceinline__ long long time_plus(long long t, uint64_t delay) {
  if (t == kTimePast || t == kTimeFuture) return t;
  return t > kTimeFuture - (long long)delay ? kTimeFuture : t + (long long)delay;
}

// Rows [from, to) that got no gate call yet: not held, begin InfinitePast, no dependencies
__global__ void k_gate_init(GateDev g, uint32_t from, uint32_t to) {
  const uint32_t r = from + blockIdx.x * blockDim.x + threadIdx.x;
  if (r >= to) return;
  g.held[r] = 0;
  g.begin[r] = kTimePast;
  g.is_or[r] = 0;
  g.open[r] = 0;
  g.ready[r] = kTimePast;
}

// set_gate: held / begin of the listed rows (null = unchanged)
__global__ void k_gate_set(GateDev g, const uint32_t* rows, uint32_t n, const uint8_t* held, const int64_t* begin) {
  const uint32_t k = blockIdx.x * blockDim.x + threadIdx.x;
  if (k >= n) return;
  if (held) g.held[rows[k]] = held[k] ? 1 : 0;
  if (begin) g.begin[rows[k]] = begin[k];
}

// depend: JobInCtld::SetDependency (CtldPublicDefs.cpp:1600-1611) on the listed rows
__global__ void k_dep_rows(GateDev g, const uint32_t* rows, uint32_t n, const uint8_t* is_or, const uint32_t* off) {
  const uint32_t k = blockIdx.x * blockDim.x + threadIdx.x;
  if (k >= n) return;
  const uint32_t r = rows[k];
  g.is_or[r] = is_or[k] ? 1 : 0;
  g.ready[r] = is_or[k] ? kTimeFuture : kTimePast;
  g.open[r] = off[k + 1] - off[k];
}

// The exclusion code of every row for this run (the filter of JobScheduler.cpp:1090-1113)
__global__ void k_gate(GateDev g, int64_t now, uint8_t* code) {
  const uint32_t r = blockIdx.x * blockDim.x + threadIdx.x;
  if (r >= g.n) return;
  uint8_t c = CRANE_REASON_NONE;
  const bool or_ = g.is_or[r] != 0;
  const bool empty = g.open[r] == 0;
  const long long ready = g.ready[r];
  if (g.dead && g.dead[r]) c = CRANE_REASON_ERASED;
  else if (g.held[r]) c = CRANE_REASON_HELD;
  else if (g.begin[r] > now) c = CRANE_REASON_BEGIN_TIME;
  else if (!((or_ || empty) && ready <= now))  // !is_met(now)
    c = (ready >= kTimeFuture && (!or_ || empty)) ? CRANE_REASON_DEPENDENCY_NEVER : CRANE_REASON_DEPENDENCY;
  code[r] = c;
}

// position in the call's list of row `r`, or 0xffffffff
__device__ __forceinline__ uint32_t event_of(const DepEvents& ev, uint32_t r) {
  uint32_t lo = 0, hi = ev.n;
  while (lo < hi) {  // lower_bound
    const uint32_t mid = lo + (hi - lo) / 2;
    if (ev.rows[mid] < r) lo = mid + 1;
    else hi = mid;
  }
  return (lo < ev.n && ev.rows[lo] == r) ? ev.pos[lo] : 0xffffffffu;
}

// One thread per entry: the call's event for the entry's dependee, applied to the
// dependent (DependenciesInJob::update) and the entry retired; in `start`, the entries
// on a started row that wait for its end move to its running row.
__global__ void k_dep_fire(GateDev g, DepEvents ev) {
  const uint32_t e = (ev.mode == kFireDepend ? ev.e0 : 0) + blockIdx.x * blockDim.x + threadIdx.x;
  if (e >= g.n_ent || !g.live[e]) return;
  const uint8_t type = g.type[e], kind = g.kind[e];
  const uint32_t row = g.dependee[e];
  long long t;
  switch (ev.mode) {
    case kFireDepend:
      if (kind == kDepEvent) t = ev.event_time[e - ev.e0];
      else if (kind == kDepRunning && type == kAfter) t = ev.run_start[row];  // AddDependent, CtldPublicDefs.cpp:1620
      else return;
      break;
    case kFireStart: {
      if (kind != kDepPending) return;
      const uint32_t k = event_of(ev, row);
      if (k == 0xffffffffu) return;
      if (type != kAfter) {  // waits for the job's end: follows it to the running table
        g.kind[e] = kDepRunning;
        g.dependee[e] = ev.base + k;
        return;
      }
      t = ev.time[row];  // JobScheduler.cpp:1549
      break;
    }
    case kFireCancel: {
      if (kind != kDepPending || event_of(ev, row) == 0xffffffffu) return;
      t = (type == kAfter || type == kAfterAny) ? ev.t : kTimeFuture;  // JobScheduler.cpp:4067-4073
      break;
    }
    default: {  // kFireEnd, JobScheduler.cpp:4531-4538
      if (kind != kDepRunning || type == kAfter) return;
      const uint32_t k = event_of(ev, row);
      if (k == 0xffffffffu) return;
      const bool ok = ev.code[k] == 0;
      t = (type == kAfterAny || (type == kAfterOk) == ok) ? (long long)ev.time[k] : kTimeFuture;
      break;
    }
  }
  const uint32_t d = g.dependent[e];
  const long long r = time_plus(t, g.delay[e]);
  if (g.is_or[d]) atomicMin(&g.ready[d], r);
  else atomicMax(&g.ready[d], r);
  atomicAdd(&g.open[d], 0xffffffffu);  // (-1)
  g.live[e] = 0;
}

}  // namespace crane
