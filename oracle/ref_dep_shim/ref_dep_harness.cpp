// ref_dep_harness.cpp — drives the REFERENCE's own DependenciesInJob.
//
// TEST INFRASTRUCTURE ONLY (oracle/ rules). deps_h.inc and deps_cpp.inc are the
// reference's unmodified text, sliced out of /root/reference at build time by
// oracle/ref_dep_build.py (never committed):
//   deps_h.inc    CtldPublicDefs.h   struct DependenciesInJob (:413-428)
//   deps_cpp.inc  CtldPublicDefs.cpp DependenciesInJob::update (:144-159)
#include "dep_shim.h"

namespace Ctld {
#include "deps_h.inc"
#include "deps_cpp.inc"
}  // namespace Ctld

extern "C" {

// One job's dependencies: SetDependency (CtldPublicDefs.cpp:1600-1611) with the given
// entries, then update(ev_id[k], ev_time[k]) in order; answers is_met(nows[k]),
// is_failed(), ready_time, the entries left and the number of ignored (unknown) events.
int crane_ref_dep_run(uint8_t is_or, uint32_t n_deps, const uint32_t* dep_id, const uint8_t* dep_type,
                      const uint64_t* dep_delay, uint32_t n_ev, const uint32_t* ev_id, const int64_t* ev_time,
                      uint32_t n_now, const int64_t* nows, uint8_t* met, uint8_t* failed, int64_t* ready,
                      uint32_t* left, uint32_t* ignored) {
  Ctld::DependenciesInJob d;
  d.is_or = is_or != 0;
  d.ready_time = is_or ? absl::InfiniteFuture() : absl::InfinitePast();
  for (uint32_t k = 0; k < n_deps; ++k)
    d.deps[dep_id[k]] = {static_cast<crane::grpc::DependencyType>(dep_type[k]), dep_delay[k]};
  g_crane_error_calls = 0;
  for (uint32_t k = 0; k < n_ev; ++k) d.update(ev_id[k], absl::Time::FromUnix(ev_time[k]));
  for (uint32_t k = 0; k < n_now; ++k) met[k] = d.is_met(absl::Time::FromUnix(nows[k])) ? 1 : 0;
  *failed = d.is_failed() ? 1 : 0;
  *ready = d.ready_time.unix_seconds();
  *left = (uint32_t)d.deps.size();
  *ignored = g_crane_error_calls;
  return 0;
}

}  // extern "C"
