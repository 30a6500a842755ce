/*
 * crane_ref_steps.h — C interface of oracle/_ref/libcrane_ref_steps.so: the
 * REFERENCE's own JobInCtld::SchedulePendingSteps, compiled from its unmodified
 * source text (oracle/ref_step_build.py, oracle/ref_step_shim/). TEST
 * INFRASTRUCTURE ONLY.
 */
#ifndef CRANE_REF_STEPS_H_
#define CRANE_REF_STEPS_H_

#include "../include/crane_sched.h"

#ifdef __cplusplus
extern "C" {
#endif

/* Same contract as crane_oracle_schedule_steps (oracle/crane_step_oracle.h), with the
 * reference's own walk: `visit` (optional, out, [node_off[n_jobs]]) receives per job
 * the positions of its nodes in the order step_res_avail_.EachNodeResMap() (a
 * std::unordered_map) walks them. `erased` (optional, [n steps]) marks steps whose
 * ids are still queued but that were removed (GetStep() == nullptr,
 * CtldPublicDefs.cpp:1883-1889); placed[j] is the reference's popped_count. */
int crane_ref_schedule_steps(const crane_cluster_t* dict, const crane_step_jobs_t* jobs, const crane_steps_t* steps,
                             const uint8_t* erased, crane_step_placements_t* out, uint32_t* visit,
                             double* elapsed_ms);

#ifdef __cplusplus
}
#endif
#endif
