/*
 * crane_step_oracle.h — C interface of the CPU oracle of the step scheduler
 * (TEST INFRASTRUCTURE ONLY; see crane_oracle.h for who may load it).
 */
#ifndef CRANE_STEP_ORACLE_H_
#define CRANE_STEP_ORACLE_H_

#include "../include/crane_sched.h"

#ifdef __cplusplus
extern "C" {
#endif

/* Restates JobInCtld::SchedulePendingSteps (CtldPublicDefs.cpp:1877-1998) for every
 * job of `jobs`: writes the crane_step_placements_t the GPU path writes and updates
 * jobs->avail in place. placed[j] is the reference's popped_count. `visit` (optional,
 * [node_off[n_jobs]]) gives, per job, the order in which its node positions
 * (0 .. nodes-1) are walked; NULL = node-index order. *elapsed_ms (optional) brackets
 * the scheduling loop alone, single thread. */
int crane_oracle_schedule_steps(const crane_cluster_t* dict, const crane_step_jobs_t* jobs,
                                const crane_steps_t* steps, crane_step_placements_t* out,
                                const uint32_t* visit, double* elapsed_ms);

#ifdef __cplusplus
}
#endif
#endif
