// step_oracle.cpp — CPU oracle of the step scheduler of running jobs (TEST
// INFRASTRUCTURE ONLY, like crane_oracle.cpp, whose containers it reuses: that file is
// compiled into this translation unit unchanged).
//
// Restates JobInCtld::SchedulePendingSteps (src/CraneCtld/CtldPublicDefs.cpp:1877-1998)
// with the reference's containers: std::set core ids and slot sets (ResInNode),
// std::priority_queue<NodeInfo> with NodeInfo::operator< = "has more tasks", a
// ResourceV3-like map per step for step_alloc_res, craned_task_map as
// map<node, set<task id>> and task_res_map as map<task id, ResInNode>.
//
// Deviation D8: the reference walks step_res_avail_.EachNodeResMap(), an unordered_map,
// so the candidate order is libstdc++ hash order. Here the walk follows `visit` (a
// per-job permutation of the job's node positions), and NULL means node-index order,
// which is the order the CUDA path uses.
#include "crane_oracle.cpp"

#include "crane_step_oracle.h"

#include <deque>

namespace {

struct StepRow {
  uint32_t node_num, ntasks, ntpn_min, ntpn_max;
  ResView req_node, req_task;
  std::unordered_set<uint32_t> included, excluded;  // node indices (0xFFFFFFFF = unknown host)
};

struct StepResult {
  bool scheduled{false};
  std::map<uint32_t, ResInNode> alloc;               // step_alloc_res, node-index order (D3)
  std::map<uint32_t, std::set<uint32_t>> task_map;   // craned_task_map
  std::map<uint32_t, ResInNode> task_res;            // task_res_map
  std::map<uint32_t, uint32_t> task_node;
};

struct JobSteps {
  std::vector<uint32_t> nodes;                     // job-local position -> node index
  std::vector<ResInNode> avail;                    // step_res_avail_, by position
  std::vector<uint32_t> walk;                      // EachNodeResMap() order, as positions
  std::deque<uint32_t> pending;                    // pending_step_ids_ (step rows)
};

// JobInCtld::SchedulePendingSteps for one job; returns popped_count
uint32_t SchedulePending(JobSteps& job, const std::vector<StepRow>& steps, std::vector<StepResult>& res) {
  uint32_t popped_count = 0;
  while (!job.pending.empty()) {
    const uint32_t sid = job.pending.front();
    const StepRow& step = steps[sid];
    struct NodeInfo {
      uint32_t ntasks_on_node;
      uint32_t pos;
      bool operator<(const NodeInfo& other) const { return ntasks_on_node > other.ntasks_on_node; }
    };
    std::priority_queue<NodeInfo> candidates;
    uint32_t sum_ntasks = 0;
    for (uint32_t pos : job.walk) {
      const uint32_t node = job.nodes[pos];
      if (step.excluded.contains(node)) continue;
      if (!step.included.empty() && !step.included.contains(node)) continue;
      ResInNode feasible_res;
      if (!step.req_node.Feasible(job.avail[pos], &feasible_res)) continue;
      ResInNode res_avail = job.avail[pos];
      res_avail.Sub(feasible_res);
      uint32_t ntasks_on_node = 0;
      while (ntasks_on_node < step.ntpn_max && step.req_task.Feasible(res_avail, &feasible_res)) {
        ++ntasks_on_node;
        res_avail.Sub(feasible_res);
      }
      if (ntasks_on_node < step.ntpn_min) continue;
      candidates.push(NodeInfo{ntasks_on_node, pos});
      sum_ntasks += ntasks_on_node;
      if (candidates.size() > step.node_num) {
        sum_ntasks -= candidates.top().ntasks_on_node;
        candidates.pop();
      }
      if (candidates.size() == step.node_num && sum_ntasks >= step.ntasks) break;
    }
    if (candidates.size() < step.node_num || sum_ntasks < step.ntasks) break;
    StepResult& r = res[sid];
    uint32_t rest_ntasks = step.ntasks - step.node_num;
    uint32_t cur_task_id = 0;
    while (!candidates.empty()) {
      const NodeInfo info = candidates.top();
      const uint32_t node = job.nodes[info.pos];
      ResInNode& res_avail = job.avail[info.pos];
      ResInNode feasible_res;
      step.req_node.Feasible(res_avail, &feasible_res);
      res_avail.Sub(feasible_res);
      r.alloc[node].Add(feasible_res);
      const uint32_t ntasks_on_node = std::min(rest_ntasks, info.ntasks_on_node - 1) + 1;
      for (uint32_t i = 0; i < ntasks_on_node; ++i) {
        step.req_task.Feasible(res_avail, &feasible_res);
        res_avail.Sub(feasible_res);
        r.task_map[node].insert(cur_task_id);
        r.task_res[cur_task_id] = feasible_res;
        r.task_node[cur_task_id] = node;
        r.alloc[node].Add(feasible_res);
        ++cur_task_id;
      }
      rest_ntasks -= ntasks_on_node - 1;
      candidates.pop();
    }
    r.scheduled = true;
    job.pending.pop_front();
    ++popped_count;
  }
  return popped_count;
}

}  // namespace

extern "C" int crane_oracle_schedule_steps(const crane_cluster_t* cl, const crane_step_jobs_t* jb,
                                           const crane_steps_t* st, crane_step_placements_t* out,
                                           const uint32_t* visit, double* elapsed_ms) {
  if (!cl || !jb || !st || !out) return CRANE_EINVAL;
  Dict d(cl);
  const uint32_t J = jb->n_jobs, S = st->n;
  if (jb->step_off[J] != S) return CRANE_EINVAL;
  std::vector<StepRow> steps(S);
  for (uint32_t s = 0; s < S; ++s) {
    StepRow& r = steps[s];
    r.node_num = st->node_num[s];
    r.ntasks = st->ntasks[s];
    r.ntpn_min = st->ntasks_per_node_min[s];
    r.ntpn_max = st->ntasks_per_node_max[s];
    if (r.node_num == 0 || r.ntasks < r.node_num || r.ntpn_min > r.ntpn_max) return CRANE_EINVAL;
    r.req_node = ViewFromAbi(d, st->req_node[s]);
    r.req_task = ViewFromAbi(d, st->req_task[s]);
    if (st->incl_off)
      for (uint32_t k = st->incl_off[s]; k < st->incl_off[s + 1]; ++k) r.included.insert(st->incl_nodes[k]);
    if (st->excl_off)
      for (uint32_t k = st->excl_off[s]; k < st->excl_off[s + 1]; ++k) r.excluded.insert(st->excl_nodes[k]);
  }
  std::vector<JobSteps> jobs(J);
  for (uint32_t j = 0; j < J; ++j) {
    JobSteps& job = jobs[j];
    const uint32_t k0 = jb->node_off[j], k1 = jb->node_off[j + 1];
    for (uint32_t k = k0; k < k1; ++k) {
      job.nodes.push_back(jb->node[k]);
      job.avail.push_back(FromAbi(d, jb->avail[k]));
      job.walk.push_back(visit ? visit[k] : k - k0);
    }
    for (uint32_t p : job.walk)
      if (p >= k1 - k0) return CRANE_EINVAL;
    for (uint32_t s = jb->step_off[j]; s < jb->step_off[j + 1]; ++s) job.pending.push_back(s);
  }
  std::vector<StepResult> res(S);
  std::vector<uint32_t> popped(J);
  const auto t0 = std::chrono::steady_clock::now();
  for (uint32_t j = 0; j < J; ++j) popped[j] = SchedulePending(jobs[j], steps, res);
  const auto t1 = std::chrono::steady_clock::now();
  if (elapsed_ms) *elapsed_ms = std::chrono::duration<double, std::milli>(t1 - t0).count();

  out->node_off[0] = 0;
  out->task_off[0] = 0;
  for (uint32_t s = 0; s < S; ++s) {
    out->node_off[s + 1] = out->node_off[s] + steps[s].node_num;
    out->task_off[s + 1] = out->task_off[s] + steps[s].ntasks;
  }
  for (uint32_t j = 0; j < J; ++j) out->placed[j] = popped[j];
  for (uint32_t s = 0; s < S; ++s) {
    const StepResult& r = res[s];
    out->scheduled[s] = r.scheduled ? 1 : 0;
    uint32_t i = out->node_off[s];
    for (uint32_t x = i; x < out->node_off[s + 1]; ++x) {
      out->alloc_node[x] = 0;
      out->alloc_ntasks[x] = 0;
      memset(&out->alloc_res[x], 0, sizeof(crane_res_in_node_t));
    }
    for (uint32_t x = out->task_off[s]; x < out->task_off[s + 1]; ++x) {
      out->task_node[x] = 0;
      memset(&out->task_res[x], 0, sizeof(crane_res_in_node_t));
    }
    if (!r.scheduled) continue;
    for (const auto& [node, a] : r.alloc) {
      out->alloc_node[i] = node;
      out->alloc_ntasks[i] = (uint32_t)r.task_map.at(node).size();
      ToAbi(d, a, &out->alloc_res[i]);
      ++i;
    }
    for (const auto& [t, a] : r.task_res) {
      out->task_node[out->task_off[s] + t] = r.task_node.at(t);
      ToAbi(d, a, &out->task_res[out->task_off[s] + t]);
    }
  }
  for (uint32_t j = 0; j < J; ++j)
    for (uint32_t k = jb->node_off[j]; k < jb->node_off[j + 1]; ++k)
      ToAbi(d, jobs[j].avail[k - jb->node_off[j]], &jb->avail[k]);
  return CRANE_OK;
}
