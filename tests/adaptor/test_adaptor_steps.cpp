// test_adaptor_steps.cpp — drives SchedulerAlgo::SchedulePendingSteps with reference-style
// objects (hostnames, queued step ids, removed steps) and checks hand-derived answers:
// popped_count counts removed ids in front of the first blocking step, never behind it.
// Linked against the product library (GPU) or the kernel-emulation library (CPU tests).
#include <cstdio>
#include <string>

#include "../../cranesched_b200/adaptor/crane_adaptor.h"

using namespace crane_b200;

static std::string NodeName(int i) { char b[32]; snprintf(b, sizeof b, "cn%04d", i); return b; }
static int bad = 0;
#define EXPECT(c) do { if (!(c)) { ++bad; printf("FAILED: %s (line %d)\n", #c, __LINE__); } } while (0)

static ResourceInNodeV3 Cores(int n) {
  ResourceInNodeV3 r;
  for (int c = 0; c < n; ++c) r.core_ids.insert(c);
  r.cpu_count_raw = n * 256;
  r.memory_bytes = r.memory_sw_bytes = 8ull << 30;
  return r;
}

int main() {
  std::map<CranedId, CranedMeta> craneds;
  std::map<PartitionId, std::set<CranedId>> parts;
  for (int i = 0; i < 4; ++i) {
    craneds[NodeName(i)].res_total = Cores(8);
    parts["p"].insert(NodeName(i));
  }
  SchedulerAlgo algo(PriorityConfig{}, 1000, 0);
  algo.SetCluster(craneds, parts);

  auto step = [](uint32_t id, uint32_t nn, uint32_t nt, uint32_t tmax, int64_t cpus) {
    CommonStepInCtld s;
    s.step_id = id;
    s.node_num = nn;
    s.ntasks = nt;
    s.ntasks_per_node_max = tmax;
    s.req_task_res_view.cpu_count_raw = cpus * 256;
    return s;
  };
  // job A on cn0001, cn0002 (4 cores each): queue 10 (removed), 1 fits, 11 (removed),
  // 2 blocks (6 cores per task), 12 (removed), 3 would fit
  CommonStepInCtld a1 = step(1, 2, 3, 2, 1), a2 = step(2, 1, 1, 1, 6), a3 = step(3, 1, 1, 1, 1);
  JobStepState A;
  A.step_res_avail[NodeName(2)] = Cores(4);
  A.step_res_avail[NodeName(1)] = Cores(4);
  A.pending_step_ids = {10, 1, 11, 2, 12, 3};
  A.steps = {{1, &a1}, {2, &a2}, {3, &a3}};
  // job B on cn0003: queue 20 (removed), 4 fits, 21 (removed): everything pops
  CommonStepInCtld b4 = step(4, 1, 2, 2, 2);
  b4.excluded_nodes = {"not-a-node"};
  JobStepState B;
  B.step_res_avail[NodeName(3)] = Cores(8);
  B.pending_step_ids = {20, 4, 21};
  B.steps = {{4, &b4}};
  // job C: only removed ids
  JobStepState C;
  C.step_res_avail[NodeName(0)] = Cores(2);
  C.pending_step_ids = {30, 31};

  std::vector<std::vector<CommonStepInCtld*>> scheduled;
  const std::vector<uint32_t> popped = algo.SchedulePendingSteps(1700000000, {&A, &B, &C}, &scheduled);
  EXPECT(popped.size() == 3);
  EXPECT(popped[0] == 3);  // 10, 1, 11; step 2 blocks, 12 and 3 stay queued
  EXPECT((A.pending_step_ids == std::deque<uint32_t>{2, 12, 3}));
  EXPECT(popped[1] == 3 && B.pending_step_ids.empty());
  EXPECT(popped[2] == 2 && C.pending_step_ids.empty());
  EXPECT(scheduled[0].size() == 1 && scheduled[0][0] == &a1 && scheduled[1].size() == 1 && scheduled[2].empty());
  // step 1: two nodes, 3 tasks; both nodes hold 2 tasks (ntasks_per_node_max), tie -> walk order:
  // cn0001 first (2 tasks: ids 0, 1), then cn0002 (1 task: id 2)
  EXPECT((a1.craned_ids == std::vector<CranedId>{NodeName(1), NodeName(2)}));
  EXPECT((a1.craned_task_map[NodeName(1)] == std::set<uint32_t>{0, 1}));
  EXPECT((a1.craned_task_map[NodeName(2)] == std::set<uint32_t>{2}));
  EXPECT(a1.task_res_map.size() == 3 && a1.task_res_map[2].core_ids == std::set<uint32_t>{0});
  EXPECT(a1.allocated_res[NodeName(1)].cpu_count_raw == 2 * 256 && a1.start_time == 1700000000);
  EXPECT(A.step_res_avail[NodeName(1)].cpu_count_raw == 2 * 256);
  EXPECT((A.step_res_avail[NodeName(2)].core_ids == std::set<uint32_t>{1, 2, 3}));
  EXPECT(a2.craned_ids.empty() && a3.craned_ids.empty());
  EXPECT((b4.craned_task_map[NodeName(3)] == std::set<uint32_t>{0, 1}));
  EXPECT((B.step_res_avail[NodeName(3)].core_ids == std::set<uint32_t>{4, 5, 6, 7}));
  printf("adaptor steps: %d mismatches\n", bad);
  return bad ? 1 : 0;
}
