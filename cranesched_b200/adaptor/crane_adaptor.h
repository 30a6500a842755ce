// crane_adaptor.h — NodeSelect-shaped C++ adaptor over the C-ABI.
//
// Host side of the drop-in boundary (SURVEY.md §8b): a class with the call
// shape of SchedulerAlgo::NodeSelect (reference: src/CraneCtld/JobScheduler.h:
// 227-257, call site JobScheduler.cpp:1141) that flattens the reference's job
// and node objects into the POD tables of include/crane_sched.h, calls
// crane_sched_node_select, and writes the results back into the pending-job
// objects in place (the fields listed at JobScheduler.h:116-132).
//
// The reference's own types need abseil/protobuf, which this image does not
// have, so the structs below MIRROR them with the same member names and
// meaning; times are int64 unix seconds instead of absl::Time/Duration and
// cpu_t is its raw fixed-point value (fpm::fixed<int64_t,__int128,8>,
// PublicHeader.h:44: cpus * 256). In the daemon the mirror types are replaced
// by the real ones; the flattening code is identical (see INTEGRATION.md).
#pragma once

#include <cstdint>
#include <deque>
#include <list>
#include <map>
#include <memory>
#include <set>
#include <string>
#include <unordered_map>
#include <unordered_set>
#include <vector>

#include "../../include/crane_sched.h"

namespace crane_b200 {

using CranedId = std::string;
using SlotId = std::string;  // device path, PublicHeader.h:408-410
using PartitionId = std::string;

// GresCount (PublicHeader.h:490-508)
struct GresCount {
  uint64_t total{0};
  std::unordered_map<std::string, uint64_t> specified;
};
using GresMap = std::unordered_map<std::string, GresCount>;

// ResourceView (PublicHeader.h:671-737)
struct ResourceView {
  int64_t cpu_count_raw{0};
  uint64_t memory_bytes{0};
  uint64_t memory_sw_bytes{0};
  GresMap gres_map;
};

// ResourceInNodeV3 (PublicHeader.h:562-615) with DedicatedResourceInNode
// (PublicHeader.h:444-479) inlined as name -> type -> slot set
struct ResourceInNodeV3 {
  std::set<uint32_t> core_ids;
  int64_t cpu_count_raw{0};
  uint64_t memory_bytes{0};
  uint64_t memory_sw_bytes{0};
  std::map<std::string, std::map<std::string, std::set<SlotId>>> gres;
};
using ResourceV3 = std::unordered_map<CranedId, ResourceInNodeV3>;  // PublicHeader.h:625-664

// RnJobInScheduler (JobScheduler.h:56-89)
struct RnJobInScheduler {
  uint32_t job_id{0};
  int64_t time_limit{0};
  PartitionId partition_id;
  int64_t submit_time{0};
  uint32_t partition_priority{0};
  uint32_t qos_priority{0};
  std::string account;
  std::string qos;
  uint32_t node_num{0};
  int64_t start_time{0};
  int64_t end_time{0};
  ResourceV3 allocated_res;
  ResourceView allocated_res_view;
};

// PdJobInScheduler (JobScheduler.h:91-164)
struct PdJobInScheduler {
  uint32_t job_id{0};
  int64_t time_limit{0};
  PartitionId partition_id;
  ResourceView req_node_res_view;
  ResourceView req_task_res_view;
  ResourceView req_total_res_view;
  uint32_t node_num{1};
  uint32_t ntasks_per_node_min{1};
  uint32_t ntasks_per_node_max{1};
  uint32_t ntasks{1};
  bool exclusive{false};
  std::unordered_set<std::string> included_nodes;
  std::unordered_set<std::string> excluded_nodes;
  int64_t submit_time{0};
  uint32_t partition_priority{0};
  uint32_t qos_priority{0};
  std::string account;
  double priority{0.0};  // in: mandated_priority (0 = compute); out: priority
  // ---- written by NodeSelect -------------------------------------------
  std::unordered_map<CranedId, uint32_t> craned_id_to_task_num;
  int64_t start_time{0};
  int64_t end_time{0};
  ResourceV3 allocated_res;
  std::vector<CranedId> craned_ids;
  std::string reason;
  std::string qos;
  std::string username;
  std::list<std::string> account_chain;
  bool is_scheduled() const { return reason.empty(); }  // JobScheduler.h:137
};

// what NodeSelect reads from g_meta_container (CranedMeta, NodeDefs.h:57-79;
// PartitionMeta, NodeDefs.h:118-121)
struct CranedMeta {
  bool alive{true};
  bool drain{false};
  ResourceInNodeV3 res_total;
};

// Config::Priority (CtldPublicDefs.h:151-163) + ScheduledBatchSize
struct PriorityConfig {
  enum TypeEnum { Basic, MultiFactor } Type{MultiFactor};
  bool FavorSmall{true};
  uint64_t MaxAge{7 * 24 * 3600};
  uint32_t WeightAge{1000}, WeightFairShare{0}, WeightJobSize{0}, WeightPartition{0}, WeightQoS{0};
};

// Qos (Account/AccountDefs.h:27-50): the limits CheckQosResource_ reads
// (AccountMetaContainer.cpp:382-491). A gres name / type absent from a max_tres
// map is unlimited, as upstream.
struct Qos {
  bool deleted{false};
  uint32_t max_jobs_per_user{UINT32_MAX};
  uint32_t max_jobs_per_account{UINT32_MAX};
  uint32_t max_jobs{UINT32_MAX};
  int64_t max_cpus_per_user_raw{INT64_MAX};
  int64_t max_wall{0};  // seconds; 0 = unlimited
  ResourceView max_tres{INT64_MAX, UINT64_MAX, UINT64_MAX, {}};
  ResourceView max_tres_per_user{INT64_MAX, UINT64_MAX, UINT64_MAX, {}};
  ResourceView max_tres_per_account{INT64_MAX, UINT64_MAX, UINT64_MAX, {}};
};

// MetaResource (Accounting/AccountMetaContainer.h:30-47) without the submit counter
// (CheckAndMallocQosResource does not touch it)
struct MetaResource {
  ResourceView resource;
  uint32_t jobs_count{0};
  int64_t wall_time{0};
};

// the usage maps of AccountMetaContainer (AccountMetaContainer.h:52-75):
// user -> qos, account -> qos, qos. An entry that is missing reads as zero.
struct QosUsage {
  std::map<std::string, std::map<std::string, MetaResource>> user;
  std::map<std::string, std::map<std::string, MetaResource>> account;
  std::map<std::string, MetaResource> qos;
};

// CommonStepInCtld (CtldPublicDefs.h:481-720): the fields JobInCtld::SchedulePendingSteps
// reads (request) and writes (placement)
struct CommonStepInCtld {
  uint32_t step_id{0};
  uint32_t node_num{1};
  uint32_t ntasks{1};
  uint32_t ntasks_per_node_min{1};
  uint32_t ntasks_per_node_max{1};
  ResourceView req_node_res_view;
  ResourceView req_task_res_view;
  std::unordered_set<std::string> included_nodes;
  std::unordered_set<std::string> excluded_nodes;
  // ---- written when the step is scheduled ---------------------------------
  std::unordered_map<CranedId, std::set<uint32_t>> craned_task_map;
  std::unordered_map<uint32_t, ResourceInNodeV3> task_res_map;
  ResourceV3 allocated_res;
  std::vector<CranedId> craned_ids;  // node-index ascending
  int64_t start_time{0};
};

// The step state of a running JobInCtld (CtldPublicDefs.h:823-824, 991-1000):
// pending_step_ids_ (a std::queue upstream), step_res_avail_, and GetStep() — an id
// without an entry in `steps` is a step that was removed while queued.
struct JobStepState {
  std::deque<uint32_t> pending_step_ids;
  ResourceV3 step_res_avail;
  std::unordered_map<uint32_t, CommonStepInCtld*> steps;
};

class SchedulerAlgo {
 public:
  SchedulerAlgo(const PriorityConfig& prio, uint32_t scheduled_batch_size, int device = 0);
  ~SchedulerAlgo();
  SchedulerAlgo(const SchedulerAlgo&) = delete;
  SchedulerAlgo& operator=(const SchedulerAlgo&) = delete;

  // Replaces the snapshot NodeSelect takes from g_meta_container each tick
  // (JobScheduler.cpp:5603-5651). Node index = rank of the hostname in sorted
  // order (the documented tie-break between equal-cost nodes).
  void SetCluster(const std::map<CranedId, CranedMeta>& craneds,
                  const std::map<PartitionId, std::set<CranedId>>& partitions);

  // Same call shape and in-place semantics as SchedulerAlgo::NodeSelect
  // (JobScheduler.h:254-257). Per-job failure is a pending reason; a malformed
  // table or a device failure throws std::runtime_error (the reference aborts
  // on invariant violations, Logger.h:114-123).
  void NodeSelect(int64_t now, const std::vector<std::unique_ptr<RnJobInScheduler>>& running_jobs,
                  const std::vector<std::unique_ptr<PdJobInScheduler>>& pending_jobs);

  // Replaces the AccountMetaContainer::CheckAndMallocQosResource call the commit
  // loop makes for every job NodeSelect starts now (JobScheduler.cpp:1262;
  // AccountMetaContainer.cpp:164-191), for the whole vector at once and in its
  // order: a job over a limit keeps pending with the reference's reason string
  // ("QosCpuResourceLimit", "QosJobsResourceLimit", "QosWallTimeLimit",
  // "QosMemResourceLimit", "QosGresResourceLimit", "InvalidQOS"), every other
  // started job is added to `usage` at its user, account-chain and qos levels.
  // Call right after NodeSelect with the same pending_jobs.
  void CheckAndMallocQosResource(const std::map<std::string, Qos>& qos_table, QosUsage& usage,
                                 const std::vector<std::unique_ptr<PdJobInScheduler>>& pending_jobs);

  // Replaces the JobInCtld::SchedulePendingSteps calls of StepScheduleThread_
  // (JobScheduler.cpp:1646-1659; CtldPublicDefs.cpp:1877-1998) for all jobs at once.
  // Per job, returns the reference's popped_count: the ids taken off the front of
  // pending_step_ids — scheduled steps and removed ones — up to the first step that
  // does not fit (removed ids behind it stay queued). Scheduled steps get
  // craned_task_map, task_res_map, allocated_res, craned_ids and start_time = now, are
  // appended to (*scheduled_steps)[j], and step_res_avail is updated. Status, the
  // ia_meta callback, the DB and the RPC stay with the daemon. Call after SetCluster.
  std::vector<uint32_t> SchedulePendingSteps(int64_t now, const std::vector<JobStepState*>& jobs,
                                             std::vector<std::vector<CommonStepInCtld*>>* scheduled_steps);

 private:
  struct Impl;
  std::unique_ptr<Impl> m_;
};

}  // namespace crane_b200
