// step_shim.h — the members of JobInCtld / CommonStepInCtld that
// JobInCtld::SchedulePendingSteps (CtldPublicDefs.cpp:1877-1998) touches, and stubs for
// what it calls outside them. TEST INFRASTRUCTURE ONLY (oracle/ rules). Included
// after the reference's resource algebra (ph_h.inc / ph_cpp.inc) and before the
// sliced function text, inside namespace Ctld.
#pragma once

#include <expected>
#include <optional>
#include <queue>

#if !defined(__cpp_lib_ranges_to_container)
// std::ranges::to<std::vector> (C++23) for standard libraries that do not have it yet
namespace std::ranges {
template <template <class...> class C>
struct shim_to_t {};
template <template <class...> class C>
constexpr shim_to_t<C> to() { return {}; }
template <class R, template <class...> class C>
auto operator|(R&& r, shim_to_t<C>) {
  C<std::ranges::range_value_t<R>> c;
  for (auto&& x : r) c.push_back(x);
  return c;
}
}  // namespace std::ranges
#endif

namespace absl {
inline Time g_shim_now{};  // absl::Now(): the harness sets it
inline Time Now() { return g_shim_now; }
}  // namespace absl

namespace crane::grpc {
enum JobStatus { Pending = 0, Running = 1, Configuring = 9 };
}  // namespace crane::grpc

namespace util {
// String.h:101: only its result's existence matters to the step scheduler
template <class T>
std::string HostNameListToStr(T const& host_list) {
  std::string s;
  for (const auto& h : host_list) s += (s.empty() ? "" : ",") + std::string(h);
  return s;
}
}  // namespace util

namespace Ctld {

// CtldPublicDefs.h:263-301 (InteractiveMeta::StepResAllocArgs, the callback type)
struct StepInteractiveMeta {
  struct StepResAllocArgs {
    job_id_t job_id;
    step_id_t step_id;
    struct ResAllocInfo {
      std::string allocated_craned_regex;
      std::vector<CranedId> allocated_craned_ids;
      std::unordered_map<CranedId, std::set<task_id_t>> craned_task_map;
      uint32_t ntasks_total;
    };
    std::expected<ResAllocInfo, std::string> res_allocate_expt;
  };
  std::function<void(StepResAllocArgs const&)> cb_step_res_allocated;
};

// CommonStepInCtld (CtldPublicDefs.h:481-720): the fields SchedulePendingSteps reads and writes
struct CommonStepInCtld {
  job_id_t job_id{0};
  uint32_t node_num{0};
  uint32_t ntasks_per_node_min{1};
  uint32_t ntasks_per_node_max{0};
  uint32_t ntasks{0};
  ResourceView req_node_res_view;
  ResourceView req_task_res_view;
  std::unordered_set<std::string> included_nodes;
  std::unordered_set<std::string> excluded_nodes;
  std::optional<StepInteractiveMeta> ia_meta;
  std::string allocated_craneds_regex;
  std::unordered_map<task_id_t, ResourceInNodeV3> task_res_map;
  std::unordered_map<CranedId, std::set<task_id_t>> craned_task_map;
  absl::Time deadline_time{};

  step_id_t m_step_id_{0};
  ResourceV3 m_allocated_res_;
  std::vector<CranedId> m_craned_ids_;
  absl::Time m_start_time_{};
  crane::grpc::JobStatus m_status_{crane::grpc::Pending};

  step_id_t StepId() const { return m_step_id_; }
  void SetAllocatedRes(const ResourceV3& res) { m_allocated_res_ = res; }
  const ResourceV3& AllocatedRes() const { return m_allocated_res_; }
  void SetCranedIds(const std::vector<CranedId>& craned_list) { m_craned_ids_ = craned_list; }
  const std::vector<CranedId>& CranedIds() const { return m_craned_ids_; }
  void SetExecutionNodes(const std::unordered_set<CranedId>&) {}
  void SetConfiguringNodes(const std::unordered_set<CranedId>&) {}
  void SetStartTime(absl::Time t) { m_start_time_ = t; }
  void SetStatus(crane::grpc::JobStatus s) { m_status_ = s; }
};

// JobInCtld (CtldPublicDefs.h:780-1016): the step queue, step_res_avail_, the steps map
struct JobInCtld {
  absl::Time deadline_time{};
  std::queue<step_id_t> pending_step_ids_;
  ResourceV3 step_res_avail_;
  std::unordered_map<step_id_t, CommonStepInCtld*> m_steps_;  // (the reference owns them through unique_ptr)

  CommonStepInCtld* GetStep(step_id_t step) const {  // :991-1000 for a non-primary step
    auto it = m_steps_.find(step);
    return it == m_steps_.end() ? nullptr : it->second;
  }
  uint32_t SchedulePendingSteps(std::vector<CommonStepInCtld*>* scheduled_steps);
};

}  // namespace Ctld
