// ref_steps_harness.cpp — drives the REFERENCE's own JobInCtld::SchedulePendingSteps.
//
// TEST INFRASTRUCTURE ONLY (oracle/ rules). Everything between the `#include "*.inc"`
// lines is the reference's unmodified text, sliced out of /root/reference at build time
// by oracle/ref_step_build.py (never committed):
//   ph_h.inc / ph_cpp.inc   PublicHeader.h / .cpp: the resource algebra (oracle/ref_build.py)
//   steps_cpp.inc           CtldPublicDefs.cpp JobInCtld::SchedulePendingSteps (:1877-1998)
// between shim declarations of JobInCtld / CommonStepInCtld holding exactly the members
// it touches (step_shim.h). step_res_avail_ is a real std::unordered_map, so the walk is
// libstdc++ hash order; crane_ref_schedule_steps reports that order per job.
#include "ctld_shim.h"

#include "ph_h.inc"
#include "ph_cpp.inc"

#include "step_shim.h"

namespace Ctld {
#include "steps_cpp.inc"
}  // namespace Ctld

#include <chrono>
#include <cstring>

#include "include/crane_sched.h"
#include "oracle/crane_ref_steps.h"

namespace {

std::string NodeName(uint32_t i) { char b[24]; snprintf(b, sizeof b, "cn%08u", i); return b; }

struct Dict {
  uint32_t n_entries{0};
  uint8_t entry_name[CRANE_GRES_ENTRIES]{};
  std::string name_str[CRANE_GRES_NAMES], type_str[CRANE_GRES_ENTRIES], slot_str[CRANE_MAX_SLOTS];
  explicit Dict(const crane_cluster_t* c) {
    n_entries = std::min<uint32_t>(c->n_gres_entries, CRANE_GRES_ENTRIES);
    for (uint32_t e = 0; e < n_entries; ++e) entry_name[e] = c->gres_entry_name[e];
    char b[32];
    for (int g = 0; g < CRANE_GRES_NAMES; ++g) { snprintf(b, sizeof b, "gres%02d", g); name_str[g] = b; }
    for (int e = 0; e < CRANE_GRES_ENTRIES; ++e) { snprintf(b, sizeof b, "type%02d", e); type_str[e] = b; }
    for (int s = 0; s < CRANE_MAX_SLOTS; ++s) { snprintf(b, sizeof b, "/dev/slot%02d", s); slot_str[s] = b; }
  }
};

ResourceInNodeV3 FromAbi(const Dict& d, const crane_res_in_node_t& r) {
  ResourceInNodeV3 x;
  x.GetCpuSet().cpu_count = cpu_t::from_raw_value(r.cpu_raw);
  for (int w = 0; w < CRANE_CORE_WORDS; ++w)
    for (int b = 0; b < 64; ++b)
      if (r.core[w] >> b & 1) x.GetCpuSet().core_ids.insert(w * 64 + b);
  x.SetMemoryBytes(r.mem);
  x.SetMemorySwBytes(r.mem_sw);
  for (uint32_t e = 0; e < d.n_entries; ++e) {
    if (!r.gres[e]) continue;
    std::set<SlotId>& s = x.GetGres()[d.name_str[d.entry_name[e]]][d.type_str[e]];
    for (int b = 0; b < CRANE_MAX_SLOTS; ++b)
      if (r.gres[e] >> b & 1) s.insert(d.slot_str[b]);
  }
  return x;
}

void ToAbi(const Dict& d, const ResourceInNodeV3& x, crane_res_in_node_t* r) {
  memset(r, 0, sizeof *r);
  r->cpu_raw = x.GetCpuSet().cpu_count.raw_value();
  r->mem = x.GetMemoryBytes();
  r->mem_sw = x.GetMemorySwBytes();
  for (uint32_t id : x.GetCpuSet().core_ids)
    if (id < 64 * CRANE_CORE_WORDS) r->core[id / 64] |= 1ull << (id % 64);
  for (uint32_t e = 0; e < d.n_entries; ++e) {
    const auto& names = x.GetGres().name_type_slots_map;
    auto nit = names.find(d.name_str[d.entry_name[e]]);
    if (nit == names.end()) continue;
    auto tit = nit->second.type_slots_map.find(d.type_str[e]);
    if (tit == nit->second.type_slots_map.end()) continue;
    for (int b = 0; b < CRANE_MAX_SLOTS; ++b)
      if (tit->second.count(d.slot_str[b])) r->gres[e] |= uint16_t(1u << b);
  }
}

ResourceView ViewFromAbi(const Dict& d, const crane_res_view_t& v) {
  ResourceView x;
  x.SetCpuCount(cpu_t::from_raw_value(v.cpu_raw));
  x.SetMemoryBytes(v.mem);
  x.SetMemorySwBytes(v.mem_sw);
  for (int g = 0; g < CRANE_GRES_NAMES; ++g) {
    bool any = v.gres_total[g] != 0;
    for (uint32_t e = 0; e < d.n_entries; ++e)
      if (d.entry_name[e] == g && v.gres_spec[e]) any = true;
    if (!any) continue;
    GresCount& gc = x.GetGresMap()[d.name_str[g]];
    gc.total = v.gres_total[g];
    for (uint32_t e = 0; e < d.n_entries; ++e)
      if (d.entry_name[e] == g && v.gres_spec[e]) gc.specified[d.type_str[e]] = v.gres_spec[e];
  }
  return x;
}

uint32_t NodeIndex(const std::string& name) { return (uint32_t)std::stoul(name.substr(2)); }

}  // namespace

extern "C" int crane_ref_schedule_steps(const crane_cluster_t* cl, const crane_step_jobs_t* jb, const crane_steps_t* st,
                                        const uint8_t* erased, crane_step_placements_t* out, uint32_t* visit,
                                        double* elapsed_ms) {
  if (!cl || !jb || !st || !out) return CRANE_EINVAL;
  Dict d(cl);
  const uint32_t J = jb->n_jobs, S = st->n;
  if (jb->step_off[J] != S) return CRANE_EINVAL;
  std::vector<Ctld::CommonStepInCtld> steps(S);
  std::vector<Ctld::JobInCtld> jobs(J);
  for (uint32_t j = 0; j < J; ++j) {
    Ctld::JobInCtld& job = jobs[j];
    for (uint32_t k = jb->node_off[j]; k < jb->node_off[j + 1]; ++k)
      job.step_res_avail_.AddResourceInNode(NodeName(jb->node[k]), FromAbi(d, jb->avail[k]));
    for (uint32_t s = jb->step_off[j]; s < jb->step_off[j + 1]; ++s) {
      Ctld::CommonStepInCtld& x = steps[s];
      x.job_id = j;
      x.m_step_id_ = s;
      x.node_num = st->node_num[s];
      x.ntasks = st->ntasks[s];
      x.ntasks_per_node_min = st->ntasks_per_node_min[s];
      x.ntasks_per_node_max = st->ntasks_per_node_max[s];
      x.req_node_res_view = ViewFromAbi(d, st->req_node[s]);
      x.req_task_res_view = ViewFromAbi(d, st->req_task[s]);
      if (st->incl_off)
        for (uint32_t k = st->incl_off[s]; k < st->incl_off[s + 1]; ++k)
          x.included_nodes.insert(st->incl_nodes[k] == 0xFFFFFFFFu ? std::string("unknown-host") : NodeName(st->incl_nodes[k]));
      if (st->excl_off)
        for (uint32_t k = st->excl_off[s]; k < st->excl_off[s + 1]; ++k)
          x.excluded_nodes.insert(st->excl_nodes[k] == 0xFFFFFFFFu ? std::string("unknown-host") : NodeName(st->excl_nodes[k]));
      job.pending_step_ids_.push(s);
      if (!erased || !erased[s]) job.m_steps_.emplace(s, &x);  // an erased step: GetStep() == nullptr (:1883-1889)
    }
  }
  // the order the reference walks each job's nodes in: step_res_avail_.EachNodeResMap()
  if (visit)
    for (uint32_t j = 0; j < J; ++j) {
      std::vector<uint32_t> pos;
      for (const auto& name : jobs[j].step_res_avail_.EachNodeResMap() | std::views::keys) {
        const uint32_t n = NodeIndex(name);
        const uint32_t* b = jb->node + jb->node_off[j];
        const uint32_t* e = jb->node + jb->node_off[j + 1];
        pos.push_back((uint32_t)(std::lower_bound(b, e, n) - b));
      }
      std::copy(pos.begin(), pos.end(), visit + jb->node_off[j]);
    }
  std::vector<std::vector<Ctld::CommonStepInCtld*>> scheduled(J);
  std::vector<uint32_t> popped(J);
  const auto t0 = std::chrono::steady_clock::now();
  for (uint32_t j = 0; j < J; ++j) popped[j] = jobs[j].SchedulePendingSteps(&scheduled[j]);
  const auto t1 = std::chrono::steady_clock::now();
  if (elapsed_ms) *elapsed_ms = std::chrono::duration<double, std::milli>(t1 - t0).count();

  out->node_off[0] = out->task_off[0] = 0;
  for (uint32_t s = 0; s < S; ++s) {
    out->node_off[s + 1] = out->node_off[s] + st->node_num[s];
    out->task_off[s + 1] = out->task_off[s] + st->ntasks[s];
    out->scheduled[s] = 0;
    for (uint32_t x = out->node_off[s]; x < out->node_off[s + 1]; ++x) {
      out->alloc_node[x] = out->alloc_ntasks[x] = 0;
      memset(&out->alloc_res[x], 0, sizeof(crane_res_in_node_t));
    }
    for (uint32_t x = out->task_off[s]; x < out->task_off[s + 1]; ++x) {
      out->task_node[x] = 0;
      memset(&out->task_res[x], 0, sizeof(crane_res_in_node_t));
    }
  }
  for (uint32_t j = 0; j < J; ++j) {
    out->placed[j] = popped[j];
    for (Ctld::CommonStepInCtld* x : scheduled[j]) {
      const uint32_t s = x->StepId();
      out->scheduled[s] = 1;
      std::map<uint32_t, const ResourceInNodeV3*> by_node;  // node rows in node-index order (D3)
      for (const auto& [name, r] : x->AllocatedRes().EachNodeResMap()) by_node[NodeIndex(name)] = &r;
      uint32_t i = out->node_off[s];
      for (const auto& [n, r] : by_node) {
        out->alloc_node[i] = n;
        out->alloc_ntasks[i] = (uint32_t)x->craned_task_map.at(NodeName(n)).size();
        ToAbi(d, *r, &out->alloc_res[i]);
        ++i;
      }
      for (const auto& [name, ids] : x->craned_task_map)
        for (uint32_t t : ids) out->task_node[out->task_off[s] + t] = NodeIndex(name);
      for (const auto& [t, r] : x->task_res_map) ToAbi(d, r, &out->task_res[out->task_off[s] + t]);
    }
  }
  for (uint32_t j = 0; j < J; ++j)
    for (uint32_t k = jb->node_off[j]; k < jb->node_off[j + 1]; ++k)
      ToAbi(d, jobs[j].step_res_avail_.At(NodeName(jb->node[k])), &jb->avail[k]);
  return CRANE_OK;
}
