// crane_adaptor.cpp — flattening between the reference's job/node objects and
// the C-ABI tables (see crane_adaptor.h). Pure host plumbing: every scheduling
// decision is taken by crane_sched_node_select on the GPU.
#include "crane_adaptor.h"

#include <algorithm>
#include <cstring>
#include <stdexcept>

namespace crane_b200 {

namespace {
const char* kReasonString[] = {"", "Priority", "Resource", "Resource Reserved", "Partition Not Found"};
const char* QosReasonString(uint8_t code) {
  switch (code) {
    case CRANE_REASON_QOS_CPU: return "QosCpuResourceLimit";
    case CRANE_REASON_QOS_JOBS: return "QosJobsResourceLimit";
    case CRANE_REASON_QOS_WALL: return "QosWallTimeLimit";
    case CRANE_REASON_QOS_MEM: return "QosMemResourceLimit";
    case CRANE_REASON_QOS_GRES: return "QosGresResourceLimit";
    case CRANE_REASON_QOS_INVALID: return "InvalidQOS";
    default: return nullptr;
  }
}
}

struct SchedulerAlgo::Impl {
  crane_sched_t* h{nullptr};
  // dictionaries (dense ids)
  std::vector<CranedId> node_names;                       // index -> hostname (sorted)
  std::unordered_map<CranedId, uint32_t> node_index;
  std::vector<PartitionId> part_names;
  std::unordered_map<PartitionId, uint32_t> part_index;
  // gres (name,type) dictionary, sorted by (name, type); per node the sorted slot lists
  std::vector<std::pair<std::string, std::string>> gres_entries;
  std::map<std::string, uint32_t> gres_name_id;
  std::map<std::pair<std::string, std::string>, uint32_t> gres_entry_id;
  std::vector<std::vector<std::vector<SlotId>>> node_slots;  // [node][entry] -> sorted slot ids
  std::unordered_map<std::string, uint32_t> account_id, qos_id, user_id;

  uint32_t Intern(std::unordered_map<std::string, uint32_t>& m, const std::string& s) {
    auto it = m.find(s);
    if (it != m.end()) return it->second;
    uint32_t id = (uint32_t)m.size();
    m.emplace(s, id);
    return id;
  }

  crane_res_in_node_t ToRow(uint32_t node, const ResourceInNodeV3& r) const {
    crane_res_in_node_t o;
    memset(&o, 0, sizeof o);
    o.cpu_raw = r.cpu_count_raw;
    o.mem = r.memory_bytes;
    o.mem_sw = r.memory_sw_bytes;
    for (uint32_t id : r.core_ids) {
      if (id >= 64u * CRANE_CORE_WORDS) throw std::runtime_error("core id beyond CRANE_CORE_WORDS");
      o.core[id / 64] |= 1ull << (id % 64);
    }
    for (const auto& [name, types] : r.gres)
      for (const auto& [type, slots] : types) {
        auto eit = gres_entry_id.find({name, type});
        if (eit == gres_entry_id.end()) throw std::runtime_error("gres entry not in the cluster dictionary: " + name + ":" + type);
        const auto& known = node_slots[node][eit->second];
        for (const SlotId& s : slots) {
          auto pos = std::lower_bound(known.begin(), known.end(), s);
          if (pos == known.end() || *pos != s) throw std::runtime_error("unknown gres slot " + s);
          o.gres[eit->second] |= (uint16_t)(1u << (pos - known.begin()));
        }
      }
    return o;
  }
  ResourceInNodeV3 FromRow(uint32_t node, const crane_res_in_node_t& o) const {
    ResourceInNodeV3 r;
    r.cpu_count_raw = o.cpu_raw;
    r.memory_bytes = o.mem;
    r.memory_sw_bytes = o.mem_sw;
    for (uint32_t w = 0; w < CRANE_CORE_WORDS; ++w)
      for (uint32_t b = 0; b < 64; ++b)
        if (o.core[w] >> b & 1) r.core_ids.insert(w * 64 + b);
    for (uint32_t e = 0; e < gres_entries.size(); ++e)
      for (uint32_t b = 0; b < CRANE_MAX_SLOTS; ++b)
        if (o.gres[e] >> b & 1) r.gres[gres_entries[e].first][gres_entries[e].second].insert(node_slots[node][e][b]);
    return r;
  }
  // a max_tres map of struct Qos: counts + which names / types are listed at all
  crane_tres_limit_t ToLimit(const ResourceView& v) const {
    crane_tres_limit_t L;
    memset(&L, 0, sizeof L);
    L.view.cpu_raw = v.cpu_count_raw;
    L.view.mem = v.memory_bytes;
    L.view.mem_sw = v.memory_sw_bytes;
    for (const auto& [name, gc] : v.gres_map) {
      auto nit = gres_name_id.find(name);
      if (nit == gres_name_id.end()) continue;  // a name no node offers: no job can ask for it
      L.gres_name_present |= (uint8_t)(1u << nit->second);
      L.view.gres_total[nit->second] = (uint16_t)std::min<uint64_t>(gc.total, 0xFFFF);
      for (const auto& [type, cnt] : gc.specified) {
        auto eit = gres_entry_id.find({name, type});
        if (eit == gres_entry_id.end()) continue;
        L.gres_spec_present |= (uint8_t)(1u << eit->second);
        L.view.gres_spec[eit->second] = (uint16_t)std::min<uint64_t>(cnt, 0xFFFF);
      }
    }
    return L;
  }
  crane_meta_resource_t ToMeta(const MetaResource& r) const {
    crane_meta_resource_t o;
    memset(&o, 0, sizeof o);
    o.cpu_raw = r.resource.cpu_count_raw;
    o.mem = r.resource.memory_bytes;
    o.mem_sw = r.resource.memory_sw_bytes;
    for (const auto& [name, gc] : r.resource.gres_map) {
      auto nit = gres_name_id.find(name);
      if (nit == gres_name_id.end()) continue;
      o.gres_total[nit->second] = (uint32_t)gc.total;
      for (const auto& [type, cnt] : gc.specified) {
        auto eit = gres_entry_id.find({name, type});
        if (eit != gres_entry_id.end()) o.gres_spec[eit->second] = (uint32_t)cnt;
      }
    }
    o.jobs_count = r.jobs_count;
    o.wall_time = r.wall_time;
    return o;
  }
  void FromMeta(const crane_meta_resource_t& o, MetaResource& r) const {
    r.resource.cpu_count_raw = o.cpu_raw;
    r.resource.memory_bytes = o.mem;
    r.resource.memory_sw_bytes = o.mem_sw;
    for (const auto& [name, g] : gres_name_id) {
      uint64_t any = o.gres_total[g];
      for (uint32_t e = 0; e < gres_entries.size(); ++e)
        if (gres_entries[e].first == name) any |= o.gres_spec[e];
      if (!any && !r.resource.gres_map.count(name)) continue;
      GresCount& gc = r.resource.gres_map[name];
      gc.total = o.gres_total[g];
      for (uint32_t e = 0; e < gres_entries.size(); ++e)
        if (gres_entries[e].first == name && (o.gres_spec[e] || gc.specified.count(gres_entries[e].second)))
          gc.specified[gres_entries[e].second] = o.gres_spec[e];
    }
    r.jobs_count = o.jobs_count;
    r.wall_time = o.wall_time;
  }
  crane_res_view_t ToView(const ResourceView& v) const {
    crane_res_view_t o;
    memset(&o, 0, sizeof o);
    o.cpu_raw = v.cpu_count_raw;
    o.mem = v.memory_bytes;
    o.mem_sw = v.memory_sw_bytes;
    for (const auto& [name, gc] : v.gres_map) {
      auto nit = gres_name_id.find(name);
      // a name no node offers can never be satisfied: keep it visible as an
      // unsatisfiable request on a spare name id if there is one
      uint32_t g = nit != gres_name_id.end() ? nit->second : (uint32_t)gres_name_id.size();
      if (g >= CRANE_GRES_NAMES) throw std::runtime_error("too many gres names");
      o.gres_total[g] = (uint16_t)std::min<uint64_t>(gc.total, 0xFFFF);
      for (const auto& [type, cnt] : gc.specified) {
        auto eit = gres_entry_id.find({name, type});
        if (eit == gres_entry_id.end()) {  // typed request nobody can serve
          o.gres_total[g] = 0xFFFF;
          continue;
        }
        o.gres_spec[eit->second] = (uint16_t)std::min<uint64_t>(cnt, 0xFFFF);
      }
    }
    return o;
  }
};

SchedulerAlgo::SchedulerAlgo(const PriorityConfig& p, uint32_t batch, int device) : m_(new Impl) {
  crane_sched_config_t c;
  memset(&c, 0, sizeof c);
  c.priority_type = p.Type == PriorityConfig::MultiFactor;
  c.favor_small = p.FavorSmall;
  c.max_age_s = p.MaxAge;
  c.weight_age = p.WeightAge;
  c.weight_fair_share = p.WeightFairShare;
  c.weight_job_size = p.WeightJobSize;
  c.weight_partition = p.WeightPartition;
  c.weight_qos = p.WeightQoS;
  c.scheduled_batch_size = batch;
  c.max_jobs_per_node = 1000;           // kAlgoMaxJobNumPerNode, JobScheduler.h:263
  c.max_time_window_s = 7 * 24 * 3600;  // kAlgoMaxTimeWindow, JobScheduler.h:264
  int rc = crane_sched_create(&c, device, &m_->h);
  if (rc != CRANE_OK) throw std::runtime_error("crane_sched_create failed: " + std::to_string(rc));
}

SchedulerAlgo::~SchedulerAlgo() {
  if (m_ && m_->h) crane_sched_destroy(m_->h);
}

void SchedulerAlgo::SetCluster(const std::map<CranedId, CranedMeta>& craneds,
                               const std::map<PartitionId, std::set<CranedId>>& partitions) {
  Impl& m = *m_;
  m.node_names.clear();
  m.node_index.clear();
  for (const auto& [id, meta] : craneds) {  // std::map: sorted hostname order
    m.node_index.emplace(id, (uint32_t)m.node_names.size());
    m.node_names.push_back(id);
  }
  // gres dictionary over all nodes, sorted by (name, type)
  std::set<std::pair<std::string, std::string>> entries;
  for (const auto& [id, meta] : craneds)
    for (const auto& [name, types] : meta.res_total.gres)
      for (const auto& [type, slots] : types) entries.insert({name, type});
  if (entries.size() > CRANE_GRES_ENTRIES) throw std::runtime_error("more than CRANE_GRES_ENTRIES gres (name,type) pairs");
  m.gres_entries.assign(entries.begin(), entries.end());
  m.gres_name_id.clear();
  m.gres_entry_id.clear();
  crane_cluster_t c;
  memset(&c, 0, sizeof c);
  for (uint32_t e = 0; e < m.gres_entries.size(); ++e) {
    auto [it, fresh] = m.gres_name_id.emplace(m.gres_entries[e].first, (uint32_t)m.gres_name_id.size());
    m.gres_entry_id[m.gres_entries[e]] = e;
    c.gres_entry_name[e] = (uint8_t)it->second;
  }
  c.n_gres_entries = (uint32_t)m.gres_entries.size();
  const uint32_t M = (uint32_t)m.node_names.size();
  m.node_slots.assign(M, std::vector<std::vector<SlotId>>(m.gres_entries.size()));
  std::vector<crane_res_in_node_t> totals(M);
  std::vector<uint8_t> alive(M), drain(M);
  uint32_t n = 0;
  for (const auto& [id, meta] : craneds) {
    for (const auto& [name, types] : meta.res_total.gres)
      for (const auto& [type, slots] : types) {
        auto& known = m.node_slots[n][m.gres_entry_id.at({name, type})];
        known.assign(slots.begin(), slots.end());  // std::set: lexicographic slot-path order
        if (known.size() > CRANE_MAX_SLOTS) throw std::runtime_error("more than CRANE_MAX_SLOTS slots of one gres type on " + id);
      }
    totals[n] = m.ToRow(n, meta.res_total);
    alive[n] = meta.alive;
    drain[n] = meta.drain;
    ++n;
  }
  m.part_names.clear();
  m.part_index.clear();
  std::vector<uint32_t> part_off{0}, part_nodes;
  for (const auto& [pid, ids] : partitions) {
    m.part_index.emplace(pid, (uint32_t)m.part_names.size());
    m.part_names.push_back(pid);
    std::vector<uint32_t> idx;
    for (const auto& id : ids) {
      auto it = m.node_index.find(id);
      if (it != m.node_index.end()) idx.push_back(it->second);
    }
    std::sort(idx.begin(), idx.end());
    part_nodes.insert(part_nodes.end(), idx.begin(), idx.end());
    part_off.push_back((uint32_t)part_nodes.size());
  }
  c.n_nodes = M;
  c.res_total = totals.data();
  c.alive = alive.data();
  c.drain = drain.data();
  c.n_partitions = (uint32_t)m.part_names.size();
  c.part_off = part_off.data();
  c.part_nodes = part_nodes.data();
  int rc = crane_sched_set_cluster(m.h, &c);
  if (rc != CRANE_OK) throw std::runtime_error(std::string("crane_sched_set_cluster: ") + crane_sched_last_error(m.h));
}

void SchedulerAlgo::NodeSelect(int64_t now, const std::vector<std::unique_ptr<RnJobInScheduler>>& running_jobs,
                               const std::vector<std::unique_ptr<PdJobInScheduler>>& pending_jobs) {
  Impl& m = *m_;
  const uint32_t N = (uint32_t)pending_jobs.size(), R = (uint32_t)running_jobs.size();
  const uint32_t P = (uint32_t)m.part_names.size();
  // ---- pending: PdJobInScheduler (JobScheduler.h:91-164) -> columns ---------
  std::vector<uint32_t> partition(N), node_num(N), ntasks(N), ntpn_min(N), ntpn_max(N), part_prio(N), qos_prio(N),
      account(N), qos(N), user(N), incl_off(N + 1, 0), excl_off(N + 1, 0), incl_nodes, excl_nodes;
  std::vector<int64_t> time_limit(N), submit(N);
  std::vector<uint8_t> exclusive(N);
  std::vector<double> mandated(N);
  std::vector<crane_res_view_t> req_node(N), req_task(N), req_total(N);
  uint64_t total_alloc = 0;
  for (uint32_t i = 0; i < N; ++i) {
    const PdJobInScheduler& j = *pending_jobs[i];
    auto pit = m.part_index.find(j.partition_id);
    partition[i] = pit != m.part_index.end() ? pit->second : P;  // unknown -> "Partition Not Found"
    time_limit[i] = j.time_limit;
    submit[i] = j.submit_time;
    node_num[i] = j.node_num;
    ntasks[i] = j.ntasks;
    ntpn_min[i] = j.ntasks_per_node_min;
    ntpn_max[i] = j.ntasks_per_node_max;
    exclusive[i] = j.exclusive;
    part_prio[i] = j.partition_priority;
    qos_prio[i] = j.qos_priority;
    account[i] = m.Intern(m.account_id, j.account);
    qos[i] = m.Intern(m.qos_id, j.qos);
    user[i] = m.Intern(m.user_id, j.username);
    mandated[i] = j.priority;
    req_node[i] = m.ToView(j.req_node_res_view);
    req_task[i] = m.ToView(j.req_task_res_view);
    req_total[i] = m.ToView(j.req_total_res_view);
    // node lists; a listed host the cluster does not know can never match
    for (const auto& id : j.included_nodes) {
      auto it = m.node_index.find(id);
      if (it != m.node_index.end()) incl_nodes.push_back(it->second);
    }
    if (!j.included_nodes.empty() && incl_nodes.size() == incl_off[i]) incl_nodes.push_back(0xFFFFFFFFu);  // "unknown host": matches nothing
    std::sort(incl_nodes.begin() + incl_off[i], incl_nodes.end());
    incl_off[i + 1] = (uint32_t)incl_nodes.size();
    for (const auto& id : j.excluded_nodes) {
      auto it = m.node_index.find(id);
      if (it != m.node_index.end()) excl_nodes.push_back(it->second);
    }
    std::sort(excl_nodes.begin() + excl_off[i], excl_nodes.end());
    excl_off[i + 1] = (uint32_t)excl_nodes.size();
    total_alloc += j.node_num;
  }
  crane_pending_t pd;
  memset(&pd, 0, sizeof pd);
  pd.n = N;
  pd.partition = partition.data();
  pd.time_limit = time_limit.data();
  pd.submit_time = submit.data();
  pd.node_num = node_num.data();
  pd.ntasks = ntasks.data();
  pd.ntasks_per_node_min = ntpn_min.data();
  pd.ntasks_per_node_max = ntpn_max.data();
  pd.exclusive = exclusive.data();
  pd.partition_priority = part_prio.data();
  pd.qos_priority = qos_prio.data();
  pd.account = account.data();
  pd.qos = qos.data();
  pd.user = user.data();
  pd.mandated_priority = mandated.data();
  pd.req_node = req_node.data();
  pd.req_task = req_task.data();
  pd.req_total = req_total.data();
  pd.incl_off = incl_off.data();
  pd.incl_nodes = incl_nodes.data();
  pd.excl_off = excl_off.data();
  pd.excl_nodes = excl_nodes.data();

  // ---- running: RnJobInScheduler (JobScheduler.h:56-89) ----------------------
  std::vector<int64_t> rs(R), re(R), rcpu(R);
  std::vector<uint32_t> rnn(R), rpp(R), rqp(R), racc(R), roff(R + 1, 0), rnode;
  std::vector<uint64_t> rmem(R);
  std::vector<crane_res_in_node_t> rres;
  for (uint32_t k = 0; k < R; ++k) {
    const RnJobInScheduler& j = *running_jobs[k];
    rs[k] = j.start_time;
    re[k] = j.end_time;
    rnn[k] = j.node_num;
    rpp[k] = j.partition_priority;
    rqp[k] = j.qos_priority;
    racc[k] = m.Intern(m.account_id, j.account);
    rcpu[k] = j.allocated_res_view.cpu_count_raw;
    rmem[k] = j.allocated_res_view.memory_bytes;
    std::vector<std::pair<uint32_t, const ResourceInNodeV3*>> nodes;
    for (const auto& [id, res] : j.allocated_res) {
      auto it = m.node_index.find(id);
      if (it != m.node_index.end()) nodes.push_back({it->second, &res});
    }
    std::sort(nodes.begin(), nodes.end(), [](const auto& a, const auto& b) { return a.first < b.first; });
    for (const auto& [idx, res] : nodes) {
      rnode.push_back(idx);
      rres.push_back(m.ToRow(idx, *res));
    }
    roff[k + 1] = (uint32_t)rnode.size();
  }
  crane_running_t rn;
  memset(&rn, 0, sizeof rn);
  rn.n = R;
  rn.start_time = rs.data();
  rn.end_time = re.data();
  rn.node_num = rnn.data();
  rn.partition_priority = rpp.data();
  rn.qos_priority = rqp.data();
  rn.account = racc.data();
  rn.view_cpu_raw = rcpu.data();
  rn.view_mem = rmem.data();
  rn.alloc_off = roff.data();
  rn.alloc_node = rnode.data();
  rn.alloc_res = rres.data();

  // ---- the call ---------------------------------------------------------------
  std::vector<uint8_t> o_reason(N);
  std::vector<double> o_prio(N);
  std::vector<int64_t> o_start(N), o_end(N);
  std::vector<uint32_t> o_nalloc(N), o_off(N + 1), o_node(total_alloc), o_ntasks(total_alloc);
  std::vector<crane_res_in_node_t> o_res(total_alloc);
  crane_placements_t out;
  out.reason = o_reason.data();
  out.priority = o_prio.data();
  out.start_time = o_start.data();
  out.end_time = o_end.data();
  out.n_alloc = o_nalloc.data();
  out.alloc_off = o_off.data();
  out.alloc_node = o_node.data();
  out.alloc_ntasks = o_ntasks.data();
  out.alloc_res = o_res.data();
  int rc = crane_sched_node_select(m.h, now, &rn, &pd, &out);
  if (rc != CRANE_OK) throw std::runtime_error(std::string("crane_sched_node_select: ") + crane_sched_last_error(m.h));

  // ---- write back: the fields NodeSelect mutates (JobScheduler.h:116-132) -----
  for (const auto& r : running_jobs) r->end_time = std::max(r->end_time, now + 1);  // JobScheduler.cpp:5547
  for (uint32_t i = 0; i < N; ++i) {
    PdJobInScheduler& j = *pending_jobs[i];
    j.priority = o_prio[i];
    j.reason = kReasonString[o_reason[i]];
    j.craned_ids.clear();
    j.craned_id_to_task_num.clear();
    j.allocated_res.clear();
    j.start_time = o_start[i];
    j.end_time = o_end[i];
    for (uint32_t k = o_off[i]; k < o_off[i] + o_nalloc[i]; ++k) {
      const CranedId& id = m.node_names[o_node[k]];
      j.craned_ids.push_back(id);  // node-index ascending
      j.craned_id_to_task_num[id] = o_ntasks[k];
      j.allocated_res.emplace(id, m.FromRow(o_node[k], o_res[k]));
    }
  }
}

void SchedulerAlgo::CheckAndMallocQosResource(const std::map<std::string, Qos>& qos_table, QosUsage& usage,
                                              const std::vector<std::unique_ptr<PdJobInScheduler>>& pending_jobs) {
  Impl& m = *m_;
  const uint32_t N = (uint32_t)pending_jobs.size();
  // account chains (PdJobInScheduler::account_chain); parents the jobs themselves never name get ids now
  std::vector<uint32_t> chain_off(N + 1, 0), chain;
  for (uint32_t i = 0; i < N; ++i) {
    for (const auto& a : pending_jobs[i]->account_chain) chain.push_back(m.Intern(m.account_id, a));
    chain_off[i + 1] = (uint32_t)chain.size();
  }
  // the qos / user ids are the ones NodeSelect uploaded with the pending table
  const uint32_t Q = (uint32_t)m.qos_id.size(), U = (uint32_t)m.user_id.size(), A = (uint32_t)m.account_id.size();
  if (N == 0 || Q == 0) return;
  std::vector<std::string> qos_name(Q), user_name(U), acct_name(A);
  for (const auto& [s, id] : m.qos_id) qos_name[id] = s;
  for (const auto& [s, id] : m.user_id) user_name[id] = s;
  for (const auto& [s, id] : m.account_id) acct_name[id] = s;
  std::vector<uint8_t> valid(Q, 0);
  std::vector<uint32_t> mju(Q, 0), mja(Q, 0), mj(Q, 0);
  std::vector<int64_t> mcpu(Q, 0), mwall(Q, 0);
  std::vector<crane_tres_limit_t> tu(Q), ta(Q), tq(Q);
  memset(tu.data(), 0, sizeof(crane_tres_limit_t) * Q);
  memset(ta.data(), 0, sizeof(crane_tres_limit_t) * Q);
  memset(tq.data(), 0, sizeof(crane_tres_limit_t) * Q);
  for (uint32_t q = 0; q < Q; ++q) {
    auto it = qos_table.find(qos_name[q]);
    if (it == qos_table.end() || it->second.deleted) continue;  // GetExistedQosInfo fails: "InvalidQOS"
    const Qos& s = it->second;
    valid[q] = 1;
    mju[q] = s.max_jobs_per_user; mja[q] = s.max_jobs_per_account; mj[q] = s.max_jobs;
    mcpu[q] = s.max_cpus_per_user_raw; mwall[q] = s.max_wall;
    tu[q] = m.ToLimit(s.max_tres_per_user); ta[q] = m.ToLimit(s.max_tres_per_account); tq[q] = m.ToLimit(s.max_tres);
  }
  // dense usage tables; what the maps do not hold is zero
  std::vector<crane_meta_resource_t> uu((size_t)U * Q), au((size_t)A * Q), qu(Q);
  memset(uu.data(), 0, uu.size() * sizeof(crane_meta_resource_t));
  memset(au.data(), 0, au.size() * sizeof(crane_meta_resource_t));
  memset(qu.data(), 0, qu.size() * sizeof(crane_meta_resource_t));
  auto load = [&](const std::map<std::string, std::map<std::string, MetaResource>>& src,
                  const std::unordered_map<std::string, uint32_t>& ids, std::vector<crane_meta_resource_t>& dst) {
    for (const auto& [key, per_qos] : src) {
      auto kit = ids.find(key);
      if (kit == ids.end()) continue;  // nobody in this queue touches it
      for (const auto& [qn, r] : per_qos) {
        auto qit = m.qos_id.find(qn);
        if (qit != m.qos_id.end()) dst[(size_t)kit->second * Q + qit->second] = m.ToMeta(r);
      }
    }
  };
  load(usage.user, m.user_id, uu);
  load(usage.account, m.account_id, au);
  for (const auto& [qn, r] : usage.qos) {
    auto qit = m.qos_id.find(qn);
    if (qit != m.qos_id.end()) qu[qit->second] = m.ToMeta(r);
  }
  const std::vector<crane_meta_resource_t> uu0 = uu, au0 = au, qu0 = qu;

  crane_qos_table_t t;
  memset(&t, 0, sizeof t);
  t.n_qos = Q; t.n_users = U; t.n_accounts = A;
  t.valid = valid.data();
  t.max_jobs_per_user = mju.data(); t.max_jobs_per_account = mja.data(); t.max_jobs = mj.data();
  t.max_cpus_per_user_raw = mcpu.data(); t.max_wall = mwall.data();
  t.max_tres_per_user = tu.data(); t.max_tres_per_account = ta.data(); t.max_tres = tq.data();
  t.chain_off = chain_off.data(); t.chain_acct = chain.data();
  t.user_usage = uu.data(); t.account_usage = au.data(); t.qos_usage = qu.data();
  std::vector<uint8_t> reason(N);
  int rc = crane_sched_qos_filter(m.h, &t, reason.data());
  if (rc != CRANE_OK) throw std::runtime_error(std::string("crane_sched_qos_filter: ") + crane_sched_last_error(m.h));

  for (uint32_t i = 0; i < N; ++i)
    if (const char* why = QosReasonString(reason[i])) pending_jobs[i]->reason = why;
  // usage back into the maps: only the entries the pass changed
  auto store = [&](const std::vector<crane_meta_resource_t>& now_, const std::vector<crane_meta_resource_t>& before,
                   const std::vector<std::string>& names, std::map<std::string, std::map<std::string, MetaResource>>& dst) {
    for (size_t k = 0; k < now_.size(); ++k)
      if (memcmp(&now_[k], &before[k], sizeof(crane_meta_resource_t)) != 0) m.FromMeta(now_[k], dst[names[k / Q]][qos_name[k % Q]]);
  };
  store(uu, uu0, user_name, usage.user);
  store(au, au0, acct_name, usage.account);
  for (uint32_t q = 0; q < Q; ++q)
    if (memcmp(&qu[q], &qu0[q], sizeof(crane_meta_resource_t)) != 0) m.FromMeta(qu[q], usage.qos[qos_name[q]]);
}

}  // namespace crane_b200

namespace crane_b200 {

std::vector<uint32_t> SchedulerAlgo::SchedulePendingSteps(int64_t now, const std::vector<JobStepState*>& jobs,
                                                          std::vector<std::vector<CommonStepInCtld*>>* scheduled_steps) {
  Impl& m = *m_;
  const uint32_t J = (uint32_t)jobs.size();
  // ---- jobs: nodes of step_res_avail_ (index-ascending) + the live steps in FIFO order ----
  std::vector<uint32_t> node_off(J + 1, 0), node, step_off(J + 1, 0);
  std::vector<crane_res_in_node_t> avail;
  std::vector<CommonStepInCtld*> live;
  for (uint32_t j = 0; j < J; ++j) {
    const JobStepState& js = *jobs[j];
    std::vector<std::pair<uint32_t, const ResourceInNodeV3*>> nodes;
    for (const auto& [id, res] : js.step_res_avail) {
      auto it = m.node_index.find(id);
      if (it == m.node_index.end()) throw std::runtime_error("step_res_avail_ node not in the cluster: " + id);
      nodes.push_back({it->second, &res});
    }
    std::sort(nodes.begin(), nodes.end(), [](const auto& a, const auto& b) { return a.first < b.first; });
    for (const auto& [idx, res] : nodes) {
      node.push_back(idx);
      avail.push_back(m.ToRow(idx, *res));
    }
    node_off[j + 1] = (uint32_t)node.size();
    for (uint32_t id : js.pending_step_ids) {
      auto it = js.steps.find(id);
      if (it != js.steps.end()) live.push_back(it->second);  // GetStep() == nullptr: removed (:1883-1889)
    }
    step_off[j + 1] = (uint32_t)live.size();
  }
  const uint32_t S = (uint32_t)live.size();
  std::vector<uint32_t> nn(S), nt(S), t0(S), t1(S), incl_off(S + 1, 0), incl, excl_off(S + 1, 0), excl;
  std::vector<crane_res_view_t> vn(S), vt(S);
  auto list_index = [&](const std::string& id) {
    auto it = m.node_index.find(id);
    return it == m.node_index.end() ? 0xFFFFFFFFu : it->second;  // a host the cluster does not know
  };
  for (uint32_t s = 0; s < S; ++s) {
    const CommonStepInCtld& x = *live[s];
    nn[s] = x.node_num;
    nt[s] = x.ntasks;
    t0[s] = x.ntasks_per_node_min;
    t1[s] = x.ntasks_per_node_max;
    vn[s] = m.ToView(x.req_node_res_view);
    vt[s] = m.ToView(x.req_task_res_view);
    for (const auto& id : x.included_nodes) incl.push_back(list_index(id));
    incl_off[s + 1] = (uint32_t)incl.size();
    for (const auto& id : x.excluded_nodes) {
      const uint32_t n = list_index(id);
      if (n != 0xFFFFFFFFu) excl.push_back(n);  // an unknown host excludes nothing
    }
    excl_off[s + 1] = (uint32_t)excl.size();
  }
  crane_step_jobs_t cj{J, node_off.data(), node.data(), avail.data(), step_off.data()};
  crane_steps_t cs{S, nn.data(), nt.data(), t0.data(), t1.data(), vn.data(), vt.data(),
                   incl_off.data(), incl.data(), excl_off.data(), excl.data()};
  uint64_t nrows = 0, trows = 0;
  for (uint32_t s = 0; s < S; ++s) { nrows += nn[s]; trows += nt[s]; }
  std::vector<uint32_t> placed(J), o_noff(S + 1), o_node(nrows), o_ntasks(nrows), o_toff(S + 1), o_tnode(trows);
  std::vector<uint8_t> sched(S);
  std::vector<crane_res_in_node_t> o_res(nrows), o_tres(trows);
  crane_step_placements_t out{placed.data(), sched.data(), o_noff.data(), o_node.data(), o_ntasks.data(),
                              o_res.data(), o_toff.data(), o_tnode.data(), o_tres.data()};
  int rc = crane_sched_schedule_steps(m.h, &cj, &cs, &out, nullptr);
  if (rc != CRANE_OK) throw std::runtime_error(std::string("crane_sched_schedule_steps: ") + crane_sched_last_error(m.h));

  // ---- write back ------------------------------------------------------------------
  if (scheduled_steps) scheduled_steps->assign(J, {});
  std::vector<uint32_t> popped(J, 0);
  for (uint32_t j = 0; j < J; ++j) {
    JobStepState& js = *jobs[j];
    for (uint32_t k = node_off[j]; k < node_off[j + 1]; ++k)
      js.step_res_avail[m.node_names[node[k]]] = m.FromRow(node[k], avail[k]);
    uint32_t live_left = placed[j];
    uint32_t s = step_off[j];
    // the reference pops removed ids and scheduled steps off the front until a step blocks
    while (!js.pending_step_ids.empty()) {
      auto it = js.steps.find(js.pending_step_ids.front());
      if (it != js.steps.end()) {
        if (live_left == 0) break;
        CommonStepInCtld& x = *it->second;
        x.craned_task_map.clear();
        x.task_res_map.clear();
        x.allocated_res.clear();
        x.craned_ids.clear();
        for (uint32_t r = o_noff[s]; r < o_noff[s + 1]; ++r) {
          const CranedId& id = m.node_names[o_node[r]];
          x.craned_ids.push_back(id);
          x.allocated_res.emplace(id, m.FromRow(o_node[r], o_res[r]));
          x.craned_task_map[id];
        }
        for (uint32_t t = 0; t < nt[s]; ++t) {
          const uint32_t r = o_toff[s] + t;
          x.craned_task_map[m.node_names[o_tnode[r]]].insert(t);
          x.task_res_map[t] = m.FromRow(o_tnode[r], o_tres[r]);
        }
        x.start_time = now;
        if (scheduled_steps) (*scheduled_steps)[j].push_back(&x);
        --live_left;
        ++s;
      }
      js.pending_step_ids.pop_front();
      ++popped[j];
    }
  }
  return popped;
}

}  // namespace crane_b200
