// sched_api.cu — C-ABI of the H100 scheduling hot path (include/crane_sched.h).
//
// Host side of the drop-in boundary behind SchedulerAlgo::NodeSelect
// (reference: src/CraneCtld/JobScheduler.cpp:1141, 5543-5868). This file only
// validates, lays tables out in HBM and launches kernels; every scheduling
// decision is taken on the device (sched_kernels.cuh). There is no CPU path:
// without a CUDA device crane_sched_create() fails with CRANE_ENODEV.
//
// Built two ways:
//   nvcc -gencode arch=compute_90a,code=sm_90a    -> libcrane_sched.so (product)
//   g++ -DCRANE_EMU (tests/cuda_emu)               -> tests/_emu/libcrane_sched_emu.so
//     a kernel-emulation harness used only by the CPU-side unit tests.
#ifdef CRANE_EMU
#include "cuda_emu.h"
#else
#include <cuda_runtime.h>
#endif

#include <algorithm>
#include <mutex>
#include <cstdarg>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <string>
#include <vector>

#include "../../include/crane_sched.h"
#include "sched_kernels.cuh"
#include "commit_v2.cuh"
#include "qos_kernels.cuh"
#include "step_kernels.cuh"
#include "running_kernels.cuh"
#include "gate_kernels.cuh"
#include "step_resident_kernels.cuh"
#include "compact_kernels.cuh"

using namespace crane;

namespace {

// A device buffer that frees itself (with the handle's device current, see ~crane_sched)
template <class T>
struct DBuf {
  T* p = nullptr;
  size_t cap = 0;
  DBuf() = default;
  DBuf(const DBuf&) = delete;
  DBuf& operator=(const DBuf&) = delete;
  DBuf(DBuf&& o) noexcept { swap(o); }
  DBuf& operator=(DBuf&& o) noexcept {
    swap(o);
    return *this;
  }
  ~DBuf() {
    if (p) cudaFree(p);
  }
  cudaError_t ensure(size_t n) {
    if (n <= cap) return cudaSuccess;
    if (p) cudaFree(p);
    p = nullptr;
    cap = 0;
    size_t want = n + n / 8 + 16;
    cudaError_t e = cudaMalloc(reinterpret_cast<void**>(&p), want * sizeof(T));
    if (e == cudaSuccess) cap = want;
    return e;
  }
  // like ensure(), but the first `keep` elements survive a reallocation
  cudaError_t grow(size_t n, size_t keep, cudaStream_t st) {
    if (n <= cap) return cudaSuccess;
    T* old = p;
    size_t want = n + n / 2 + 16;
    T* q = nullptr;
    cudaError_t e = cudaMalloc(reinterpret_cast<void**>(&q), want * sizeof(T));
    if (e != cudaSuccess) return e;
    if (old && keep) {
      e = cudaMemcpyAsync(q, old, keep * sizeof(T), cudaMemcpyDeviceToDevice, st);
      if (e == cudaSuccess) e = cudaStreamSynchronize(st);
    }
    if (old) cudaFree(old);
    p = q;
    cap = want;
    return e;
  }
  void swap(DBuf& o) {
    std::swap(p, o.p);
    std::swap(cap, o.cap);
  }
  void release() {
    if (p) cudaFree(p);
    p = nullptr;
    cap = 0;
  }
};

// Each table below lists its fixed-width columns once, in each(o, f), which calls
// f(column, o's column) for every column the table has: allocation, growth and the
// gathers of crane_sched_compact and of the regroup go through that list. A table is
// replaced as a whole (std::swap): compaction builds a fresh one.

// Every fixed-width column of table `t` holds `rows` rows (their contents go)
template <class Table>
cudaError_t ensure_cols(Table& t, size_t rows) {
  cudaError_t e = cudaSuccess;
  t.each(t, [&](auto& c, auto&) { if (e == cudaSuccess) e = c.ensure(std::max<size_t>(rows, 1)); });
  return e;
}

// Every fixed-width column of table `t` grows to `rows` rows, keeping its first `keep`
template <class Table>
cudaError_t grow_cols(Table& t, size_t rows, size_t keep, cudaStream_t st) {
  cudaError_t e = cudaSuccess;
  t.each(t, [&](auto& c, auto&) { if (e == cudaSuccess) e = c.grow(rows, keep, st); });
  return e;
}

// A gather visitor: each column pair (old, new) it is given joins `cs`, for the new rows [0, rows)
inline auto gather_to(ColSet& cs, uint32_t rows) {
  return [&cs, rows](const auto& from, auto& to) {
    if (cs.n < kMaxCols) cs.col[cs.n] = ColCopy{from.p, to.p, (uint32_t)sizeof(*from.p), rows};
    cs.n++;
  };
}

// A resident table's rows keep their index until crane_sched_compact; an erased row
// stays behind as a tombstone.
struct Tombstones {
  uint32_t n = 0;  // rows, tombstones included
  uint32_t n_dead = 0;
  std::vector<uint8_t> h_dead;
  DBuf<uint8_t> d_dead;
  const uint8_t* dead() const { return n_dead ? d_dead.p : nullptr; }
  // `rows` rows, all live
  cudaError_t alloc_live(uint32_t rows, cudaStream_t st) {
    n = rows;
    n_dead = 0;
    h_dead.assign(rows, 0);
    cudaError_t e = d_dead.ensure(std::max<uint32_t>(rows, 1));
    return e == cudaSuccess ? cudaMemsetAsync(d_dead.p, 0, std::max<uint32_t>(rows, 1), st) : e;
  }
};

// The resident pending table (crane_sched_pending_append)
struct PendingTable : Tombstones {
  uint64_t total_alloc = 0;  // allocation rows of a run's placements: the sum of node_num
  // optional columns, all-or-nothing over the life of the table
  bool have_qos_cols = false, have_mandated = false, have_pd_resv = false, have_lists_incl = false,
       have_lists_excl = false;
  DBuf<uint32_t> d_partition, d_node_num, d_ntpn, d_ntpn_max, d_ntasks, d_part_prio, d_qos_prio, d_account, d_qos,
      d_user, d_pd_resv;
  DBuf<int64_t> d_time_limit, d_submit;
  DBuf<uint8_t> d_exclusive;
  DBuf<double> d_mandated;
  DBuf<View> d_req_node, d_req_task, d_req_total;
  // CSR tables: the rows' allocation slots of a run (the prefix sum of node_num), the node lists
  DBuf<uint32_t> d_alloc_off, d_incl_off, d_incl_nodes, d_excl_off, d_excl_nodes;
  // host mirrors
  std::vector<uint32_t> h_alloc_off = {0}, h_incl_off = {0}, h_excl_off = {0}, h_pd_account;

  template <class F>
  void each(PendingTable& o, F f) {
    f(d_partition, o.d_partition);
    f(d_time_limit, o.d_time_limit);
    f(d_submit, o.d_submit);
    f(d_node_num, o.d_node_num);
    f(d_ntpn, o.d_ntpn);
    f(d_ntpn_max, o.d_ntpn_max);
    f(d_ntasks, o.d_ntasks);
    f(d_exclusive, o.d_exclusive);
    f(d_part_prio, o.d_part_prio);
    f(d_qos_prio, o.d_qos_prio);
    f(d_account, o.d_account);
    f(d_req_node, o.d_req_node);
    f(d_req_task, o.d_req_task);
    f(d_req_total, o.d_req_total);
    if (have_qos_cols) {
      f(d_qos, o.d_qos);
      f(d_user, o.d_user);
    }
    if (have_mandated) f(d_mandated, o.d_mandated);
    if (have_pd_resv) f(d_pd_resv, o.d_pd_resv);
  }

  void reset() {
    n = n_dead = 0;
    total_alloc = 0;
    h_dead.clear();
    h_alloc_off.assign(1, 0);
    h_incl_off.assign(1, 0);
    h_excl_off.assign(1, 0);
    h_pd_account.clear();
  }

  PendingDev dev() const {
    PendingDev pd{};
    pd.n = n;
    pd.partition = d_partition.p;
    pd.time_limit = d_time_limit.p;
    pd.submit_time = d_submit.p;
    pd.node_num = d_node_num.p;
    pd.ntasks_per_node_min = d_ntpn.p;
    pd.ntasks_per_node_max = d_ntpn_max.p;
    pd.ntasks = d_ntasks.p;
    pd.exclusive = d_exclusive.p;
    pd.partition_priority = d_part_prio.p;
    pd.qos_priority = d_qos_prio.p;
    pd.account = d_account.p;
    pd.mandated_priority = have_mandated ? d_mandated.p : nullptr;
    pd.req_node = d_req_node.p;
    pd.req_task = d_req_task.p;
    pd.req_total = d_req_total.p;
    pd.incl_off = have_lists_incl ? d_incl_off.p : nullptr;
    pd.incl_nodes = d_incl_nodes.p;
    pd.excl_off = have_lists_excl ? d_excl_off.p : nullptr;
    pd.excl_nodes = d_excl_nodes.p;
    pd.alloc_off = d_alloc_off.p;
    pd.reservation = have_pd_resv ? d_pd_resv.p : nullptr;
    pd.dead = dead();
    return pd;
  }
};

// The gate state of the pending rows [0, n) (gate_kernels.cuh): off until a gate call
// after pending_reset
struct GateRows {
  bool on = false;
  uint32_t n = 0;
  std::vector<uint8_t> h_has_deps;  // [n] the row got its dependency list
  DBuf<uint8_t> d_g_held, d_g_is_or;
  DBuf<int64_t> d_g_begin;
  DBuf<long long> d_g_ready;
  DBuf<uint32_t> d_g_open;

  template <class F>
  void each(GateRows& o, F f) {
    f(d_g_held, o.d_g_held);
    f(d_g_begin, o.d_g_begin);
    f(d_g_is_or, o.d_g_is_or);
    f(d_g_open, o.d_g_open);
    f(d_g_ready, o.d_g_ready);
  }
};

// The dependency entries of the gate, live or retired
struct DepEntries {
  uint32_t n = 0;
  DBuf<uint32_t> d_e_dependent, d_e_dependee;
  DBuf<uint8_t> d_e_kind, d_e_type, d_e_live;
  DBuf<uint64_t> d_e_delay;

  template <class F>
  void each(DepEntries& o, F f) {
    f(d_e_dependent, o.d_e_dependent);
    f(d_e_dependee, o.d_e_dependee);
    f(d_e_kind, o.d_e_kind);
    f(d_e_type, o.d_e_type);
    f(d_e_live, o.d_e_live);
    f(d_e_delay, o.d_e_delay);
  }
};

GateDev gate_dev(GateRows& g, DepEntries& e, const uint8_t* pd_dead) {
  GateDev d{};
  d.n = g.n;
  d.dead = pd_dead;
  d.held = g.d_g_held.p;
  d.begin = g.d_g_begin.p;
  d.is_or = g.d_g_is_or.p;
  d.open = g.d_g_open.p;
  d.ready = g.d_g_ready.p;
  d.n_ent = e.n;
  d.dependent = e.d_e_dependent.p;
  d.dependee = e.d_e_dependee.p;
  d.kind = e.d_e_kind.p;
  d.type = e.d_e_type.p;
  d.live = e.d_e_live.p;
  d.delay = e.d_e_delay.p;
  return d;
}

// The fixed-width columns of running jobs: the resident table's, and the tick's dense
// view of its live rows (RunningDev)
struct RunCols {
  DBuf<int64_t> d_rr_start, d_rr_end, d_rr_cpu;
  DBuf<uint32_t> d_rr_node_num, d_rr_part_prio, d_rr_qos_prio, d_rr_account;
  DBuf<uint64_t> d_rr_mem;

  template <class F>
  void each(RunCols& o, F f) {
    f(d_rr_start, o.d_rr_start);
    f(d_rr_end, o.d_rr_end);
    f(d_rr_node_num, o.d_rr_node_num);
    f(d_rr_part_prio, o.d_rr_part_prio);
    f(d_rr_qos_prio, o.d_rr_qos_prio);
    f(d_rr_account, o.d_rr_account);
    f(d_rr_cpu, o.d_rr_cpu);
    f(d_rr_mem, o.d_rr_mem);
  }
};

// The resident running table (crane_sched_running_append, crane_sched_start)
struct RunningTable : Tombstones, RunCols {
  uint32_t node_bound = 0;  // every node index of a row is below this
  bool dirty = true;        // rows or the node-state layout changed since the last regroup
  DBuf<uint32_t> d_rr_resv;  // not in the dense view: the regroup reads it to group allocations by node state
  DBuf<uint32_t> d_rr_alloc_off, d_rr_alloc_node;  // CSR over (node, res) entries
  DBuf<Row> d_rr_alloc_res;
  // host mirrors
  std::vector<uint32_t> h_rr_alloc_off = {0}, h_rr_account;

  template <class F>
  void each(RunningTable& o, F f) {
    RunCols::each(o, f);
    f(d_rr_resv, o.d_rr_resv);
  }

  void reset() {
    n = n_dead = 0;
    h_dead.clear();
    h_rr_alloc_off.assign(1, 0);
    h_rr_account.clear();
    node_bound = 0;
    dirty = true;
  }

  RunTableDev dev() {
    RunTableDev rt{};
    rt.n = n;
    rt.start_time = d_rr_start.p;
    rt.end_time = d_rr_end.p;
    rt.node_num = d_rr_node_num.p;
    rt.partition_priority = d_rr_part_prio.p;
    rt.qos_priority = d_rr_qos_prio.p;
    rt.account = d_rr_account.p;
    rt.reservation = d_rr_resv.p;
    rt.view_cpu_raw = d_rr_cpu.p;
    rt.view_mem = d_rr_mem.p;
    rt.alloc_off = d_rr_alloc_off.p;
    rt.alloc_node = d_rr_alloc_node.p;
    rt.alloc_res = d_rr_alloc_res.p;
    rt.dead = d_dead.p;
    return rt;
  }
};

// The resident step jobs (crane_sched_step_jobs_start, _append): each job's nodes and
// one avail row per node, in a node pool. Rows keep their index; an erased row has no
// device tombstone, since every kernel reaches the rows through lists the host builds.
struct StepJobTable {
  uint32_t n = 0;
  // host mirrors
  std::vector<uint32_t> h_node_off = {0};      // [n + 1]
  std::vector<uint8_t> h_dead, h_dirty;
  std::vector<uint32_t> h_dirty_rows;          // the rows with h_dirty set
  std::vector<std::vector<uint32_t>> h_queue;  // live pending step rows of each job, row order
  DBuf<uint32_t> d_node_off, d_node;
  DBuf<Row> d_avail;

  // no fixed-width columns: a job is its CSR rows (d_node_off, d_node, d_avail)
  template <class F>
  void each(StepJobTable&, F) {}

  void mark_dirty(uint32_t j) {
    if (!h_dirty[j]) {
      h_dirty[j] = 1;
      h_dirty_rows.push_back(j);
    }
  }

  // New rows whose nodes and avail are in the pool up to off.back()
  void commit(const std::vector<uint32_t>& off) {
    for (size_t k = 0; k + 1 < off.size(); ++k) {
      h_node_off.push_back(off[k + 1]);
      h_dead.push_back(0);
      h_dirty.push_back(0);
      h_queue.emplace_back();
      mark_dirty(n++);
    }
  }

  void reset() {
    n = 0;
    h_node_off.assign(1, 0);
    h_dead.clear();
    h_dirty.clear();
    h_dirty_rows.clear();
    h_queue.clear();
  }
};

enum : uint8_t { kSpPending = 0, kSpScheduled = 1, kSpErased = 2 };

// The resident steps (crane_sched_steps_append), and the allocation pool that holds the
// node rows of the scheduled ones
struct StepTable {
  uint32_t n = 0, n_alloc = 0;  // step rows, allocation-pool rows
  // host mirrors
  std::vector<uint32_t> h_job, h_nn, h_nt, h_incl_off = {0}, h_excl_off = {0};
  std::vector<uint8_t> h_state;  // kSpPending, kSpScheduled, kSpErased
  DBuf<uint32_t> d_job, d_nn, d_nt, d_t0, d_t1, d_incl_off, d_incl, d_excl_off, d_excl, d_alloc_at;
  DBuf<View> d_req_node, d_req_task;
  DBuf<uint32_t> d_sa_node;
  DBuf<Row> d_sa_res;

  // (the list CSRs d_incl_off / d_incl, d_excl_off / d_excl and the allocation pool are not here)
  template <class F>
  void each(StepTable& o, F f) {
    f(d_job, o.d_job);
    f(d_nn, o.d_nn);
    f(d_nt, o.d_nt);
    f(d_t0, o.d_t0);
    f(d_t1, o.d_t1);
    f(d_req_node, o.d_req_node);
    f(d_req_task, o.d_req_task);
    f(d_alloc_at, o.d_alloc_at);
  }

  void reset() {
    n = n_alloc = 0;
    h_job.clear();
    h_nn.clear();
    h_nt.clear();
    h_state.clear();
    h_incl_off.assign(1, 0);
    h_excl_off.assign(1, 0);
  }
};

StepPoolDev step_pool(const StepJobTable& sj, const StepTable& sp) {
  StepPoolDev p{};
  p.sj_node_off = sj.d_node_off.p;
  p.sj_node = sj.d_node.p;
  p.sj_avail = sj.d_avail.p;
  p.job = sp.d_job.p;
  p.node_num = sp.d_nn.p;
  p.ntasks = sp.d_nt.p;
  p.ntpn_min = sp.d_t0.p;
  p.ntpn_max = sp.d_t1.p;
  p.req_node = sp.d_req_node.p;
  p.req_task = sp.d_req_task.p;
  p.incl_off = sp.d_incl_off.p;
  p.incl_nodes = sp.d_incl.p;
  p.excl_off = sp.d_excl_off.p;
  p.excl_nodes = sp.d_excl.p;
  p.alloc_at = sp.d_alloc_at.p;
  p.sa_node = sp.d_sa_node.p;
  p.sa_res = sp.d_sa_res.p;
  return p;
}

// The results of the last steps_run: its scheduled steps in ascending row order
struct StepResults {
  bool valid = false;    // steps_fetch may be called
  uint32_t sa_base = 0;  // their node rows start here in the allocation pool
  std::vector<uint32_t> h_rows, h_node_off, h_task_off;
  DBuf<uint32_t> d_u32;  // ntasks | task_node
  DBuf<Row> d_rows;      // task_res

  void clear() {
    valid = false;
    h_rows.clear();
    h_node_off.assign(1, 0);
    h_task_off.assign(1, 0);
  }
};

// Sizes buffers in turn, each to at least one element, and keeps the first error
struct Sizes {
  cudaError_t e = cudaSuccess;
  template <class T>
  void operator()(DBuf<T>& b, size_t n) {
    if (e == cudaSuccess) e = b.ensure(std::max<size_t>(n, 1));
  }
};

// The reservations of the cluster (crane_sched_set_reservations): each one's nodes,
// ascending, with the resources it holds on them
struct Reservations {
  uint32_t n = 0;
  std::vector<int64_t> start, end;
  std::vector<uint32_t> node_off = {0}, node;
  std::vector<Row> res;

  void reset() {
    n = 0;
    start.clear();
    end.clear();
    node_off.assign(1, 0);
    node.clear();
    res.clear();
  }
};

// The cluster as set_cluster and set_reservations store it, the slot layout of its node
// states that build_layout derives from it, and the device copies of both with the
// timelines. A new layout reuses the device buffers: the timelines alone hold
// n_slots x tl_cap entries.
struct ClusterLayout {
  // the inputs
  uint32_t n_nodes = 0, n_parts = 0;
  GresDict dict{};
  std::vector<Row> res_total;
  std::vector<uint8_t> alive, drain;
  std::vector<uint32_t> part_off, part_nodes;
  Reservations resv;
  uint32_t tl_cap = 0;  // timeline entries per node state: max_jobs_per_node + 1
  // the slot layout
  uint32_t n_slots = 0, max_part_slots = 0, words_per_row = 0, v2_ring = 0;
  uint32_t n_vparts = 0;  // schedulers = groups of overlapping partitions + reservations
  uint32_t n_comp = 0, max_comp_parts = 1;
  std::vector<uint32_t> h_part_comp, h_part_cidx, h_sched_nparts, h_part_base, h_slot_node, h_node_slot;
  // device copies
  DBuf<uint32_t> d_part_base, d_slot_node, d_node_slot, d_slot_resv, d_rsv_off, d_rsv_id, d_sched_nparts, d_part_comp,
      d_part_cidx, d_r_node_off, d_r_node;
  DBuf<Row> d_slot_total, d_class_rows, d_rsv_res;
  DBuf<uint8_t> d_slot_class, d_slot_memb;
  DBuf<int64_t> d_resv_start, d_resv_end;
  // the timelines
  DBuf<uint32_t> d_tl_n;
  DBuf<TlEntry> d_tl_ent;
  DBuf<Row> d_avail0;
  DBuf<double> d_cost0;
  DBuf<uint8_t> d_skip;
  DBuf<int64_t> d_first_resv;
  // per scheduler: a run's queued jobs, k_commit2's profile counters
  DBuf<uint32_t> d_part_count, d_part_job_off;
  DBuf<unsigned long long> d_prof;

  ClusterDev dev() const {
    ClusterDev cl{};
    cl.n_slots = n_slots;
    cl.n_parts = n_parts;
    cl.n_vparts = n_vparts;
    cl.n_comp = n_comp;
    cl.part_comp = d_part_comp.p;
    cl.part_cidx = d_part_cidx.p;
    cl.slot_memb = max_comp_parts > 1 ? d_slot_memb.p : nullptr;
    cl.n_resv = resv.n;
    cl.resv_start = d_resv_start.p;
    cl.resv_end = d_resv_end.p;
    cl.slot_resv = d_slot_resv.p;
    cl.rsv_off = d_rsv_off.p;
    cl.rsv_id = d_rsv_id.p;
    cl.rsv_res = d_rsv_res.p;
    cl.max_part_slots = max_part_slots;
    cl.part_base = d_part_base.p;
    cl.slot_node = d_slot_node.p;
    cl.node_slot = d_node_slot.p;
    cl.slot_total = d_slot_total.p;
    cl.slot_class = d_slot_class.p;
    cl.class_rows = d_class_rows.p;
    return cl;
  }

  TimelineDev timelines() const {
    TimelineDev tl{};
    tl.cap = tl_cap;
    tl.n = d_tl_n.p;
    tl.ent = d_tl_ent.p;
    tl.avail0 = d_avail0.p;
    tl.cost0 = d_cost0.p;
    tl.skip = d_skip.p;
    tl.first_resv = d_first_resv.p;
    return tl;
  }

  NodeStateMap node_states() const {
    return NodeStateMap{n_nodes, n_slots, n_comp, resv.n, d_node_slot.p, d_part_base.p, d_r_node_off.p, d_r_node.p};
  }
};

// The tick's view of the running table's live rows (RunningDev), built by the regroup:
// their dense columns, their allocations grouped by node state, the jobs grouped by account
struct RunView {
  uint32_t n = 0, n_accounts = 0;  // live rows, accounts (pending rows' included)
  RunCols rn;
  DBuf<uint32_t> d_slot_off, d_acc_off, d_acc_job;
  DBuf<int64_t> d_slot_end;
  DBuf<Row> d_slot_res;
  DBuf<uint64_t> d_acc_key;
  DBuf<uint8_t> d_acc_present;

  // R live rows with E allocation entries (tombstones' included), n_slots node states, A accounts
  cudaError_t ensure(uint32_t R, uint32_t E, uint32_t n_slots, uint32_t A) {
    Sizes s{ensure_cols(rn, R)};
    s(d_acc_key, R);
    s(d_acc_job, R);
    s(d_slot_off, (size_t)n_slots + 1);
    s(d_slot_end, E);
    s(d_slot_res, E);
    s(d_acc_off, (size_t)A + 1);
    s(d_acc_present, A);
    return s.e;
  }

  RunningDev dev() const {
    RunningDev d{};
    d.n = n;
    d.start_time = rn.d_rr_start.p;
    d.end_time = rn.d_rr_end.p;
    d.node_num = rn.d_rr_node_num.p;
    d.partition_priority = rn.d_rr_part_prio.p;
    d.qos_priority = rn.d_rr_qos_prio.p;
    d.account = rn.d_rr_account.p;
    d.view_cpu_raw = rn.d_rr_cpu.p;
    d.view_mem = rn.d_rr_mem.p;
    d.slot_off = d_slot_off.p;
    d.slot_end = d_slot_end.p;
    d.slot_res = d_slot_res.p;
    d.n_accounts = n_accounts;
    d.acc_off = d_acc_off.p;
    d.acc_job = d_acc_job.p;
    d.acc_present = d_acc_present.p;
    return d;
  }
};

// The last run's placements of the pending rows (PlaceDev)
struct RunOutputs {
  DBuf<uint8_t> d_reason;
  DBuf<double> d_prio;
  DBuf<int64_t> d_start, d_end;
  DBuf<uint32_t> d_nalloc, d_node, d_ntasks;  // per row | per allocation row
  DBuf<Row> d_res;

  cudaError_t ensure(size_t n_jobs, size_t n_alloc_rows) {
    Sizes s;
    s(d_reason, n_jobs);
    s(d_prio, n_jobs);
    s(d_start, n_jobs);
    s(d_end, n_jobs);
    s(d_nalloc, n_jobs);
    s(d_node, n_alloc_rows);
    s(d_ntasks, n_alloc_rows);
    s(d_res, n_alloc_rows);
    return s.e;
  }

  void release() {
    d_reason.release(); d_prio.release(); d_start.release(); d_end.release();
    d_nalloc.release(); d_node.release(); d_ntasks.release(); d_res.release();
  }

  PlaceDev dev() const {
    return PlaceDev{d_reason.p, d_prio.p, d_start.p, d_end.p, d_nalloc.p, d_node.p, d_ntasks.p, d_res.p};
  }
};

// The run's work buffers; the regroup, compaction and qos_filter sort in the priority
// sort's keys and values. release() frees every buffer sized by the tables' rows, and
// each is sized again before its next use: by ensure() in keep_running, by ensure_sort()
// in the other calls that sort, by the run (d_vpart, d_g_code) or by radix_sort (d_hist).
// d_bounds (one record) and d_acc_service (one entry per account) are not released.
struct RunWork {
  DBuf<Bounds> d_bounds;
  DBuf<double> d_acc_service, d_prio;
  DBuf<uint64_t> d_keys_a, d_keys_b;
  DBuf<uint32_t> d_vals_a, d_vals_b, d_hist, d_vpart, d_bitmap;
  DBuf<uint8_t> d_g_code;  // the run's exclusion code of every pending row (k_gate)
  DBuf<JobQ> d_jobq;

  cudaError_t ensure_sort(size_t n) {
    Sizes s;
    s(d_keys_a, n);
    s(d_keys_b, n);
    s(d_vals_a, n);
    s(d_vals_b, n);
    return s.e;
  }

  // N pending rows, sorts of n_sort keys, A accounts, nq queued jobs over bitmap rows of words_per_row
  cudaError_t ensure(uint32_t N, size_t n_sort, uint32_t A, uint32_t nq, uint32_t words_per_row) {
    Sizes s;
    s(d_bounds, 1);
    s(d_acc_service, A);
    s(d_prio, N);
    if (s.e == cudaSuccess) s.e = ensure_sort(n_sort);
    s(d_jobq, nq);
    s(d_bitmap, (size_t)std::max<uint32_t>(nq, 1) * words_per_row);
    return s.e;
  }

  void release() {
    d_keys_a.release(); d_keys_b.release(); d_vals_a.release(); d_vals_b.release(); d_hist.release();
    d_prio.release(); d_vpart.release(); d_g_code.release(); d_jobq.release(); d_bitmap.release();
  }
};

// How far a handle has got; each stage needs every earlier one. A call that replaces
// the tables of a stage lowers the handle to the stage before it.
enum Stage { kNone, kCluster, kUploaded, kRan };

// The handle's CUDA events
enum Ev {
  kEvH2dBegin, kEvH2dEnd,                                                  // crane_sched_upload
  kEvRunBegin, kEvInitEnd, kEvPrioEnd, kEvFeasEnd, kEvRunEnd, kEvD2hEnd,  // run, fetch
  kEvQosBegin, kEvQosEnd,                                                  // qos_filter
  kEvStepsBegin, kEvStepsEnd,                                              // schedule_steps
  kEvKeepBegin, kEvKeepEnd,                                                // keep_running
  kEvSpBegin, kEvSpMid, kEvSpScatter, kEvSpEnd,                            // steps_run
  kNumEv
};

// c_dicts[] slots in use, per device
std::mutex g_slot_mu;
uint32_t g_slots_used[64] = {0};

}  // namespace

struct crane_sched {
  crane_sched_config_t cfg{};
  int device = 0;
  cudaStream_t stream = nullptr;
  cudaEvent_t ev[kNumEv]{};
  std::string err;
  crane_sched_timing_t timing{};
  size_t v2_budget = 0;       // dynamic shared memory k_commit2 may use
  uint32_t n_sm = 0;          // SMs of the device: grid caps of the grid-stride kernels
  bool h2d_timed = false;     // kEvH2dBegin, kEvH2dEnd were recorded (crane_sched_upload)
  Stage stage = kNone;
  int dict_slot = -1;  // this handle's entry of c_dicts[] on its device

  ClusterLayout layout;
  // the resident tables
  PendingTable pd;
  GateRows gate;
  DepEntries ent;
  RunningTable rr;
  // the run: its view of the running table, work buffers and placements
  RunView view;
  RunWork work;
  RunOutputs outputs;
  DBuf<uint32_t> d_erase_rows, d_start_rows, d_flag;  // per call: erased rows, started rows, a device flag
  DBuf<uint32_t> d_ev_rows, d_ev_u32;  // per call: sorted rows + their positions | exit codes, offsets
  DBuf<int64_t> d_ev_i64;              // per call: end / event times, begin times
  DBuf<uint8_t> d_ev_u8;               // per call: held, is_or
  // one queue over several GPUs
  uint32_t shard_rank = 0, shard_n = 1;
  std::vector<uint32_t> h_part_owner, h_part_list;
  DBuf<uint32_t> d_part_owner, d_part_list, d_sched_owner;
  // QoS post-filter (R12)
  DBuf<uint32_t> d_q_off, d_q_u32, d_q_chain_off, d_q_chain;
  DBuf<int64_t> d_q_i64;
  DBuf<uint8_t> d_q_valid;
  DBuf<crane_tres_limit_t> d_q_tres;
  DBuf<crane_meta_resource_t> d_q_user_usage, d_q_acct_usage, d_q_qos_usage;
  // the resident step state (step_resident_kernels.cuh)
  StepJobTable sj;
  StepTable sp;
  StepResults sr;
  // per call, nothing in them outlives the call: the dense tables of a k_steps launch (u32 columns |
  // avail, alloc_res, task_res | req_node, req_task | scheduled), each entry point with its own layout
  DBuf<uint32_t> d_steps_u32;
  DBuf<Row> d_steps_rows;
  DBuf<View> d_steps_views;
  DBuf<uint8_t> d_steps_sched;
  DBuf<uint32_t> d_sp_call;  // per call: rows and offsets

  // the buffers free themselves after this, on the handle's device
  ~crane_sched() {
    cudaSetDevice(device);
    if (stream) cudaStreamSynchronize(stream);
    for (auto& e : ev)
      if (e) cudaEventDestroy(e);
    if (stream) cudaStreamDestroy(stream);
    if (dict_slot >= 0) {
      std::lock_guard<std::mutex> lk(g_slot_mu);
      g_slots_used[device] &= ~(1u << dict_slot);
    }
  }
};

namespace {

int fail(crane_sched* h, int code, const char* fmt, ...) {
  char buf[512];
  va_list ap;
  va_start(ap, fmt);
  vsnprintf(buf, sizeof buf, fmt, ap);
  va_end(ap);
  if (h) h->err = buf;
  return code;
}

#define CU(call)                                                                              \
  do {                                                                                        \
    cudaError_t e__ = (call);                                                                 \
    if (e__ != cudaSuccess)                                                                   \
      return fail(h, e__ == 2 ? CRANE_ENOMEM : CRANE_ECUDA, "%s failed: %s", #call, cudaGetErrorString(e__)); \
  } while (0)

#define TRY(call)                        \
  do {                                   \
    int rc__ = (call);                   \
    if (rc__ != CRANE_OK) return rc__;   \
  } while (0)

// "<call>: <step> first" unless the handle has reached `want`
int require(crane_sched* h, Stage want, const char* call) {
  static const char* const step[] = {"", "set_cluster", "upload", "run"};
  return h->stage >= want ? CRANE_OK : fail(h, CRANE_EINVAL, "%s: %s first", call, step[want]);
}

void lower_stage(crane_sched* h, Stage s) { h->stage = std::min(h->stage, s); }

// The offsets of a CSR table of n rows: present, off[0] == 0, non-decreasing
int check_offsets(crane_sched* h, const char* what, const uint32_t* off, uint32_t n) {
  if (!off) return fail(h, CRANE_EINVAL, "%s: null offsets", what);
  if (off[0] != 0) return fail(h, CRANE_EINVAL, "%s: offsets must start at 0", what);
  for (uint32_t i = 0; i < n; ++i)
    if (off[i + 1] < off[i]) return fail(h, CRANE_EINVAL, "%s[%u]: offsets are not monotonic", what, i);
  return CRANE_OK;
}

// An include / exclude list CSR of n rows: its offsets, and every entry a node index
// or 0xFFFFFFFF, a host the cluster does not know
int check_node_list(crane_sched* h, const char* what, const uint32_t* off, const uint32_t* nodes, uint32_t n) {
  TRY(check_offsets(h, what, off, n));
  if (off[n] && !nodes) return fail(h, CRANE_EINVAL, "%s: node list CSR without node array", what);
  for (uint32_t k = 0; k < off[n]; ++k)
    if (nodes[k] >= h->layout.n_nodes && nodes[k] != 0xFFFFFFFFu) return fail(h, CRANE_EINVAL, "%s: listed node out of range", what);
  return CRANE_OK;
}

// The rows of a crane_steps_t (crane_sched_schedule_steps, crane_sched_steps_append);
// *nrows / *trows = their node / task rows
int check_steps(crane_sched* h, const crane_steps_t* st, uint64_t* nrows, uint64_t* trows) {
  const uint32_t S = st->n;
  if (S && (!st->node_num || !st->ntasks || !st->ntasks_per_node_min || !st->ntasks_per_node_max || !st->req_node ||
            !st->req_task))
    return fail(h, CRANE_EINVAL, "steps: null column");
  *nrows = *trows = 0;
  for (uint32_t s = 0; s < S; ++s) {
    const uint32_t nn = st->node_num[s], nt = st->ntasks[s], t0 = st->ntasks_per_node_min[s], t1 = st->ntasks_per_node_max[s];
    if (nn == 0) return fail(h, CRANE_EINVAL, "steps[%u]: node_num == 0", s);
    if (nt < nn) return fail(h, CRANE_EINVAL, "steps[%u]: ntasks < node_num", s);
    if (t0 > t1) return fail(h, CRANE_EINVAL, "steps[%u]: ntasks_per_node_min > ntasks_per_node_max", s);
    if (nn >= (uint32_t)kStepHeapMax) return fail(h, CRANE_ENOSYS, "steps[%u]: node_num above %d", s, kStepHeapMax - 1);
    // (a node could then be picked for no task; the reference hands it ntasks - node_num + 1 unchecked allocations)
    if (t0 == 0) return fail(h, CRANE_ENOSYS, "steps[%u]: ntasks_per_node_min == 0", s);
    if (st->req_node[s].cpu_raw < 0 || st->req_task[s].cpu_raw < 0) return fail(h, CRANE_EINVAL, "steps[%u]: negative cpu request", s);
    *nrows += nn;
    *trows += nt;
  }
  if (*nrows > 0xfffffff0ull || *trows > 0xfffffff0ull) return fail(h, CRANE_EINVAL, "steps: too many node / task rows");
  if (st->incl_off) TRY(check_node_list(h, "steps: include list", st->incl_off, st->incl_nodes, S));
  if (st->excl_off) TRY(check_node_list(h, "steps: exclude list", st->excl_off, st->excl_nodes, S));
  return CRANE_OK;
}

float elapsed_ms(const crane_sched* h, Ev from, Ev to) {
  float ms = 0.f;
  cudaEventElapsedTime(&ms, h->ev[from], h->ev[to]);
  return ms;
}

// The phase times of the last run (its events have completed)
void read_run_times(crane_sched* h) {
  h->timing.init_ms = elapsed_ms(h, kEvRunBegin, kEvInitEnd);
  h->timing.priority_ms = elapsed_ms(h, kEvInitEnd, kEvPrioEnd);
  h->timing.feas_ms = elapsed_ms(h, kEvPrioEnd, kEvFeasEnd);
  h->timing.commit_ms = elapsed_ms(h, kEvFeasEnd, kEvRunEnd);
  h->timing.total_ms = elapsed_ms(h, kEvRunBegin, kEvRunEnd);
}

template <class T>
int h2d(crane_sched* h, DBuf<T>& dst, const T* src, size_t n) {
  CU(dst.ensure(n ? n : 1));
  if (n) CU(cudaMemcpyAsync(dst.p, src, n * sizeof(T), cudaMemcpyHostToDevice, h->stream));
  return CRANE_OK;
}
#define H2D(buf, src, n) TRY(h2d(h, buf, src, (size_t)(n)))

// stable LSD radix sort over bits [0, nbits) of d_keys_a with payload
// d_vals_a; result pointers returned in keys/vals.
int radix_sort(crane_sched* h, uint32_t n, int nbits, uint64_t** keys, uint32_t** vals) {
  uint64_t* ka = h->work.d_keys_a.p;
  uint64_t* kb = h->work.d_keys_b.p;
  uint32_t* va = h->work.d_vals_a.p;
  uint32_t* vb = h->work.d_vals_b.p;
  uint32_t nblocks = (n + kSortTile - 1) / kSortTile;
  CU(h->work.d_hist.ensure((size_t)256 * nblocks));
  for (int shift = 0; shift < nbits; shift += 8) {
    CRANE_LAUNCH(k_sort_hist, nblocks, 256, 0, h->stream, ka, n, shift, h->work.d_hist.p, nblocks);
    CRANE_LAUNCH(k_sort_scan, 1, 1024, 0, h->stream, h->work.d_hist.p, 256u * nblocks);
    CRANE_LAUNCH(k_sort_scatter, nblocks, 32, 0, h->stream, ka, va, kb, vb, n, shift, h->work.d_hist.p, nblocks);
    h->timing.kernel_launches += 3;
    std::swap(ka, kb);
    std::swap(va, vb);
  }
  *keys = ka;
  *vals = va;
  return CRANE_OK;
}

// k_cp_cols over the new rows [0, n)
int gather(crane_sched* h, const ColSet& cs, const uint32_t* live, uint32_t n) {
  if (cs.n > kMaxCols) return fail(h, CRANE_ECUDA, "gather: %u columns, more than %d", cs.n, kMaxCols);
  if (n) CRANE_LAUNCH(k_cp_cols, (n + 255) / 256, 256, 0, h->stream, cs, live, n);
  return CRANE_OK;
}

// Slot layout of the node states: the usable nodes of every partition (contiguous per
// partition), then the nodes of every reservation; device copies of the cluster tables.
int build_layout(crane_sched* h) {
  ClusterLayout& L = h->layout;
  L.h_node_slot.assign(L.n_nodes, 0xffffffffu);
  L.h_slot_node.clear();
  std::vector<Row> slot_total;
  uint32_t max_mp = 0;
  // Partitions that share a node share its NodeState (JobScheduler.cpp:5622): their job
  // loops are coupled through its timeline, so one scheduler (one CTA) takes every
  // connected component of overlapping partitions; each partition keeps its own order.
  std::vector<uint32_t> uf(L.n_parts);
  for (uint32_t p = 0; p < L.n_parts; ++p) uf[p] = p;
  auto find = [&](uint32_t x) { while (uf[x] != x) { uf[x] = uf[uf[x]]; x = uf[x]; } return x; };
  {
    std::vector<uint32_t> first(L.n_nodes, 0xffffffffu);
    for (uint32_t p = 0; p < L.n_parts; ++p) {
      uint32_t prev = 0;
      for (uint32_t k = L.part_off[p]; k < L.part_off[p + 1]; ++k) {
        const uint32_t n = L.part_nodes[k];
        if (n >= L.n_nodes) return fail(h, CRANE_EINVAL, "cluster: node index %u out of range", n);
        if (k > L.part_off[p] && n <= prev) return fail(h, CRANE_EINVAL, "cluster: partition %u node list must be ascending", p);
        prev = n;
        if (first[n] == 0xffffffffu) first[n] = p;
        else { const uint32_t a = find(first[n]), c = find(p); if (a != c) uf[std::max(a, c)] = std::min(a, c); }
      }
    }
  }
  L.h_part_comp.assign(L.n_parts, 0);
  L.h_part_cidx.assign(L.n_parts, 0);
  L.h_sched_nparts.clear();
  std::vector<std::vector<uint32_t>> comp_parts;
  {
    std::vector<uint32_t> id(L.n_parts, 0xffffffffu);
    for (uint32_t p = 0; p < L.n_parts; ++p) {
      const uint32_t r = find(p);
      if (id[r] == 0xffffffffu) { id[r] = (uint32_t)comp_parts.size(); comp_parts.emplace_back(); }
      L.h_part_comp[p] = id[r];
      L.h_part_cidx[p] = (uint32_t)comp_parts[id[r]].size();
      comp_parts[id[r]].push_back(p);
    }
  }
  L.n_comp = (uint32_t)comp_parts.size();
  L.h_part_base.assign(L.n_comp + 1, 0);
  L.h_part_base.reserve(L.n_comp + L.resv.n + 1);
  std::vector<uint8_t> slot_memb;
  uint32_t max_cp = 1;
  for (uint32_t c = 0; c < L.n_comp; ++c) {
    L.h_part_base[c] = (uint32_t)L.h_slot_node.size();
    if (comp_parts[c].size() > (size_t)kMaxCompParts)
      return fail(h, CRANE_ENOSYS, "cluster: %zu partitions overlap in one connected group (at most %d)", comp_parts[c].size(), kMaxCompParts);
    max_cp = std::max<uint32_t>(max_cp, (uint32_t)comp_parts[c].size());
    L.h_sched_nparts.push_back((uint32_t)comp_parts[c].size());
    std::vector<std::pair<uint32_t, uint8_t>> nodes;  // (node, membership bits), ascending node index
    for (uint32_t i = 0; i < comp_parts[c].size(); ++i) {
      const uint32_t p = comp_parts[c][i];
      for (uint32_t k = L.part_off[p]; k < L.part_off[p + 1]; ++k) nodes.push_back({L.part_nodes[k], (uint8_t)(1u << i)});
    }
    std::sort(nodes.begin(), nodes.end());
    for (size_t i = 0; i < nodes.size();) {
      const uint32_t n = nodes[i].first;
      uint8_t bits = 0;
      for (; i < nodes.size() && nodes[i].first == n; ++i) bits |= nodes[i].second;
      if (!L.alive[n] || L.drain[n]) continue;  // JobScheduler.cpp:5629
      const Row& t = L.res_total[n];
      if (t.cpu_raw < 0 || t.cpu_raw > (int64_t)1 << 40) return fail(h, CRANE_EINVAL, "cluster: node %u cpu out of range", n);
      for (uint32_t e = L.dict.n_entries; e < CRANE_GRES_ENTRIES; ++e)
        if (field16(t.g, e)) return fail(h, CRANE_EINVAL, "cluster: node %u has slots for an undeclared gres entry", n);
      L.h_node_slot[n] = (uint32_t)L.h_slot_node.size();
      L.h_slot_node.push_back(n);
      slot_total.push_back(t);
      slot_memb.push_back(bits);
    }
    max_mp = std::max(max_mp, (uint32_t)L.h_slot_node.size() - L.h_part_base[c]);
  }
  L.h_part_base[L.n_comp] = (uint32_t)L.h_slot_node.size();
  L.max_comp_parts = max_cp;
  const uint32_t n_phys = (uint32_t)L.h_slot_node.size();
  // one more scheduler per reservation: node states holding exactly the reserved
  // resources (JobScheduler.cpp:5689-5703), whatever the node's own state
  L.n_vparts = L.n_comp + L.resv.n;
  std::vector<uint32_t> slot_resv(n_phys, 0xffffffffu);
  for (uint32_t r = 0; r < L.resv.n; ++r) {
    for (uint32_t k = L.resv.node_off[r]; k < L.resv.node_off[r + 1]; ++k) {
      L.h_slot_node.push_back(L.resv.node[k]);
      slot_total.push_back(L.resv.res[k]);
      slot_resv.push_back(r);
      slot_memb.push_back(1);
    }
    L.h_sched_nparts.push_back(1);
    L.h_part_base.push_back((uint32_t)L.h_slot_node.size());
    max_mp = std::max(max_mp, L.resv.node_off[r + 1] - L.resv.node_off[r]);
  }
  // reservations holding resources of a partition's node, ascending reservation id
  std::vector<uint32_t> rsv_off((size_t)L.h_slot_node.size() + 1, 0), rsv_id;
  std::vector<Row> rsv_res;
  {
    std::vector<std::vector<std::pair<uint32_t, uint32_t>>> per(n_phys);
    for (uint32_t r = 0; r < L.resv.n; ++r)
      for (uint32_t k = L.resv.node_off[r]; k < L.resv.node_off[r + 1]; ++k) {
        const uint32_t g = L.h_node_slot[L.resv.node[k]];
        if (g != 0xffffffffu) per[g].push_back({r, k});  // (nodes outside node_state_map are skipped, :5680)
      }
    for (uint32_t g = 0; g < n_phys; ++g) {
      for (auto& e : per[g]) { rsv_id.push_back(e.first); rsv_res.push_back(L.resv.res[e.second]); }
      rsv_off[g + 1] = (uint32_t)rsv_id.size();
    }
    for (size_t g = n_phys; g < L.h_slot_node.size(); ++g) rsv_off[g + 1] = (uint32_t)rsv_id.size();
  }
  L.n_slots = (uint32_t)L.h_slot_node.size();
  L.max_part_slots = max_mp;
  L.words_per_row = std::max<uint32_t>(4, ((max_mp + 31) / 32 + 3) / 4 * 4);  // 16-byte rows for the bulk copies
  L.v2_ring = commit2_ring_slots(max_mp, L.words_per_row, L.dict.n_entries > 0, h->v2_budget, L.max_comp_parts);
  if (max_mp > 65000 || L.v2_ring == 0)
    return fail(h, CRANE_ENOSYS, "cluster: partition with %u usable nodes exceeds the per-SM state budget", max_mp);
  // res_total classes per partition (distinct rows), cached in shared memory by the commit kernel
  std::vector<uint8_t> slot_class(std::max<size_t>(slot_total.size(), 1), 0xff);
  std::vector<Row> class_rows((size_t)std::max<uint32_t>(L.n_vparts, 1) * kMaxClasses);
  memset(class_rows.data(), 0, class_rows.size() * sizeof(Row));
  for (uint32_t p = 0; p < L.n_vparts; ++p) {
    uint32_t ncls = 0;
    for (uint32_t g = L.h_part_base[p]; g < L.h_part_base[p + 1]; ++g) {
      uint32_t k = 0;
      for (; k < ncls; ++k)
        if (memcmp(&class_rows[(size_t)p * kMaxClasses + k], &slot_total[g], sizeof(Row)) == 0) break;
      if (k == ncls) {
        if (ncls == (uint32_t)kMaxClasses) continue;  // no class: the kernel reads slot_total
        class_rows[(size_t)p * kMaxClasses + ncls++] = slot_total[g];
      }
      slot_class[g] = (uint8_t)k;
    }
  }

  H2D(L.d_part_base, L.h_part_base.data(), L.h_part_base.size());
  H2D(L.d_slot_node, L.h_slot_node.data(), L.h_slot_node.size());
  H2D(L.d_node_slot, L.h_node_slot.data(), L.h_node_slot.size());
  H2D(L.d_slot_total, slot_total.data(), slot_total.size());
  H2D(L.d_slot_class, slot_class.data(), slot_class.size());
  H2D(L.d_class_rows, class_rows.data(), class_rows.size());
  H2D(L.d_slot_resv, slot_resv.data(), slot_resv.size());
  H2D(L.d_slot_memb, slot_memb.data(), slot_memb.size());
  H2D(L.d_sched_nparts, L.h_sched_nparts.data(), L.h_sched_nparts.size());
  H2D(L.d_part_comp, L.h_part_comp.data(), L.h_part_comp.size());
  H2D(L.d_part_cidx, L.h_part_cidx.data(), L.h_part_cidx.size());
  H2D(L.d_rsv_off, rsv_off.data(), rsv_off.size());
  H2D(L.d_rsv_id, rsv_id.data(), rsv_id.size());
  H2D(L.d_rsv_res, rsv_res.data(), rsv_res.size());
  H2D(L.d_resv_start, L.resv.start.data(), L.resv.start.size());
  H2D(L.d_resv_end, L.resv.end.data(), L.resv.end.size());
  H2D(L.d_r_node_off, L.resv.node_off.data(), L.resv.node_off.size());
  H2D(L.d_r_node, L.resv.node.data(), L.resv.node.size());
  CU(cudaMemcpyToSymbolAsync(c_dicts, &L.dict, sizeof(GresDict), (size_t)h->dict_slot * sizeof(GresDict), cudaMemcpyHostToDevice, h->stream));
  size_t ns = std::max<uint32_t>(L.n_slots, 1);
  CU(L.d_tl_n.ensure(ns));
  CU(L.d_tl_ent.ensure(ns * L.tl_cap));
  CU(L.d_avail0.ensure(ns));
  CU(L.d_cost0.ensure(ns));
  CU(L.d_skip.ensure(ns));
  CU(L.d_first_resv.ensure(ns));
  CU(L.d_part_count.ensure(L.n_vparts + 2));
  CU(L.d_part_job_off.ensure(L.n_vparts + 2));
  CU(L.d_prof.ensure((size_t)L.n_vparts * 16));
  CU(cudaStreamSynchronize(h->stream));
  h->stage = kCluster;
  h->rr.dirty = true;  // the running view is grouped by node state
  h->shard_rank = 0;
  h->shard_n = 1;  // a new cluster: the partition -> rank table has to be set again
  return CRANE_OK;
}

template <class T>
int h2d_at(crane_sched* h, DBuf<T>& dst, const T* src, size_t base, size_t n) {
  CU(dst.grow(std::max<size_t>(base + n, 1), base, h->stream));
  if (n) CU(cudaMemcpyAsync(dst.p + base, src, n * sizeof(T), cudaMemcpyHostToDevice, h->stream));
  return CRANE_OK;
}
#define H2D_AT(buf, src, base, n) TRY(h2d_at(h, buf, src, (size_t)(base), (size_t)(n)))

// Appends the rows of `pd` to the device-resident pending table (rows keep job-id
// order: the reference's pending map is a btree over job ids, JobScheduler.cpp:1092).
int pending_append(crane_sched* h, const crane_pending_t* pd) {
  const uint32_t base = h->pd.n, N = pd->n;
  if (N && (!pd->partition || !pd->time_limit || !pd->submit_time || !pd->node_num || !pd->ntasks ||
            !pd->ntasks_per_node_min || !pd->ntasks_per_node_max || !pd->exclusive || !pd->partition_priority ||
            !pd->qos_priority || !pd->account || !pd->req_node || !pd->req_task || !pd->req_total))
    return fail(h, CRANE_EINVAL, "pending: null column");
  if ((uint64_t)base + N > 0xfffffff0ull) return fail(h, CRANE_EINVAL, "pending: too many rows");
  // optional columns are all-or-nothing over the life of the table
  if (base) {
    if ((pd->qos != nullptr && pd->user != nullptr) != h->pd.have_qos_cols || (pd->mandated_priority != nullptr) != h->pd.have_mandated ||
        (pd->reservation != nullptr) != h->pd.have_pd_resv || (pd->incl_off != nullptr) != h->pd.have_lists_incl ||
        (pd->excl_off != nullptr) != h->pd.have_lists_excl)
      return fail(h, CRANE_EINVAL, "pending_append: optional columns (qos/user, mandated_priority, reservation, node lists) must match the table's");
  } else {
    h->pd.reset();
    h->pd.have_qos_cols = pd->qos != nullptr && pd->user != nullptr;
    h->pd.have_mandated = pd->mandated_priority != nullptr;
    h->pd.have_pd_resv = pd->reservation != nullptr;
    h->pd.have_lists_incl = pd->incl_off != nullptr;
    h->pd.have_lists_excl = pd->excl_off != nullptr;
  }
  // ---- validation + alloc_off (prefix sum of node_num over all rows) -----------
  uint64_t acc = h->pd.h_alloc_off.back();
  for (uint32_t i = 0; i < N; ++i) {
    if (pd->node_num[i] == 0) return fail(h, CRANE_EINVAL, "pending[%u]: node_num == 0", i);
    if (pd->time_limit[i] < 1) return fail(h, CRANE_EINVAL, "pending[%u]: time_limit < 1", i);
    const uint32_t t = pd->ntasks_per_node_min[i], tmax = pd->ntasks_per_node_max[i];
    if (t == 0 || tmax < t) return fail(h, CRANE_EINVAL, "pending[%u]: ntasks_per_node_min/max", i);
    // general task distribution (the top-K heaps of JobScheduler.cpp:5193-5205): heaps of up to 127 nodes
    if ((tmax != t || (uint64_t)t * pd->node_num[i] != pd->ntasks[i]) && pd->node_num[i] >= (uint32_t)kHeapMax)
      return fail(h, CRANE_ENOSYS, "pending[%u]: a job with a ntasks_per_node range wider than %d nodes", i, kHeapMax - 1);
    if ((uint64_t)tmax * pd->node_num[i] < pd->ntasks[i] || (uint64_t)t * pd->node_num[i] > pd->ntasks[i])
      return fail(h, CRANE_EINVAL, "pending[%u]: ntasks outside [node_num*ntpn_min, node_num*ntpn_max]", i);
    if (pd->req_node[i].cpu_raw < 0 || pd->req_task[i].cpu_raw < 0)
      return fail(h, CRANE_EINVAL, "pending[%u]: negative cpu request", i);
    if (pd->account[i] > (1u << 24)) return fail(h, CRANE_EINVAL, "account ids must be dense (< 2^24)");
    acc += pd->node_num[i];
    if (acc > 0xfffffff0ull) return fail(h, CRANE_EINVAL, "pending: sum(node_num) overflows");
  }
  if (pd->incl_off) TRY(check_node_list(h, "pending: include list", pd->incl_off, pd->incl_nodes, N));
  if (pd->excl_off) TRY(check_node_list(h, "pending: exclude list", pd->excl_off, pd->excl_nodes, N));
  // ---- columns ----------------------------------------------------------------
  H2D_AT(h->pd.d_partition, pd->partition, base, N);
  H2D_AT(h->pd.d_time_limit, pd->time_limit, base, N);
  H2D_AT(h->pd.d_submit, pd->submit_time, base, N);
  H2D_AT(h->pd.d_node_num, pd->node_num, base, N);
  H2D_AT(h->pd.d_ntpn, pd->ntasks_per_node_min, base, N);
  H2D_AT(h->pd.d_ntpn_max, pd->ntasks_per_node_max, base, N);
  H2D_AT(h->pd.d_ntasks, pd->ntasks, base, N);
  H2D_AT(h->pd.d_exclusive, pd->exclusive, base, N);
  H2D_AT(h->pd.d_part_prio, pd->partition_priority, base, N);
  H2D_AT(h->pd.d_qos_prio, pd->qos_priority, base, N);
  H2D_AT(h->pd.d_account, pd->account, base, N);
  if (h->pd.have_qos_cols) {
    H2D_AT(h->pd.d_qos, pd->qos, base, N);
    H2D_AT(h->pd.d_user, pd->user, base, N);
  }
  if (h->pd.have_mandated) H2D_AT(h->pd.d_mandated, pd->mandated_priority, base, N);
  H2D_AT(h->pd.d_req_node, reinterpret_cast<const View*>(pd->req_node), base, N);
  H2D_AT(h->pd.d_req_task, reinterpret_cast<const View*>(pd->req_task), base, N);
  H2D_AT(h->pd.d_req_total, reinterpret_cast<const View*>(pd->req_total), base, N);
  if (h->pd.have_pd_resv) H2D_AT(h->pd.d_pd_resv, pd->reservation, base, N);
  {
    std::vector<uint8_t> zeros(N, 0);
    H2D_AT(h->pd.d_dead, zeros.data(), base, N);
    CU(cudaStreamSynchronize(h->stream));
  }
  // host mirrors
  for (uint32_t i = 0; i < N; ++i) {
    h->pd.h_alloc_off.push_back(h->pd.h_alloc_off.back() + pd->node_num[i]);
    h->pd.h_pd_account.push_back(pd->account[i]);
    h->pd.h_dead.push_back(0);
  }
  H2D_AT(h->pd.d_alloc_off, h->pd.h_alloc_off.data() + base, base, (size_t)N + 1);
  if (h->pd.have_lists_incl) {
    const uint32_t nb = h->pd.h_incl_off.back();
    for (uint32_t i = 0; i < N; ++i) h->pd.h_incl_off.push_back(nb + pd->incl_off[i + 1]);
    H2D_AT(h->pd.d_incl_off, h->pd.h_incl_off.data() + base, base, (size_t)N + 1);
    H2D_AT(h->pd.d_incl_nodes, pd->incl_nodes, nb, pd->incl_off[N]);
  }
  if (h->pd.have_lists_excl) {
    const uint32_t nb = h->pd.h_excl_off.back();
    for (uint32_t i = 0; i < N; ++i) h->pd.h_excl_off.push_back(nb + pd->excl_off[i + 1]);
    H2D_AT(h->pd.d_excl_off, h->pd.h_excl_off.data() + base, base, (size_t)N + 1);
    H2D_AT(h->pd.d_excl_nodes, pd->excl_nodes, nb, pd->excl_off[N]);
  }
  CU(cudaStreamSynchronize(h->stream));
  h->pd.n = base + N;
  h->pd.total_alloc = h->pd.h_alloc_off.back();
  return CRANE_OK;
}

// The rows of a host running table: the checks of crane_sched_running_append (`replace`:
// the rows will replace the table rather than extend it)
int running_check(crane_sched* h, const crane_running_t* rn, bool replace) {
  const uint32_t R = rn ? rn->n : 0;
  if (!R) return CRANE_OK;
  if (!rn->start_time || !rn->end_time || !rn->node_num || !rn->partition_priority || !rn->qos_priority ||
      !rn->account || !rn->view_cpu_raw || !rn->view_mem)
    return fail(h, CRANE_EINVAL, "running: null column");
  TRY(check_offsets(h, "running: alloc_off", rn->alloc_off, R));
  const uint32_t E = rn->alloc_off[R];
  if (E && (!rn->alloc_node || !rn->alloc_res)) return fail(h, CRANE_EINVAL, "running: null allocation table");
  const uint64_t rows = replace ? 0 : h->rr.n, entries = replace ? 0 : h->rr.h_rr_alloc_off.back();
  if (rows + R > 0xfffffff0ull || entries + E > 0xfffffff0ull)
    return fail(h, CRANE_EINVAL, "running: too many rows");
  for (uint32_t j = 0; j < R; ++j) {
    if (rn->account[j] > (1u << 24)) return fail(h, CRANE_EINVAL, "account ids must be dense (< 2^24)");
    for (uint32_t k = rn->alloc_off[j]; k < rn->alloc_off[j + 1]; ++k)
      if (rn->alloc_node[k] >= h->layout.n_nodes) return fail(h, CRANE_EINVAL, "running[%u]: node out of range", j);
  }
  return CRANE_OK;
}

// Appends the rows of a checked host running table to the resident table
int running_append(crane_sched* h, const crane_running_t* rn) {
  const uint32_t base = h->rr.n, R = rn ? rn->n : 0;
  if (!R) return CRANE_OK;
  const uint32_t eb = h->rr.h_rr_alloc_off.back(), E = rn->alloc_off[R];
  H2D_AT(h->rr.d_rr_start, rn->start_time, base, R);
  H2D_AT(h->rr.d_rr_end, rn->end_time, base, R);
  H2D_AT(h->rr.d_rr_node_num, rn->node_num, base, R);
  H2D_AT(h->rr.d_rr_part_prio, rn->partition_priority, base, R);
  H2D_AT(h->rr.d_rr_qos_prio, rn->qos_priority, base, R);
  H2D_AT(h->rr.d_rr_account, rn->account, base, R);
  H2D_AT(h->rr.d_rr_cpu, rn->view_cpu_raw, base, R);
  H2D_AT(h->rr.d_rr_mem, rn->view_mem, base, R);
  std::vector<uint32_t> no_resv(rn->reservation ? 0 : R, 0xffffffffu);
  H2D_AT(h->rr.d_rr_resv, rn->reservation ? rn->reservation : no_resv.data(), base, R);
  std::vector<uint8_t> zeros(R, 0);
  H2D_AT(h->rr.d_dead, zeros.data(), base, R);
  for (uint32_t j = 0; j < R; ++j) {
    h->rr.h_rr_alloc_off.push_back(eb + rn->alloc_off[j + 1]);
    h->rr.h_rr_account.push_back(rn->account[j]);
    h->rr.h_dead.push_back(0);
  }
  H2D_AT(h->rr.d_rr_alloc_off, h->rr.h_rr_alloc_off.data() + base, base, (size_t)R + 1);
  H2D_AT(h->rr.d_rr_alloc_node, rn->alloc_node, eb, E);
  H2D_AT(h->rr.d_rr_alloc_res, reinterpret_cast<const Row*>(rn->alloc_res), eb, E);
  for (uint32_t k = 0; k < E; ++k) h->rr.node_bound = std::max(h->rr.node_bound, rn->alloc_node[k] + 1);
  CU(cudaStreamSynchronize(h->stream));  // (the staging vectors are pageable)
  h->rr.n = base + R;
  h->rr.dirty = true;
  return CRANE_OK;
}

// The tick's RunningDev view of the live rows, on the device: the dense per-job columns
// (live rows in row order), the allocations grouped by node state and the jobs grouped by
// account, both stable (order inside a node state / account is row order, deviation D6).
int regroup(crane_sched* h, uint32_t R, uint32_t max_rn_account) {
  cudaStream_t st = h->stream;
  const uint32_t Rt = h->rr.n, E = h->rr.h_rr_alloc_off.back();
  const RunTableDev rt = h->rr.dev();
  const ClusterLayout& L = h->layout;
  RunView& v = h->view;
  CU(h->d_flag.ensure(1));
  CU(cudaMemsetAsync(h->d_flag.p, 0, sizeof(uint32_t), st));
  uint64_t* keys;
  uint32_t* vals;
  // live rows in row order -> the dense columns (without tombstones: every row, in order)
  if (R) {
    vals = nullptr;
    if (h->rr.n_dead) {
      CRANE_LAUNCH(k_rt_live_keys, (Rt + 255) / 256, 256, 0, st, rt.dead, Rt, h->work.d_keys_a.p, h->work.d_vals_a.p);
      TRY(radix_sort(h, Rt, 8, &keys, &vals));
    }
    ColSet cs{};
    h->rr.RunCols::each(v.rn, gather_to(cs, R));
    TRY(gather(h, cs, vals, R));
  }
  // allocations by node state: stable sort of the entries (row order) by slot
  if (E) {
    const uint32_t nb = std::min<uint32_t>((Rt + 7) / 8, 8 * h->n_sm);
    CRANE_LAUNCH(k_rt_entry_keys, nb, 256, 0, st, rt, L.node_states(), h->work.d_keys_a.p, h->work.d_vals_a.p, h->d_flag.p);
    int bits = 8;
    while ((1ull << bits) <= (uint64_t)L.n_slots) bits += 8;
    TRY(radix_sort(h, E, bits, &keys, &vals));
    CRANE_LAUNCH(k_rt_offsets, (L.n_slots + 1 + 255) / 256, 256, 0, st, keys, E, L.n_slots, v.d_slot_off.p);
    CRANE_LAUNCH(k_rt_slot_gather, (E + 255) / 256, 256, 0, st, rt, keys, vals, E, v.d_slot_off.p + L.n_slots,
                 v.d_slot_end.p, v.d_slot_res.p);
  } else {
    CU(cudaMemsetAsync(v.d_slot_off.p, 0, sizeof(uint32_t) * ((size_t)L.n_slots + 1), st));
  }
  // jobs by account: stable sort of the view's jobs by account
  if (R) {
    CRANE_LAUNCH(k_rt_acc_keys, (R + 255) / 256, 256, 0, st, v.rn.d_rr_account.p, R, h->work.d_keys_a.p, h->work.d_vals_a.p);
    int bits = 8;
    while ((1ull << bits) <= (uint64_t)max_rn_account) bits += 8;
    TRY(radix_sort(h, R, bits, &keys, &vals));
    CU(cudaMemcpyAsync(v.d_acc_key.p, keys, sizeof(uint64_t) * R, cudaMemcpyDeviceToDevice, st));
    CU(cudaMemcpyAsync(v.d_acc_job.p, vals, sizeof(uint32_t) * R, cudaMemcpyDeviceToDevice, st));
  }
  CU(cudaGetLastError());
  // a cluster with fewer nodes than the rows name: one flag read back
  if (E && h->rr.node_bound > L.n_nodes) {
    uint32_t bad = 0;
    CU(cudaMemcpyAsync(&bad, h->d_flag.p, sizeof(uint32_t), cudaMemcpyDeviceToHost, st));
    CU(cudaStreamSynchronize(st));
    if (bad) return fail(h, CRANE_EINVAL, "running: node out of range");
  }
  h->rr.dirty = false;
  return CRANE_OK;
}

// "The next run uses the running table as it stands on the device": the view of the
// live rows (regrouped when the rows or the node-state layout changed) and the work and
// output buffers for the resident pending table.
int keep_running(crane_sched* h) {
  cudaStream_t st = h->stream;
  const uint32_t N = h->pd.n, Rt = h->rr.n, R = Rt - h->rr.n_dead;
  const uint32_t E = h->rr.h_rr_alloc_off.back();
  uint32_t max_rn_account = 0, max_account = 0;
  for (uint32_t r = 0; r < Rt; ++r)
    if (!h->rr.h_dead[r]) max_rn_account = std::max(max_rn_account, h->rr.h_rr_account[r]);
  for (uint32_t i = 0; i < N; ++i) max_account = std::max(max_account, h->pd.h_pd_account[i]);
  max_account = std::max(max_account, max_rn_account);
  const uint32_t A = (N + R) ? max_account + 1 : 0;

  const uint32_t nq = std::min<uint32_t>(N, h->cfg.scheduled_batch_size);
  CU(h->view.ensure(R, E, h->layout.n_slots, A));
  CU(h->work.ensure(N, std::max<size_t>({(size_t)N, (size_t)Rt, (size_t)E}), A, nq, h->layout.words_per_row));
  CU(h->outputs.ensure(N, h->pd.total_alloc));

  CU(cudaEventRecord(h->ev[kEvKeepBegin], st));
  if (h->rr.dirty) TRY(regroup(h, R, max_rn_account));
  // ---- accounts: offsets of the account groups, accounts present (pending included) ----
  RunView& v = h->view;
  CRANE_LAUNCH(k_rt_offsets, (A + 1 + 255) / 256, 256, 0, st, v.d_acc_key.p, R, A, v.d_acc_off.p);
  CU(cudaMemsetAsync(v.d_acc_present.p, 0, std::max<uint32_t>(A, 1), st));
  if (N + R)
    CRANE_LAUNCH(k_acc_present, (N + R + 255) / 256, 256, 0, st, h->pd.d_account.p, h->pd.n_dead ? h->pd.d_dead.p : nullptr, N,
                 v.rn.d_rr_account.p, R, v.d_acc_present.p);
  CU(cudaEventRecord(h->ev[kEvKeepEnd], st));
  CU(cudaGetLastError());
  v.n = R;
  v.n_accounts = A;
  return CRANE_OK;
}

// The running table of this tick from a host table: reset + append + keep_running
int set_running(crane_sched* h, const crane_running_t* rn) {
  TRY(running_check(h, rn, true));
  h->rr.reset();
  TRY(running_append(h, rn));
  return keep_running(h);
}

GateDev gate_dev(crane_sched* h) { return gate_dev(h->gate, h->ent, h->pd.dead()); }

// Turns the gate on and gives the rows appended since the last gate call their state:
// not held, beginning at InfinitePast, no dependencies
int gate_fit(crane_sched* h) {
  h->gate.on = true;
  const uint32_t from = h->gate.n, to = h->pd.n;
  if (to <= from) return CRANE_OK;
  cudaStream_t st = h->stream;
  CU(grow_cols(h->gate, to, from, st));
  h->gate.n = to;
  h->gate.h_has_deps.resize(to, 0);
  CRANE_LAUNCH(k_gate_init, (to - from + 255) / 256, 256, 0, st, gate_dev(h), from, to);
  CU(cudaGetLastError());
  return CRANE_OK;
}

// The rows of an erase / start / read call: in [0, n_rows), not erased, none listed twice
template <class Erased>
int check_rows(crane_sched* h, const char* call, const uint32_t* rows, uint32_t n, uint32_t n_rows, Erased erased) {
  if (n && !rows) return fail(h, CRANE_EINVAL, "%s: null rows", call);
  std::vector<uint32_t> sorted(rows, rows + n);
  std::sort(sorted.begin(), sorted.end());
  for (uint32_t k = 0; k < n; ++k) {
    if (sorted[k] >= n_rows) return fail(h, CRANE_EINVAL, "%s: row %u out of range", call, sorted[k]);
    if (erased(sorted[k])) return fail(h, CRANE_EINVAL, "%s: row %u was erased", call, sorted[k]);
    if (k && sorted[k] == sorted[k - 1]) return fail(h, CRANE_EINVAL, "%s: row %u listed twice", call, sorted[k]);
  }
  return CRANE_OK;
}

// Erases rows of a table: rows out of range fail, rows already erased and rows listed twice do not
int erase_rows(crane_sched* h, const char* call, Tombstones& t, const uint32_t* rows, uint32_t n) {
  if (n && !rows) return CRANE_EINVAL;
  CU(cudaSetDevice(h->device));
  for (uint32_t k = 0; k < n; ++k)
    if (rows[k] >= t.n) return fail(h, CRANE_EINVAL, "%s: row %u out of range", call, rows[k]);
  lower_stage(h, kCluster);
  if (!n) return CRANE_OK;
  for (uint32_t k = 0; k < n; ++k)
    if (!t.h_dead[rows[k]]) { t.h_dead[rows[k]] = 1; t.n_dead++; }
  H2D(h->d_erase_rows, rows, n);
  CRANE_LAUNCH(k_mark_dead, (n + 255) / 256, 256, 0, h->stream, h->d_erase_rows.p, n, t.d_dead.p);
  CU(cudaGetLastError());
  CU(cudaStreamSynchronize(h->stream));
  return CRANE_OK;
}

// The rows of a call on the device, sorted, followed by their places in the call's list
int upload_call_rows(crane_sched* h, const uint32_t* rows, uint32_t n) {
  std::vector<uint32_t> idx(n), buf(2 * (size_t)n);
  for (uint32_t k = 0; k < n; ++k) idx[k] = k;
  std::stable_sort(idx.begin(), idx.end(), [&](uint32_t a, uint32_t b) { return rows[a] < rows[b]; });
  for (uint32_t k = 0; k < n; ++k) {
    buf[k] = rows[idx[k]];
    buf[n + k] = idx[k];
  }
  H2D(h->d_ev_rows, buf.data(), buf.size());
  CU(cudaStreamSynchronize(h->stream));  // (buf is pageable)
  return CRANE_OK;
}

// k_dep_fire over `threads` entries for the events of the call whose rows upload_call_rows placed
int dep_fire(crane_sched* h, DepEvents ev, uint32_t n_rows, uint32_t threads) {
  if (!threads) return CRANE_OK;
  ev.n = n_rows;
  ev.rows = h->d_ev_rows.p;
  ev.pos = h->d_ev_rows.p + n_rows;
  CRANE_LAUNCH(k_dep_fire, (threads + 255) / 256, 256, 0, h->stream, gate_dev(h), ev);
  CU(cudaGetLastError());
  return CRANE_OK;
}

// The live rows of a table of n rows, in row order (the stable sort by tombstone flag),
// into live[0, n_live), and the old -> new map into map[0, n)
int live_rows(crane_sched* h, const uint8_t* dead, uint32_t n, uint32_t n_live, uint32_t* live, uint32_t* map) {
  cudaStream_t st = h->stream;
  uint64_t* keys;
  uint32_t* vals;
  CRANE_LAUNCH(k_rt_live_keys, (n + 255) / 256, 256, 0, st, dead, n, h->work.d_keys_a.p, h->work.d_vals_a.p);
  TRY(radix_sort(h, n, 8, &keys, &vals));
  if (n_live) CU(cudaMemcpyAsync(live, vals, sizeof(uint32_t) * n_live, cudaMemcpyDeviceToDevice, st));
  CU(cudaMemsetAsync(map, 0xff, sizeof(uint32_t) * n, st));
  if (n_live) CRANE_LAUNCH(k_cp_map, (n_live + 255) / 256, 256, 0, st, live, n_live, map);
  return CRANE_OK;
}

// new_off[0, n_live] = the offsets of the live rows of a CSR table
int csr_offsets(crane_sched* h, const uint32_t* off, const uint32_t* live, uint32_t n_live, uint32_t* new_off) {
  CRANE_LAUNCH(k_cp_lengths, (n_live + 1 + 255) / 256, 256, 0, h->stream, off, live, n_live, new_off);
  CRANE_LAUNCH(k_sort_scan, 1, 1024, 0, h->stream, new_off, n_live + 1);
  return CRANE_OK;
}

// The entries of the live rows of a CSR table at their new offsets
template <class T>
int csr_copy(crane_sched* h, const uint32_t* off, const T* src, const uint32_t* live, uint32_t n_live,
             const uint32_t* new_off, T* dst) {
  if (!n_live) return CRANE_OK;
  const uint32_t nb = std::min<uint32_t>((n_live + 7) / 8, 8 * h->n_sm);
  CRANE_LAUNCH(k_cp_csr<T>, nb, 256, 0, h->stream, off, src, live, n_live, new_off, dst);
  return CRANE_OK;
}

// Host mirror of a CSR table's offsets for its live rows
std::vector<uint32_t> live_offsets(const std::vector<uint32_t>& off, const std::vector<uint8_t>& dead) {
  std::vector<uint32_t> o(1, 0);
  for (size_t r = 0; r < dead.size(); ++r)
    if (!dead[r]) o.push_back(o.back() + (off[r + 1] - off[r]));
  return o;
}

template <class T>
std::vector<T> live_only(const std::vector<T>& v, const std::vector<uint8_t>& dead) {
  std::vector<T> o;
  for (size_t r = 0; r < dead.size(); ++r)
    if (!dead[r]) o.push_back(v[r]);
  return o;
}

// The compacted pending table and gate: the host state of the live rows of the handle's,
// no tombstones, the other device buffers allocated for pending_copy
int pending_fresh(crane_sched* h, PendingTable& pd, GateRows& g) {
  const PendingTable& o = h->pd;
  pd.have_qos_cols = o.have_qos_cols;
  pd.have_mandated = o.have_mandated;
  pd.have_pd_resv = o.have_pd_resv;
  pd.have_lists_incl = o.have_lists_incl;
  pd.have_lists_excl = o.have_lists_excl;
  pd.h_alloc_off = live_offsets(o.h_alloc_off, o.h_dead);
  if (o.have_lists_incl) pd.h_incl_off = live_offsets(o.h_incl_off, o.h_dead);
  if (o.have_lists_excl) pd.h_excl_off = live_offsets(o.h_excl_off, o.h_dead);
  pd.h_pd_account = live_only(o.h_pd_account, o.h_dead);
  pd.total_alloc = pd.h_alloc_off.back();
  const uint32_t n = o.n - o.n_dead, n1 = std::max<uint32_t>(n, 1);
  CU(pd.alloc_live(n, h->stream));
  CU(ensure_cols(pd, n));
  CU(pd.d_alloc_off.ensure(n1 + 1));
  if (pd.have_lists_incl) {
    CU(pd.d_incl_off.ensure(n1 + 1));
    CU(pd.d_incl_nodes.ensure(std::max<uint32_t>(pd.h_incl_off.back(), 1)));
  }
  if (pd.have_lists_excl) {
    CU(pd.d_excl_off.ensure(n1 + 1));
    CU(pd.d_excl_nodes.ensure(std::max<uint32_t>(pd.h_excl_off.back(), 1)));
  }
  // the gate state of the live rows below the gate's end
  g.on = h->gate.on;
  g.h_has_deps = live_only(h->gate.h_has_deps, std::vector<uint8_t>(o.h_dead.begin(), o.h_dead.begin() + h->gate.n));
  g.n = (uint32_t)g.h_has_deps.size();
  if (h->gate.n) CU(ensure_cols(g, g.n));
  return CRANE_OK;
}

// The live rows of the handle's pending table and gate into the fresh ones (one gather)
int pending_copy(crane_sched* h, PendingTable& pd, GateRows& g, const uint32_t* live) {
  PendingTable& o = h->pd;
  ColSet cs{};
  o.each(pd, gather_to(cs, pd.n));
  h->gate.each(g, gather_to(cs, g.n));
  TRY(gather(h, cs, live, pd.n));
  TRY(csr_offsets(h, o.d_alloc_off.p, live, pd.n, pd.d_alloc_off.p));
  if (pd.have_lists_incl) {
    TRY(csr_offsets(h, o.d_incl_off.p, live, pd.n, pd.d_incl_off.p));
    TRY(csr_copy(h, o.d_incl_off.p, o.d_incl_nodes.p, live, pd.n, pd.d_incl_off.p, pd.d_incl_nodes.p));
  }
  if (pd.have_lists_excl) {
    TRY(csr_offsets(h, o.d_excl_off.p, live, pd.n, pd.d_excl_off.p));
    TRY(csr_copy(h, o.d_excl_off.p, o.d_excl_nodes.p, live, pd.n, pd.d_excl_off.p, pd.d_excl_nodes.p));
  }
  return CRANE_OK;
}

// The compacted running table: the host state of the live rows of the handle's, no
// tombstones, the other device buffers allocated for running_copy
int running_fresh(crane_sched* h, RunningTable& rr) {
  const RunningTable& o = h->rr;
  rr.node_bound = o.node_bound;
  rr.dirty = o.dirty;  // (the run's view of the running table is the live rows in row order)
  rr.h_rr_alloc_off = live_offsets(o.h_rr_alloc_off, o.h_dead);
  rr.h_rr_account = live_only(o.h_rr_account, o.h_dead);
  const uint32_t n = o.n - o.n_dead, e1 = std::max<uint32_t>(rr.h_rr_alloc_off.back(), 1);
  CU(rr.alloc_live(n, h->stream));
  CU(ensure_cols(rr, n));
  CU(rr.d_rr_alloc_off.ensure((size_t)std::max<uint32_t>(n, 1) + 1));
  CU(rr.d_rr_alloc_node.ensure(e1));
  CU(rr.d_rr_alloc_res.ensure(e1));
  return CRANE_OK;
}

// The live rows of the handle's running table into the fresh one
int running_copy(crane_sched* h, RunningTable& rr, const uint32_t* live) {
  RunningTable& o = h->rr;
  ColSet cs{};
  o.each(rr, gather_to(cs, rr.n));
  TRY(gather(h, cs, live, rr.n));
  TRY(csr_offsets(h, o.d_rr_alloc_off.p, live, rr.n, rr.d_rr_alloc_off.p));
  TRY(csr_copy(h, o.d_rr_alloc_off.p, o.d_rr_alloc_node.p, live, rr.n, rr.d_rr_alloc_off.p, rr.d_rr_alloc_node.p));
  TRY(csr_copy(h, o.d_rr_alloc_off.p, o.d_rr_alloc_res.p, live, rr.n, rr.d_rr_alloc_off.p, rr.d_rr_alloc_res.p));
  return CRANE_OK;
}

// ---- the step scheduler --------------------------------------------------------------

// The nodes of a host step-job table (crane_sched_schedule_steps, crane_sched_step_jobs_append):
// its node_off, and each job's nodes in range, ascending and distinct
int check_step_jobs(crane_sched* h, const crane_step_jobs_t* jb) {
  const uint32_t J = jb->n_jobs;
  TRY(check_offsets(h, "step jobs: node_off", jb->node_off, J));
  if (jb->node_off[J] && (!jb->node || !jb->avail)) return fail(h, CRANE_EINVAL, "step jobs: null node table");
  for (uint32_t j = 0; j < J; ++j)
    for (uint32_t k = jb->node_off[j]; k < jb->node_off[j + 1]; ++k) {
      if (jb->node[k] >= h->layout.n_nodes) return fail(h, CRANE_EINVAL, "step jobs[%u]: node %u out of range", j, jb->node[k]);
      if (k > jb->node_off[j] && jb->node[k] <= jb->node[k - 1])
        return fail(h, CRANE_EINVAL, "step jobs[%u]: nodes must be ascending and distinct", j);
    }
  return CRANE_OK;
}

// k_steps over the jobs of dj, one warp per job
void launch_steps(crane_sched* h, const StepJobsDev& dj, const StepsDev& ds, const StepOutDev& dout) {
  const uint32_t grid = std::min<uint32_t>((dj.n_jobs + kStepWarps - 1) / kStepWarps, 16 * h->n_sm);
  CRANE_LAUNCH(k_steps, grid, 32 * kStepWarps, 0, h->stream, dj, ds, dout, (uint32_t)h->dict_slot);
}

// grid of a kernel with one warp per item, 256 threads per block
uint32_t warp_grid(const crane_sched* h, uint64_t items) {
  return (uint32_t)std::max<uint64_t>(1, std::min<uint64_t>((items + 7) / 8, 8ull * h->n_sm));
}

// What crane_sched_steps_compact keeps, decided on the host from its mirrors: a step-job
// row unless step_jobs_erase erased it; a step row unless it was erased or its job was
// (such a step is still pending or scheduled in h_state). Kept rows keep their order.
struct StepsKept {
  std::vector<uint8_t> jdead, sdead;  // [old rows] the row goes
  std::vector<uint32_t> jmap, smap;   // [old rows] its new row, or kRowNone
  uint32_t Jl = 0, Sl = 0, K = 0, A = 0;  // kept jobs, steps, scheduled steps, allocation rows
  // uploaded: live jobs [Jl] | live steps [Sl] | their new job rows [Sl] | the kept scheduled steps [K],
  // their new rows [K], their new allocation offsets [K] (the exclusive scan of node_num over them)
  std::vector<uint32_t> u;

  StepsKept(const StepJobTable& sj, const StepTable& sp)
      : jdead(sj.h_dead), sdead(sp.n), jmap(sj.n, kRowNone), smap(sp.n, kRowNone) {
    std::vector<uint32_t> sched, sched_new, sched_at, job;
    for (uint32_t j = 0; j < sj.n; ++j)
      if (!jdead[j]) {
        jmap[j] = Jl++;
        u.push_back(j);
      }
    for (uint32_t s = 0; s < sp.n; ++s) {
      sdead[s] = sp.h_state[s] == kSpErased || jdead[sp.h_job[s]];
      if (sdead[s]) continue;
      if (sp.h_state[s] == kSpScheduled) {
        sched.push_back(s);
        sched_new.push_back(Sl);
        sched_at.push_back(A);
        A += sp.h_nn[s];
      }
      job.push_back(jmap[sp.h_job[s]]);
      smap[s] = Sl++;
      u.push_back(s);
    }
    K = (uint32_t)sched.size();
    for (const auto* v : {&job, &sched, &sched_new, &sched_at}) u.insert(u.end(), v->begin(), v->end());
  }
};

// The compacted step tables: the host state of the kept rows of the handle's, the device
// buffers allocated for steps_copy
int steps_fresh(crane_sched* h, const StepsKept& kp, StepJobTable& sj, StepTable& sp) {
  const StepJobTable& oj = h->sj;
  const StepTable& os = h->sp;
  sj.n = kp.Jl;
  sj.h_node_off = live_offsets(oj.h_node_off, kp.jdead);
  sj.h_dead.assign(kp.Jl, 0);
  sj.h_dirty = live_only(oj.h_dirty, kp.jdead);
  for (uint32_t j : oj.h_dirty_rows)  // (old rows)
    if (!kp.jdead[j]) sj.h_dirty_rows.push_back(kp.jmap[j]);
  for (uint32_t j = 0; j < oj.n; ++j) {
    if (kp.jdead[j]) continue;
    sj.h_queue.emplace_back();
    for (uint32_t s : oj.h_queue[j]) sj.h_queue.back().push_back(kp.smap[s]);
  }
  sp.n = kp.Sl;
  sp.n_alloc = kp.A;
  sp.h_job.assign(kp.u.begin() + kp.Jl + kp.Sl, kp.u.begin() + kp.Jl + 2 * (size_t)kp.Sl);
  sp.h_nn = live_only(os.h_nn, kp.sdead);
  sp.h_nt = live_only(os.h_nt, kp.sdead);
  sp.h_state = live_only(os.h_state, kp.sdead);
  sp.h_incl_off = live_offsets(os.h_incl_off, kp.sdead);
  sp.h_excl_off = live_offsets(os.h_excl_off, kp.sdead);
  const size_t j1 = std::max<uint32_t>(kp.Jl, 1), s1 = std::max<uint32_t>(kp.Sl, 1);
  CU(ensure_cols(sj, kp.Jl));
  CU(sj.d_node_off.ensure(j1 + 1));
  CU(sj.d_node.ensure(std::max<uint32_t>(sj.h_node_off.back(), 1)));
  CU(sj.d_avail.ensure(std::max<uint32_t>(sj.h_node_off.back(), 1)));
  CU(ensure_cols(sp, kp.Sl));
  CU(sp.d_incl_off.ensure(s1 + 1));
  CU(sp.d_excl_off.ensure(s1 + 1));
  CU(sp.d_incl.ensure(std::max<uint32_t>(sp.h_incl_off.back(), 1)));
  CU(sp.d_excl.ensure(std::max<uint32_t>(sp.h_excl_off.back(), 1)));
  CU(sp.d_sa_node.ensure(std::max<uint32_t>(kp.A, 1)));
  CU(sp.d_sa_res.ensure(std::max<uint32_t>(kp.A, 1)));
  return CRANE_OK;
}

// The kept rows of the handle's step tables into the fresh ones; du = the uploaded StepsKept::u
int steps_copy(crane_sched* h, const StepsKept& kp, StepJobTable& sj, StepTable& sp, const uint32_t* du) {
  StepJobTable& oj = h->sj;
  StepTable& os = h->sp;
  const uint32_t Jl = kp.Jl, Sl = kp.Sl, K = kp.K;
  const uint32_t* jl = du, *sl = du + Jl, *job = sl + Sl, *sched = job + Sl;
  ColSet cs{};
  oj.each(sj, gather_to(cs, Jl));
  os.each(sp, gather_to(cs, Sl));
  TRY(gather(h, cs, sl, Sl));
  // the job column through the job map
  if (Sl) CU(cudaMemcpyAsync(sp.d_job.p, job, sizeof(uint32_t) * Sl, cudaMemcpyDeviceToDevice, h->stream));
  TRY(csr_offsets(h, oj.d_node_off.p, jl, Jl, sj.d_node_off.p));
  TRY(csr_copy(h, oj.d_node_off.p, oj.d_node.p, jl, Jl, sj.d_node_off.p, sj.d_node.p));
  TRY(csr_copy(h, oj.d_node_off.p, oj.d_avail.p, jl, Jl, sj.d_node_off.p, sj.d_avail.p));
  TRY(csr_offsets(h, os.d_incl_off.p, sl, Sl, sp.d_incl_off.p));
  TRY(csr_copy(h, os.d_incl_off.p, os.d_incl.p, sl, Sl, sp.d_incl_off.p, sp.d_incl.p));
  TRY(csr_offsets(h, os.d_excl_off.p, sl, Sl, sp.d_excl_off.p));
  TRY(csr_copy(h, os.d_excl_off.p, os.d_excl.p, sl, Sl, sp.d_excl_off.p, sp.d_excl.p));
  if (K)
    CRANE_LAUNCH(k_cp_spans, warp_grid(h, K), 256, 0, h->stream, os.d_alloc_at.p, os.d_nn.p, os.d_sa_node.p,
                 os.d_sa_res.p, sched, sched + K, sched + 2 * K, K, sp.d_alloc_at.p, sp.d_sa_node.p, sp.d_sa_res.p);
  return CRANE_OK;
}

}  // namespace

extern "C" {

const char* crane_sched_last_error(const crane_sched_t* h) { return h ? h->err.c_str() : "null handle"; }

int crane_sched_create(const crane_sched_config_t* cfg, int device, crane_sched_t** out) {
  if (!cfg || !out) return CRANE_EINVAL;
  *out = nullptr;
  int ndev = 0;
  if (cudaGetDeviceCount(&ndev) != cudaSuccess || ndev <= 0 || device < 0 || device >= ndev) return CRANE_ENODEV;
  if (cfg->max_jobs_per_node < 2 || cfg->max_jobs_per_node > 65000) return CRANE_EINVAL;
  if (cfg->cost_policy > 1) return CRANE_ENOSYS;  // 0 MinCpuTimeRatioFirst (JobScheduler.h:40), 1 BestFit (ours, config 4)
  if (device >= 64) return CRANE_EINVAL;
  int slot = -1;
  {
    std::lock_guard<std::mutex> lk(g_slot_mu);
    for (int k = 0; k < kDictSlots; ++k)
      if (!(g_slots_used[device] >> k & 1u)) { slot = k; g_slots_used[device] |= 1u << k; break; }
  }
  if (slot < 0) return CRANE_ENOSYS;  // more than kDictSlots live handles on one device
  crane_sched* h = new crane_sched();
  h->cfg = *cfg;
  h->device = device;
  h->dict_slot = slot;
  if (cudaSetDevice(device) != cudaSuccess || cudaStreamCreateWithFlags(&h->stream, cudaStreamNonBlocking) != cudaSuccess) {
    delete h;
    return CRANE_ENODEV;
  }
  for (auto& e : h->ev) cudaEventCreate(&e);
  int n_sm = 0, smem_optin = 0;
  if (cudaDeviceGetAttribute(&n_sm, cudaDevAttrMultiProcessorCount, device) != cudaSuccess ||
      cudaDeviceGetAttribute(&smem_optin, cudaDevAttrMaxSharedMemoryPerBlockOptin, device) != cudaSuccess || n_sm <= 0) {
    delete h;
    return CRANE_ENODEV;
  }
  h->n_sm = (uint32_t)n_sm;
  {
    // k_commit2: everything a block may opt in to (227 KB on H100) beyond the kernel's static tables
    size_t stat = 20 * 1024;
#ifndef CRANE_EMU
    cudaFuncAttributes fa;
    if (cudaFuncGetAttributes(&fa, k_commit2) == cudaSuccess) stat = fa.sharedSizeBytes;
#endif
    const size_t sm_total = (size_t)smem_optin;
    h->v2_budget = sm_total > stat + 1024 ? sm_total - stat - 1024 : 0;
    cudaFuncSetAttribute(k_commit2, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)h->v2_budget);
  }
  h->layout.tl_cap = cfg->max_jobs_per_node + 1;
  *out = h;
  return CRANE_OK;
}

void crane_sched_destroy(crane_sched_t* h) { delete h; }

int crane_sched_set_cluster(crane_sched_t* h, const crane_cluster_t* c) {
  if (!h || !c) return CRANE_EINVAL;
  if (!c->res_total || !c->alive || !c->drain || !c->part_off || (!c->part_nodes && c->n_nodes))
    return fail(h, CRANE_EINVAL, "cluster: null table");
  if (c->n_gres_entries > CRANE_GRES_ENTRIES) return fail(h, CRANE_EINVAL, "cluster: too many gres entries");
  for (uint32_t e = 0; e < c->n_gres_entries; ++e) {
    if (c->gres_entry_name[e] >= CRANE_GRES_NAMES) return fail(h, CRANE_EINVAL, "cluster: gres name id out of range");
    if (e && c->gres_entry_name[e] < c->gres_entry_name[e - 1])
      return fail(h, CRANE_EINVAL, "cluster: gres entries must be grouped by ascending name id");
  }
  CU(cudaSetDevice(h->device));
  lower_stage(h, kNone);  // state of the previous cluster / tick is void from here on
  TRY(check_offsets(h, "cluster: part_off", c->part_off, c->n_partitions));
  ClusterLayout& L = h->layout;
  L.n_nodes = c->n_nodes;
  L.n_parts = c->n_partitions;
  memset(&L.dict, 0, sizeof L.dict);
  L.dict.n_entries = c->n_gres_entries;
  for (int e = 0; e < CRANE_GRES_ENTRIES; ++e) L.dict.entry_name[e] = c->gres_entry_name[e];
  for (uint32_t e = 0; e < c->n_gres_entries; ++e) {
    const uint8_t g = c->gres_entry_name[e];
    if (L.dict.name_count[g] == 0) L.dict.name_first[g] = (uint8_t)e;
    L.dict.name_count[g]++;
    L.dict.name_mask8[g] |= 0xFFull << (8 * e);
  }
  L.res_total.assign(reinterpret_cast<const Row*>(c->res_total), reinterpret_cast<const Row*>(c->res_total) + c->n_nodes);
  L.alive.assign(c->alive, c->alive + c->n_nodes);
  L.drain.assign(c->drain, c->drain + c->n_nodes);
  L.part_off.assign(c->part_off, c->part_off + c->n_partitions + 1);
  L.part_nodes.assign(c->part_nodes, c->part_nodes + (c->n_partitions ? c->part_off[c->n_partitions] : 0));
  L.resv.reset();  // a new cluster has no reservations yet
  return build_layout(h);
}

int crane_sched_set_reservations(crane_sched_t* h, const crane_reservations_t* rv) {
  if (!h) return CRANE_EINVAL;
  TRY(require(h, kCluster, "set_reservations"));
  CU(cudaSetDevice(h->device));
  const uint32_t n = rv ? rv->n : 0;
  if (n && (!rv->start_time || !rv->end_time)) return fail(h, CRANE_EINVAL, "reservations: null table");
  if (n) TRY(check_offsets(h, "reservations: node_off", rv->node_off, n));
  for (uint32_t r = 0; r < n; ++r) {
    if (rv->end_time[r] < rv->start_time[r]) return fail(h, CRANE_EINVAL, "reservations[%u]: end before start", r);
    for (uint32_t k = rv->node_off[r]; k < rv->node_off[r + 1]; ++k) {
      if (!rv->node || !rv->res) return fail(h, CRANE_EINVAL, "reservations: null node table");
      if (rv->node[k] >= h->layout.n_nodes) return fail(h, CRANE_EINVAL, "reservations[%u]: node out of range", r);
      for (uint32_t k2 = rv->node_off[r]; k2 < k; ++k2)
        if (rv->node[k2] == rv->node[k]) return fail(h, CRANE_EINVAL, "reservations[%u]: node %u listed twice", r, rv->node[k]);
    }
  }
  lower_stage(h, kNone);
  Reservations& rs = h->layout.resv;
  rs.reset();
  rs.n = n;
  rs.start.assign(rv ? rv->start_time : nullptr, rv ? rv->start_time + n : nullptr);
  rs.end.assign(rv ? rv->end_time : nullptr, rv ? rv->end_time + n : nullptr);
  for (uint32_t r = 0; r < n; ++r) {
    // node states in node-index order: equal-cost nodes are ordered by index (deviation D1)
    std::vector<uint32_t> idx(rv->node_off[r + 1] - rv->node_off[r]);
    for (uint32_t k = 0; k < idx.size(); ++k) idx[k] = rv->node_off[r] + k;
    std::sort(idx.begin(), idx.end(), [&](uint32_t x, uint32_t y) { return rv->node[x] < rv->node[y]; });
    for (uint32_t k : idx) {
      rs.node.push_back(rv->node[k]);
      rs.res.push_back(reinterpret_cast<const Row&>(rv->res[k]));
    }
    rs.node_off.push_back((uint32_t)rs.node.size());
  }
  return build_layout(h);
}

int crane_sched_set_shard(crane_sched_t* h, uint32_t rank, uint32_t n_ranks, const uint32_t* part_owner) {
  if (!h) return CRANE_EINVAL;
  TRY(require(h, kCluster, "set_shard"));
  if (n_ranks == 0 || rank >= n_ranks) return fail(h, CRANE_EINVAL, "set_shard: rank %u of %u", rank, n_ranks);
  CU(cudaSetDevice(h->device));
  h->shard_rank = rank;
  h->shard_n = n_ranks;
  h->h_part_owner.clear();
  h->h_part_list.clear();
  if (n_ranks > 1) {
    if (!part_owner && h->layout.n_parts) return fail(h, CRANE_EINVAL, "set_shard: null owner table");
    std::vector<uint32_t> sched_owner(h->layout.n_vparts, 0);  // reservations: rank 0
    for (uint32_t p = 0; p < h->layout.n_parts; ++p) {
      if (part_owner[p] >= n_ranks) return fail(h, CRANE_EINVAL, "set_shard: partition %u owned by rank %u of %u", p, part_owner[p], n_ranks);
      h->h_part_owner.push_back(part_owner[p]);
      const uint32_t c = h->layout.h_part_comp[p];
      if (h->layout.h_part_cidx[p] == 0) sched_owner[c] = part_owner[p];
      else if (sched_owner[c] != part_owner[p])
        return fail(h, CRANE_EINVAL, "set_shard: partitions that share nodes must have one owner (partition %u)", p);
    }
    for (uint32_t c = 0; c < h->layout.n_vparts; ++c)
      if (sched_owner[c] == rank) h->h_part_list.push_back(c);
    H2D(h->d_sched_owner, sched_owner.data(), sched_owner.size());
    H2D(h->d_part_owner, h->h_part_owner.data(), h->h_part_owner.size());
    H2D(h->d_part_list, h->h_part_list.data(), h->h_part_list.size());
    CU(cudaStreamSynchronize(h->stream));
  }
  return CRANE_OK;
}

int crane_sched_device_placements(crane_sched_t* h, crane_device_placements_t* out) {
  if (!h || !out) return CRANE_EINVAL;
  TRY(require(h, kRan, "device_placements"));
  const RunOutputs& o = h->outputs;
  out->reason = o.d_reason.p;
  out->start_time = o.d_start.p;
  out->end_time = o.d_end.p;
  out->n_alloc = o.d_nalloc.p;
  out->alloc_node = o.d_node.p;
  out->alloc_ntasks = o.d_ntasks.p;
  out->alloc_res = o.d_res.p;
  out->n_jobs = h->pd.n;
  out->n_rows = h->pd.total_alloc;
  return CRANE_OK;
}

uint32_t crane_sched_pending_rows(const crane_sched_t* h) { return h ? h->pd.n : 0; }

int crane_sched_pending_reset(crane_sched_t* h) {
  if (!h) return CRANE_EINVAL;
  h->pd.reset();
  h->gate.on = false;
  h->gate.n = 0;
  h->gate.h_has_deps.clear();
  h->ent.n = 0;
  lower_stage(h, kCluster);
  return CRANE_OK;
}

int crane_sched_pending_append(crane_sched_t* h, const crane_pending_t* rows, uint32_t* first_row) {
  if (!h || !rows) return CRANE_EINVAL;
  TRY(require(h, kCluster, "pending_append"));
  CU(cudaSetDevice(h->device));
  lower_stage(h, kCluster);  // the running table and the work buffers follow with crane_sched_set_running
  const uint32_t base = h->pd.n;
  TRY(pending_append(h, rows));
  if (first_row) *first_row = base;
  return CRANE_OK;
}

int crane_sched_pending_erase(crane_sched_t* h, const uint32_t* rows, uint32_t n) {
  if (!h) return CRANE_EINVAL;
  return erase_rows(h, "pending_erase", h->pd, rows, n);
}

uint32_t crane_sched_running_rows(const crane_sched_t* h) { return h ? h->rr.n : 0; }

int crane_sched_running_append(crane_sched_t* h, const crane_running_t* rows, uint32_t* first_row) {
  if (!h || !rows) return CRANE_EINVAL;
  TRY(require(h, kCluster, "running_append"));
  CU(cudaSetDevice(h->device));
  TRY(running_check(h, rows, false));
  lower_stage(h, kCluster);  // the next run needs crane_sched_keep_running
  const uint32_t base = h->rr.n;
  TRY(running_append(h, rows));
  if (first_row) *first_row = base;
  return CRANE_OK;
}

int crane_sched_running_erase(crane_sched_t* h, const uint32_t* rows, uint32_t n) {
  if (!h) return CRANE_EINVAL;
  TRY(erase_rows(h, "running_erase", h->rr, rows, n));
  if (n) h->rr.dirty = true;
  return CRANE_OK;
}

int crane_sched_start(crane_sched_t* h, const uint32_t* rows, uint32_t n, uint32_t* first_row) {
  if (!h || (n && !rows)) return CRANE_EINVAL;
  if (h->shard_n > 1)  // other ranks' placement columns are zero until the caller's all-reduce
    return fail(h, CRANE_ENOSYS, "start: not available on a sharded handle (set_shard n_ranks > 1)");
  TRY(require(h, kRan, "start"));
  CU(cudaSetDevice(h->device));
  cudaStream_t st = h->stream;
  const uint32_t base = h->rr.n, eb = h->rr.h_rr_alloc_off.back();
  TRY(check_rows(h, "start", rows, n, h->pd.n, [&](uint32_t r) { return h->pd.h_dead[r] != 0; }));
  // the new rows' allocation offsets: node_num of the started rows (host mirror of alloc_off)
  std::vector<uint32_t> off(n + 1, eb);
  for (uint32_t k = 0; k < n; ++k) {
    const uint64_t e = (uint64_t)off[k] + (h->pd.h_alloc_off[rows[k] + 1] - h->pd.h_alloc_off[rows[k]]);
    if (e > 0xfffffff0ull || (uint64_t)base + n > 0xfffffff0ull) return fail(h, CRANE_EINVAL, "start: too many running rows");
    off[k + 1] = (uint32_t)e;
  }
  if (n) {
    // every row must hold a start-now placement of the last run (after any qos_filter)
    H2D(h->d_start_rows, rows, n);
    CU(h->d_flag.ensure(1));
    CU(cudaMemsetAsync(h->d_flag.p, 0, sizeof(uint32_t), st));
    CRANE_LAUNCH(k_start_check, (n + 255) / 256, 256, 0, st, h->d_start_rows.p, n, h->outputs.d_reason.p, h->d_flag.p);
    uint32_t bad = 0;
    CU(cudaMemcpyAsync(&bad, h->d_flag.p, sizeof(uint32_t), cudaMemcpyDeviceToHost, st));
    CU(cudaStreamSynchronize(st));
    CU(cudaGetLastError());
    if (bad) return fail(h, CRANE_EINVAL, "start: a row does not hold a start-now placement of the last run");
  }
  lower_stage(h, kCluster);  // the run's outputs are void from here on
  if (!n) {
    if (first_row) *first_row = base;
    return CRANE_OK;
  }
  const uint32_t rows_end = base + n, ent_end = off[n];
  CU(grow_cols(h->rr, rows_end, base, st));
  CU(h->rr.d_rr_alloc_node.grow(ent_end, eb, st));
  CU(h->rr.d_rr_alloc_res.grow(ent_end, eb, st));
  H2D_AT(h->rr.d_rr_alloc_off, off.data(), base, (size_t)n + 1);
  std::vector<uint8_t> zeros(n, 0);
  H2D_AT(h->rr.d_dead, zeros.data(), base, n);
  const uint32_t nb = std::min<uint32_t>((n + 7) / 8, 8 * h->n_sm);
  CRANE_LAUNCH(k_start, nb, 256, 0, st, h->pd.dev(), h->outputs.dev(), h->d_start_rows.p, n, base, h->rr.dev());
  // the pending rows leave the pending table (m_pending_job_map_.erase, JobScheduler.cpp:1305)
  CRANE_LAUNCH(k_mark_dead, (n + 255) / 256, 256, 0, st, h->d_start_rows.p, n, h->pd.d_dead.p);
  CU(cudaGetLastError());
  if (h->ent.n) {  // AFTER fires at the placement's start (JobScheduler.cpp:1549), the rest follow the job
    TRY(upload_call_rows(h, rows, n));
    DepEvents ev{};
    ev.mode = kFireStart;
    ev.time = h->outputs.d_start.p;
    ev.base = base;
    TRY(dep_fire(h, ev, n, h->ent.n));
  }
  for (uint32_t k = 0; k < n; ++k) {
    h->pd.h_dead[rows[k]] = 1;
    h->rr.h_rr_account.push_back(h->pd.h_pd_account[rows[k]]);
    h->rr.h_dead.push_back(0);
    h->rr.h_rr_alloc_off.push_back(off[k + 1]);
  }
  h->pd.n_dead += n;
  h->rr.n = rows_end;
  h->rr.node_bound = std::max(h->rr.node_bound, h->layout.n_nodes);  // (placements are on this cluster's nodes)
  h->rr.dirty = true;
  CU(cudaStreamSynchronize(st));
  if (first_row) *first_row = base;
  return CRANE_OK;
}

int crane_sched_pending_set_gate(crane_sched_t* h, const uint32_t* rows, uint32_t n, const uint8_t* held,
                                 const int64_t* begin_time) {
  if (!h || (n && !rows)) return CRANE_EINVAL;
  TRY(require(h, kCluster, "pending_set_gate"));
  CU(cudaSetDevice(h->device));
  for (uint32_t k = 0; k < n; ++k)
    if (rows[k] >= h->pd.n) return fail(h, CRANE_EINVAL, "pending_set_gate: row %u out of range", rows[k]);
  lower_stage(h, kCluster);
  TRY(gate_fit(h));
  if (n && (held || begin_time)) {
    H2D(h->d_ev_rows, rows, n);
    if (held) H2D(h->d_ev_u8, held, n);
    if (begin_time) H2D(h->d_ev_i64, begin_time, n);
    CRANE_LAUNCH(k_gate_set, (n + 255) / 256, 256, 0, h->stream, gate_dev(h), h->d_ev_rows.p, n,
                 held ? h->d_ev_u8.p : nullptr, begin_time ? h->d_ev_i64.p : nullptr);
    CU(cudaGetLastError());
  }
  CU(cudaStreamSynchronize(h->stream));
  return CRANE_OK;
}

int crane_sched_pending_depend(crane_sched_t* h, const crane_dependencies_t* d) {
  if (!h || !d) return CRANE_EINVAL;
  TRY(require(h, kCluster, "pending_depend"));
  CU(cudaSetDevice(h->device));
  const uint32_t n = d->n;
  if (n && (!d->row || !d->is_or)) return fail(h, CRANE_EINVAL, "depend: null column");
  TRY(check_offsets(h, "depend: dep_off", d->dep_off, n));
  const uint32_t m = d->dep_off[n];
  if (m && (!d->kind || !d->dependee || !d->type || !d->delay_s)) return fail(h, CRANE_EINVAL, "depend: null entry column");
  if ((uint64_t)h->ent.n + m > 0xfffffff0ull) return fail(h, CRANE_EINVAL, "depend: too many entries");
  {
    std::vector<uint32_t> sorted(d->row, d->row + n);
    std::sort(sorted.begin(), sorted.end());
    for (uint32_t k = 1; k < n; ++k)
      if (sorted[k] == sorted[k - 1]) return fail(h, CRANE_EINVAL, "depend: row %u listed twice", sorted[k]);
  }
  std::vector<uint32_t> dependent(m), dependee(m);
  for (uint32_t k = 0; k < n; ++k) {
    const uint32_t r = d->row[k];
    if (r >= h->pd.n) return fail(h, CRANE_EINVAL, "depend: row %u out of range", r);
    if (h->pd.h_dead[r]) return fail(h, CRANE_EINVAL, "depend: row %u was erased", r);
    if (r < h->gate.h_has_deps.size() && h->gate.h_has_deps[r]) return fail(h, CRANE_EINVAL, "depend: row %u already has its list", r);
    for (uint32_t e = d->dep_off[k]; e < d->dep_off[k + 1]; ++e) {
      const uint8_t kind = d->kind[e];
      const uint32_t q = d->dependee[e];
      if (kind > CRANE_DEPENDEE_EVENT) return fail(h, CRANE_EINVAL, "depend: row %u: dependee kind %u", r, kind);
      if (d->type[e] > CRANE_DEP_AFTER_NOT_OK) return fail(h, CRANE_EINVAL, "depend: row %u: type %u", r, d->type[e]);
      if (d->delay_s[e] >= (1ull << 62)) return fail(h, CRANE_EINVAL, "depend: row %u: delay out of range", r);
      if (kind == CRANE_DEPENDEE_EVENT) {
        if (!d->event_time) return fail(h, CRANE_EINVAL, "depend: EVENT entries without event_time");
      } else if (kind == CRANE_DEPENDEE_PENDING) {
        if (q >= h->pd.n || h->pd.h_dead[q]) return fail(h, CRANE_EINVAL, "depend: row %u: pending dependee %u missing", r, q);
        if (q == r) return fail(h, CRANE_EINVAL, "depend: row %u depends on itself", r);
      } else if (q >= h->rr.n || h->rr.h_dead[q]) {
        return fail(h, CRANE_EINVAL, "depend: row %u: running dependee %u missing", r, q);
      }
      for (uint32_t e2 = d->dep_off[k]; e2 < e && kind != CRANE_DEPENDEE_EVENT; ++e2)  // `deps` is a map
        if (d->kind[e2] == kind && d->dependee[e2] == q) return fail(h, CRANE_EINVAL, "depend: row %u lists a dependee twice", r);
      dependent[e] = r;
      dependee[e] = kind == CRANE_DEPENDEE_EVENT ? 0 : q;
    }
  }
  lower_stage(h, kCluster);
  TRY(gate_fit(h));
  cudaStream_t st = h->stream;
  const uint32_t e0 = h->ent.n;
  if (m) {
    std::vector<uint8_t> live(m, 1);
    H2D_AT(h->ent.d_e_dependent, dependent.data(), e0, m);
    H2D_AT(h->ent.d_e_dependee, dependee.data(), e0, m);
    H2D_AT(h->ent.d_e_kind, d->kind, e0, m);
    H2D_AT(h->ent.d_e_type, d->type, e0, m);
    H2D_AT(h->ent.d_e_delay, d->delay_s, e0, m);
    H2D_AT(h->ent.d_e_live, live.data(), e0, m);
    if (d->event_time) H2D(h->d_ev_i64, d->event_time, m);
    CU(cudaStreamSynchronize(st));  // (the staging vectors are pageable)
  }
  h->ent.n = e0 + m;
  if (n) {
    H2D(h->d_ev_rows, d->row, n);
    H2D(h->d_ev_u8, d->is_or, n);
    H2D(h->d_ev_u32, d->dep_off, (size_t)n + 1);
    CRANE_LAUNCH(k_dep_rows, (n + 255) / 256, 256, 0, st, gate_dev(h), h->d_ev_rows.p, n, h->d_ev_u8.p, h->d_ev_u32.p);
    CU(cudaGetLastError());
  }
  // entries resolved on arrival: EVENT, and AFTER on a running dependee
  DepEvents ev{};
  ev.mode = kFireDepend;
  ev.run_start = h->rr.d_rr_start.p;
  ev.event_time = d->event_time ? h->d_ev_i64.p : nullptr;
  ev.e0 = e0;
  TRY(dep_fire(h, ev, 0, m));
  for (uint32_t k = 0; k < n; ++k) h->gate.h_has_deps[d->row[k]] = 1;
  CU(cudaStreamSynchronize(st));
  return CRANE_OK;
}

int crane_sched_pending_cancel(crane_sched_t* h, const uint32_t* rows, uint32_t n, int64_t cancel_time) {
  TRY(crane_sched_pending_erase(h, rows, n));
  if (!n || !h->ent.n) return CRANE_OK;
  TRY(upload_call_rows(h, rows, n));
  DepEvents ev{};
  ev.mode = kFireCancel;
  ev.t = cancel_time;
  TRY(dep_fire(h, ev, n, h->ent.n));
  CU(cudaStreamSynchronize(h->stream));
  return CRANE_OK;
}

int crane_sched_running_end(crane_sched_t* h, const uint32_t* rows, uint32_t n, const int64_t* end_time,
                            const uint32_t* exit_code) {
  if (!h) return CRANE_EINVAL;
  if (n && (!end_time || !exit_code)) return fail(h, CRANE_EINVAL, "running_end: null column");
  TRY(crane_sched_running_erase(h, rows, n));
  if (!n || !h->ent.n) return CRANE_OK;
  TRY(upload_call_rows(h, rows, n));
  H2D(h->d_ev_i64, end_time, n);
  H2D(h->d_ev_u32, exit_code, n);
  DepEvents ev{};
  ev.mode = kFireEnd;
  ev.time = h->d_ev_i64.p;
  ev.code = h->d_ev_u32.p;
  TRY(dep_fire(h, ev, n, h->ent.n));
  CU(cudaStreamSynchronize(h->stream));
  return CRANE_OK;
}

int crane_sched_compact(crane_sched_t* h, uint32_t* pending_map, uint32_t* running_map) {
  if (!h) return CRANE_EINVAL;
  TRY(require(h, kCluster, "compact"));
  CU(cudaSetDevice(h->device));
  lower_stage(h, kCluster);  // the run's outputs are indexed by the old rows
  cudaStream_t st = h->stream;
  const uint32_t N = h->pd.n, Rt = h->rr.n, M = h->ent.n;
  const bool cp_pd = h->pd.n_dead > 0, cp_rr = h->rr.n_dead > 0;
  const uint32_t Nl = N - h->pd.n_dead, Rl = Rt - h->rr.n_dead;

  // ---- work buffers, then the live rows, the maps and the open entries ----
  CU(h->work.ensure_sort(std::max<size_t>({(size_t)N, (size_t)Rt, (size_t)M})));
  CU(h->d_flag.ensure(1));
  DBuf<uint32_t> pd_live, pd_map, rr_live, rr_map, keep;
  if (cp_pd) {
    CU(pd_live.ensure(std::max<uint32_t>(Nl, 1)));
    CU(pd_map.ensure(N));
    TRY(live_rows(h, h->pd.d_dead.p, N, Nl, pd_live.p, pd_map.p));
  }
  if (cp_rr) {
    CU(rr_live.ensure(std::max<uint32_t>(Rl, 1)));
    CU(rr_map.ensure(Rt));
    TRY(live_rows(h, h->rr.d_dead.p, Rt, Rl, rr_live.p, rr_map.p));
  }
  uint32_t n_keep = 0;
  if (M) {
    CU(keep.ensure(M));
    CU(cudaMemsetAsync(h->d_flag.p, 0, sizeof(uint32_t), st));
    CRANE_LAUNCH(k_cp_ent_keys, (M + 255) / 256, 256, 0, st, gate_dev(h), h->pd.dead(),
                 h->work.d_keys_a.p, h->work.d_vals_a.p, h->d_flag.p);
    uint64_t* keys;
    uint32_t* vals;
    TRY(radix_sort(h, M, 8, &keys, &vals));
    CU(cudaMemcpyAsync(keep.p, vals, sizeof(uint32_t) * M, cudaMemcpyDeviceToDevice, st));
    CU(cudaMemcpyAsync(&n_keep, h->d_flag.p, sizeof(uint32_t), cudaMemcpyDeviceToHost, st));
  }
  CU(cudaStreamSynchronize(st));
  CU(cudaGetLastError());
  const bool cp_ent = M && (n_keep < M || cp_pd || cp_rr);

  // ---- every new buffer before the first gather: CRANE_ENOMEM leaves the tables as they were ----
  PendingTable pd;
  GateRows gate;
  RunningTable rr;
  DepEntries ent;
  if (cp_pd) TRY(pending_fresh(h, pd, gate));
  if (cp_rr) TRY(running_fresh(h, rr));
  if (cp_ent) {
    ent.n = n_keep;
    CU(ensure_cols(ent, n_keep));
  }

  // ---- gathers ----
  if (cp_pd) TRY(pending_copy(h, pd, gate, pd_live.p));
  if (cp_rr) TRY(running_copy(h, rr, rr_live.p));
  if (cp_ent && n_keep)
    CRANE_LAUNCH(k_cp_entries, (n_keep + 255) / 256, 256, 0, st, gate_dev(h), gate_dev(gate, ent, nullptr), keep.p,
                 n_keep, cp_pd ? pd_map.p : nullptr, cp_rr ? rr_map.p : nullptr);
  CU(cudaGetLastError());
  CU(cudaStreamSynchronize(st));

  // ---- the new tables replace the old ones (whose buffers go with the locals) ----
  if (cp_pd) {
    std::swap(h->pd, pd);
    std::swap(h->gate, gate);
  }
  if (cp_rr) std::swap(h->rr, rr);
  if (cp_ent) std::swap(h->ent, ent);
  if (cp_pd || cp_rr) {  // (sized for the old tables)
    h->work.release();
    h->outputs.release();
  }

  // ---- the maps ----
  if (pending_map) {
    if (cp_pd) CU(cudaMemcpyAsync(pending_map, pd_map.p, sizeof(uint32_t) * N, cudaMemcpyDeviceToHost, st));
    else for (uint32_t r = 0; r < N; ++r) pending_map[r] = r;
  }
  if (running_map) {
    if (cp_rr) CU(cudaMemcpyAsync(running_map, rr_map.p, sizeof(uint32_t) * Rt, cudaMemcpyDeviceToHost, st));
    else for (uint32_t r = 0; r < Rt; ++r) running_map[r] = r;
  }
  CU(cudaStreamSynchronize(st));
  return CRANE_OK;
}

int crane_sched_keep_running(crane_sched_t* h, float* device_ms) {
  if (!h) return CRANE_EINVAL;
  TRY(require(h, kCluster, "keep_running"));
  CU(cudaSetDevice(h->device));
  lower_stage(h, kCluster);
  TRY(keep_running(h));
  if (device_ms) {
    CU(cudaEventSynchronize(h->ev[kEvKeepEnd]));
    *device_ms = elapsed_ms(h, kEvKeepBegin, kEvKeepEnd);
  }
  h->stage = kUploaded;
  return CRANE_OK;
}

int crane_sched_set_running(crane_sched_t* h, const crane_running_t* rn) {
  if (!h) return CRANE_EINVAL;
  TRY(require(h, kCluster, "set_running"));
  CU(cudaSetDevice(h->device));
  lower_stage(h, kCluster);
  TRY(set_running(h, rn));
  h->stage = kUploaded;
  return CRANE_OK;
}

int crane_sched_upload(crane_sched_t* h, const crane_running_t* rn, const crane_pending_t* pd) {
  if (!h || !pd) return CRANE_EINVAL;
  TRY(require(h, kCluster, "upload"));
  CU(cudaSetDevice(h->device));
  lower_stage(h, kCluster);  // a failed upload leaves nothing runnable behind
  CU(cudaEventRecord(h->ev[kEvH2dBegin], h->stream));
  crane_sched_pending_reset(h);
  int rc = pending_append(h, pd);
  if (rc != CRANE_OK) { crane_sched_pending_reset(h); return rc; }
  TRY(set_running(h, rn));
  CU(cudaEventRecord(h->ev[kEvH2dEnd], h->stream));
  h->h2d_timed = true;
  h->stage = kUploaded;
  return CRANE_OK;
}

int crane_sched_run(crane_sched_t* h, int64_t now) {
  if (!h) return CRANE_EINVAL;
  TRY(require(h, kUploaded, "run"));
  CU(cudaSetDevice(h->device));
  lower_stage(h, kUploaded);  // the previous run's outputs are void from here on
  (void)cudaGetLastError();  // a stale error of an earlier, unrelated call in this process is not this run's
  cudaStream_t st = h->stream;
  const ClusterLayout& L = h->layout;
  RunWork& w = h->work;
  const uint32_t N = h->pd.n, R = h->view.n, A = h->view.n_accounts;
  h->timing.kernel_launches = 0;
  PendingDev pd = h->pd.dev();
  const RunningDev rn = h->view.dev();
  const ClusterDev cl = L.dev();
  const TimelineDev tl = L.timelines();
  const PlaceDev out = h->outputs.dev();

  // ---- node state / timelines (R2,R3,R4) -----------------------------------
  CU(cudaEventRecord(h->ev[kEvRunBegin], st));
  if (h->pd.total_alloc) {  // allocation slots of jobs without a placement read as zero
    CU(cudaMemsetAsync(out.alloc_node, 0, sizeof(uint32_t) * h->pd.total_alloc, st));
    CU(cudaMemsetAsync(out.alloc_ntasks, 0, sizeof(uint32_t) * h->pd.total_alloc, st));
    CU(cudaMemsetAsync(out.alloc_res, 0, sizeof(Row) * h->pd.total_alloc, st));
  }
  if (L.n_slots) {
    CRANE_LAUNCH(k_node_init, (L.n_slots + 127) / 128, 128, 0, st, cl, rn, tl, now, h->cfg.max_jobs_per_node, h->cfg.cost_policy);
    h->timing.kernel_launches++;
  }
  CU(cudaEventRecord(h->ev[kEvInitEnd], st));

  // ---- the gate: held, not-yet-begun and dependent rows sit this run out ----
  const bool gated = h->gate.on && N;
  if (gated) {
    TRY(gate_fit(h));
    CU(w.d_g_code.ensure(N));
    CRANE_LAUNCH(k_gate, (N + 255) / 256, 256, 0, st, gate_dev(h), now, w.d_g_code.p);
    pd.dead = w.d_g_code.p;
    h->timing.kernel_launches++;
    // an account with only gated rows does not seed the fair-share bounds
    if (A) {
      CU(cudaMemsetAsync(h->view.d_acc_present.p, 0, A, st));
      CRANE_LAUNCH(k_acc_present, (N + R + 255) / 256, 256, 0, st, h->pd.d_account.p, w.d_g_code.p, N,
                   rn.account, R, h->view.d_acc_present.p);
      h->timing.kernel_launches++;
    }
  }

  // ---- priority + queue (R5,R6) --------------------------------------------
  uint32_t nq_cap = std::min<uint32_t>(N, h->cfg.scheduled_batch_size);
  CU(cudaMemsetAsync(L.d_part_count.p, 0, sizeof(uint32_t) * (L.n_vparts + 2), st));
  CU(w.d_vpart.ensure(std::max<uint32_t>(N, 1)));
  if (N) {
    PrioCfg pc{};
    pc.type = h->cfg.priority_type;
    pc.favor_small = h->cfg.favor_small;
    pc.w_age = h->cfg.weight_age;
    pc.w_fs = h->cfg.weight_fair_share;
    pc.w_size = h->cfg.weight_job_size;
    pc.w_part = h->cfg.weight_partition;
    pc.w_qos = h->cfg.weight_qos;
    pc.max_age = h->cfg.max_age_s;
    uint64_t* keys = w.d_keys_a.p;
    uint32_t* vals = w.d_vals_a.p;
    if (pc.type != 0) {
      CRANE_LAUNCH(k_bounds_init, 1, 32, 0, st, w.d_bounds.p);
      uint32_t nb = std::min<uint32_t>((N + R + 255) / 256, 4 * h->n_sm);
      CRANE_LAUNCH(k_bounds, nb, 256, 0, st, pd, rn, now, (uint64_t)h->cfg.max_age_s, w.d_bounds.p);
      h->timing.kernel_launches += 2;
      if (A) {
        CU(cudaMemsetAsync(w.d_acc_service.p, 0, sizeof(double) * A, st));
        CRANE_LAUNCH(k_service, (A + 127) / 128, 128, 0, st, rn, now, w.d_bounds.p, w.d_acc_service.p);
        h->timing.kernel_launches++;
      }
    }
    CRANE_LAUNCH(k_priority, (N + 255) / 256, 256, 0, st, pd, pc, now, w.d_bounds.p, w.d_acc_service.p,
                 w.d_prio.p, w.d_keys_a.p, w.d_vals_a.p);
    h->timing.kernel_launches++;
    if (pc.type != 0 || h->pd.n_dead || gated)  // (FIFO keeps input order; excluded rows only have to go behind the others)
      TRY(radix_sort(h, N, pc.type != 0 ? 64 : 8, &keys, &vals));
    // keys2 go to the buffer not holding `vals`
    uint64_t* key2 = w.d_keys_a.p;
    uint32_t* order = vals;
    if (order != w.d_vals_a.p) {
      // radix_sort works on the (keys_a, vals_a) pair: bring the order back
      CU(cudaMemcpyAsync(w.d_vals_a.p, order, sizeof(uint32_t) * N, cudaMemcpyDeviceToDevice, st));
      order = w.d_vals_a.p;
    }
    CRANE_LAUNCH(k_queue_keys, (N + 255) / 256, 256, 0, st, pd, order, w.d_prio.p, h->cfg.scheduled_batch_size,
                 cl, now, key2, out, L.d_part_count.p, w.d_vpart.p);
    CRANE_LAUNCH(k_part_offsets, 1, 32, 0, st, L.d_part_count.p, L.n_vparts, L.d_part_job_off.p);
    h->timing.kernel_launches += 2;
    int bits = 8;
    while ((1ull << bits) < (uint64_t)L.n_vparts + 2) bits += 8;
    uint64_t* k2s;
    uint32_t* queue;
    TRY(radix_sort(h, N, bits, &k2s, &queue));
    if (nq_cap) {
      // n_queued <= nq_cap lives on the device (part_job_off[n_parts]); the
      // kernels below bound themselves with it.
      CRANE_LAUNCH(k_build_jobq, (nq_cap + 127) / 128, 128, 0, st, pd, queue, L.d_part_job_off.p + L.n_vparts, w.d_jobq.p, (uint32_t)h->dict_slot, w.d_vpart.p, L.n_comp, L.d_part_cidx.p);
      h->timing.kernel_launches++;
    }
  } else {
    CRANE_LAUNCH(k_part_offsets, 1, 32, 0, st, L.d_part_count.p, L.n_vparts, L.d_part_job_off.p);
    h->timing.kernel_launches++;
  }
  CU(cudaEventRecord(h->ev[kEvPrioEnd], st));

  // ---- capability bitmap (R7 predicate + R8) -------------------------------
  if (nq_cap && L.n_vparts) {
    uint32_t wpb = 8;
    uint32_t nb = std::min<uint32_t>((nq_cap + wpb - 1) / wpb, 8 * h->n_sm);
    CRANE_LAUNCH(k_feas_bitmap, nb, wpb * 32, 0, st, cl, pd, w.d_jobq.p, L.d_part_job_off.p + L.n_vparts, L.words_per_row, w.d_bitmap.p,
                 h->shard_n > 1 ? h->d_sched_owner.p : nullptr, h->shard_rank, (uint32_t)h->dict_slot);
    h->timing.kernel_launches++;
  }
  CU(cudaEventRecord(h->ev[kEvFeasEnd], st));

  // ---- sequential commit (R7,R9,R10,R11) -----------------------------------
  if (nq_cap && L.n_vparts) {
    Commit2Args c2{};
    c2.cl = cl; c2.tl = tl; c2.jobq = w.d_jobq.p; c2.part_job_off = L.d_part_job_off.p; c2.bitmap = w.d_bitmap.p;
    c2.words_per_row = L.words_per_row; c2.ring = L.v2_ring; c2.out = out; c2.now = now;
    c2.max_window = h->cfg.max_time_window_s; c2.max_jobs = h->cfg.max_jobs_per_node; c2.cost_policy = h->cfg.cost_policy;
    c2.prof = L.d_prof.p;
    c2.gres = L.dict.n_entries > 0 ? 1u : 0u;
    c2.sched_nparts = L.max_comp_parts > 1 ? L.d_sched_nparts.p : nullptr;
    c2.slot_memb = L.d_slot_memb.p;
    c2.dslot = (uint32_t)h->dict_slot;
    c2.req_node = h->pd.d_req_node.p;
    c2.req_task = h->pd.d_req_task.p;
    size_t smem = commit2_smem_bytes(L.max_part_slots, L.words_per_row, c2.gres != 0, L.v2_ring, L.max_comp_parts);
    uint32_t grid = L.n_vparts;
    if (h->shard_n > 1) {
      c2.part_list = h->d_part_list.p;
      grid = (uint32_t)h->h_part_list.size();
    }
    if (grid) CRANE_LAUNCH(k_commit2, grid, kT2, smem, st, c2);
    h->timing.kernel_launches++;
    if (h->shard_n > 1 && N) {
      CRANE_LAUNCH(k_shard_mask, (N + 255) / 256, 256, 0, st, pd, out, h->d_part_owner.p, L.n_parts, h->shard_rank);
      h->timing.kernel_launches++;
    }
  }
  CU(cudaEventRecord(h->ev[kEvRunEnd], st));
  CU(cudaGetLastError());
  h->stage = kRan;
  return CRANE_OK;
}

int crane_sched_fetch(crane_sched_t* h, crane_placements_t* out) {
  if (!h || !out) return CRANE_EINVAL;
  TRY(require(h, kRan, "fetch"));
  CU(cudaSetDevice(h->device));
  cudaStream_t st = h->stream;
  const uint32_t N = h->pd.n;
  if (N && (!out->reason || !out->priority || !out->start_time || !out->end_time || !out->n_alloc || !out->alloc_off))
    return fail(h, CRANE_EINVAL, "placements: null column");
  if (h->pd.total_alloc && (!out->alloc_node || !out->alloc_ntasks || !out->alloc_res))
    return fail(h, CRANE_EINVAL, "placements: null allocation table");
  const RunOutputs& o = h->outputs;
  // slots of jobs without a placement stay zero
  if (N) {
    CU(cudaMemcpyAsync(out->reason, o.d_reason.p, N, cudaMemcpyDeviceToHost, st));
    CU(cudaMemcpyAsync(out->priority, o.d_prio.p, sizeof(double) * N, cudaMemcpyDeviceToHost, st));
    CU(cudaMemcpyAsync(out->start_time, o.d_start.p, sizeof(int64_t) * N, cudaMemcpyDeviceToHost, st));
    CU(cudaMemcpyAsync(out->end_time, o.d_end.p, sizeof(int64_t) * N, cudaMemcpyDeviceToHost, st));
    CU(cudaMemcpyAsync(out->n_alloc, o.d_nalloc.p, sizeof(uint32_t) * N, cudaMemcpyDeviceToHost, st));
  }
  if (h->pd.total_alloc) {
    CU(cudaMemcpyAsync(out->alloc_node, o.d_node.p, sizeof(uint32_t) * h->pd.total_alloc, cudaMemcpyDeviceToHost, st));
    CU(cudaMemcpyAsync(out->alloc_ntasks, o.d_ntasks.p, sizeof(uint32_t) * h->pd.total_alloc, cudaMemcpyDeviceToHost, st));
    CU(cudaMemcpyAsync(out->alloc_res, o.d_res.p, sizeof(Row) * h->pd.total_alloc, cudaMemcpyDeviceToHost, st));
  }
  memcpy(out->alloc_off, h->pd.h_alloc_off.data(), sizeof(uint32_t) * ((size_t)N + 1));
  CU(cudaEventRecord(h->ev[kEvD2hEnd], st));
  CU(cudaStreamSynchronize(st));
  CU(cudaGetLastError());
  // (the upload events exist only after crane_sched_upload: a resident table is filled piecewise)
  h->timing.h2d_ms = h->h2d_timed ? elapsed_ms(h, kEvH2dBegin, kEvH2dEnd) : 0.f;
  read_run_times(h);
  h->timing.d2h_ms = elapsed_ms(h, kEvRunEnd, kEvD2hEnd);
  return CRANE_OK;
}

int crane_sched_node_select(crane_sched_t* h, int64_t now, const crane_running_t* running,
                            const crane_pending_t* pending, crane_placements_t* out) {
  TRY(crane_sched_upload(h, running, pending));
  TRY(crane_sched_run(h, now));
  return crane_sched_fetch(h, out);
}

int crane_sched_sync(crane_sched_t* h, float* run_ms) {
  if (!h) return CRANE_EINVAL;
  CU(cudaSetDevice(h->device));
  CU(cudaStreamSynchronize(h->stream));
  CU(cudaGetLastError());
  if (h->stage == kRan) read_run_times(h);
  if (run_ms) *run_ms = h->stage == kRan ? h->timing.total_ms : 0.f;
  return CRANE_OK;
}

int crane_sched_debug_profile(crane_sched_t* h, unsigned long long* dst, size_t cap) {
  if (!h || !dst) return CRANE_EINVAL;
  TRY(require(h, kRan, "debug_profile"));
  CU(cudaSetDevice(h->device));
  size_t n = std::min(cap, (size_t)h->layout.n_vparts * 16);
  CU(cudaStreamSynchronize(h->stream));
  if (n) CU(cudaMemcpy(dst, h->layout.d_prof.p, n * sizeof(unsigned long long), cudaMemcpyDeviceToHost));
  return CRANE_OK;
}

int crane_sched_qos_filter(crane_sched_t* h, const crane_qos_table_t* qt, uint8_t* reason) {
  if (!h || !qt || !reason) return CRANE_EINVAL;
  TRY(require(h, kRan, "qos_filter"));
  if (!h->pd.have_qos_cols) return fail(h, CRANE_EINVAL, "qos_filter: pending.qos / pending.user were not uploaded");
  CU(cudaSetDevice(h->device));
  const uint32_t N = h->pd.n, Q = qt->n_qos, U = qt->n_users, A = qt->n_accounts;
  if (Q == 0 || Q >= 65535) return fail(h, CRANE_EINVAL, "qos_filter: n_qos out of range");
  if (A > 65535) return fail(h, CRANE_ENOSYS, "qos_filter: more than 65535 accounts");
  if (!qt->valid || !qt->max_jobs_per_user || !qt->max_jobs_per_account || !qt->max_jobs ||
      !qt->max_cpus_per_user_raw || !qt->max_wall || !qt->max_tres_per_user || !qt->max_tres_per_account ||
      !qt->max_tres || !qt->user_usage || !qt->qos_usage || (A && !qt->account_usage))
    return fail(h, CRANE_EINVAL, "qos_filter: null column");
  TRY(check_offsets(h, "qos_filter: chain_off", qt->chain_off, N));
  // the levels of one job are checked lane-parallel: user + chain + qos <= 32
  // lanes, and one usage entry per lane (a chain never repeats an account)
  for (uint32_t i = 0; i < N; ++i) {
    const uint32_t c0 = qt->chain_off[i], c1 = qt->chain_off[i + 1];
    if (c1 - c0 > 30) return fail(h, CRANE_ENOSYS, "qos_filter: pending[%u]: account chain longer than 30", i);
    for (uint32_t a = c0; a < c1; ++a) {
      if (qt->chain_acct[a] >= A) return fail(h, CRANE_EINVAL, "qos_filter: pending[%u]: account out of range", i);
      for (uint32_t b = c0; b < a; ++b)
        if (qt->chain_acct[a] == qt->chain_acct[b])
          return fail(h, CRANE_EINVAL, "qos_filter: pending[%u]: account repeated in chain", i);
    }
  }
  // user ids are checked on the device side of the table: against n_users here
  // (pending.user was validated only for presence at upload)
  {
    std::vector<uint32_t> users(N);
    if (N) CU(cudaMemcpyAsync(users.data(), h->pd.d_user.p, (size_t)N * 4, cudaMemcpyDeviceToHost, h->stream));
    CU(cudaStreamSynchronize(h->stream));
    for (uint32_t i = 0; i < N; ++i)
      if (users[i] >= U) return fail(h, CRANE_EINVAL, "qos_filter: pending[%u]: user out of range", i);
  }
  std::vector<uint32_t> u32(3 * (size_t)Q);
  std::vector<int64_t> i64(2 * (size_t)Q);
  std::vector<crane_tres_limit_t> tres(3 * (size_t)Q);
  for (uint32_t k = 0; k < Q; ++k) {
    u32[k] = qt->max_jobs_per_user[k]; u32[Q + k] = qt->max_jobs_per_account[k]; u32[2 * Q + k] = qt->max_jobs[k];
    i64[k] = qt->max_cpus_per_user_raw[k]; i64[Q + k] = qt->max_wall[k];
    tres[k] = qt->max_tres_per_user[k]; tres[Q + k] = qt->max_tres_per_account[k]; tres[2 * Q + k] = qt->max_tres[k];
  }
  H2D(h->d_q_u32, u32.data(), u32.size());
  H2D(h->d_q_i64, i64.data(), i64.size());
  H2D(h->d_q_tres, tres.data(), tres.size());
  H2D(h->d_q_valid, qt->valid, Q);
  H2D(h->d_q_chain_off, qt->chain_off, N + 1);
  H2D(h->d_q_chain, qt->chain_acct, qt->chain_off[N]);
  H2D(h->d_q_user_usage, qt->user_usage, (size_t)U * Q);
  H2D(h->d_q_acct_usage, qt->account_usage, (size_t)A * Q);
  H2D(h->d_q_qos_usage, qt->qos_usage, Q);
  QosDev q{};
  q.n_qos = Q; q.n_users = U; q.n_accounts = A; q.n_jobs = N;
  q.valid = h->d_q_valid.p;
  q.max_jobs_per_user = h->d_q_u32.p; q.max_jobs_per_account = h->d_q_u32.p + Q; q.max_jobs = h->d_q_u32.p + 2 * Q;
  q.max_cpus_per_user_raw = h->d_q_i64.p; q.max_wall = h->d_q_i64.p + Q;
  q.tres_user = h->d_q_tres.p; q.tres_account = h->d_q_tres.p + Q; q.tres_qos = h->d_q_tres.p + 2 * Q;
  q.chain_off = h->d_q_chain_off.p; q.chain_acct = h->d_q_chain.p;
  q.user_usage = h->d_q_user_usage.p; q.account_usage = h->d_q_acct_usage.p; q.qos_usage = h->d_q_qos_usage.p;
  q.qos = h->pd.d_qos.p; q.user = h->pd.d_user.p; q.time_limit = h->pd.d_time_limit.p;
  q.n_alloc = h->outputs.d_nalloc.p; q.alloc_off = h->pd.d_alloc_off.p; q.alloc_res = h->outputs.d_res.p;
  q.reason = h->outputs.d_reason.p;
  if (N) {
    // the jobs the pass walks, grouped by qos in job-id order: key + stable radix sort
    const int bits = Q < 255 ? 8 : 16;
    const uint64_t sentinel = (1ull << bits) - 1;
    CU(cudaEventRecord(h->ev[kEvQosBegin], h->stream));
    CU(h->work.ensure_sort(N));
    CRANE_LAUNCH(k_qos_keys, (N + 255) / 256, 256, 0, h->stream, q, h->work.d_keys_a.p, h->work.d_vals_a.p, sentinel);
    uint64_t* keys;
    uint32_t* list;
    TRY(radix_sort(h, N, bits, &keys, &list));
    CU(h->d_q_off.ensure((size_t)Q + 1));
    CRANE_LAUNCH(k_qos_offsets, (Q + 1 + 127) / 128, 128, 0, h->stream, keys, N, Q, h->d_q_off.p);
    // the usage column of one qos in shared memory when it fits beside the job buffers
    const size_t table_bytes = ((size_t)U + A) * sizeof(crane_meta_resource_t);
    const bool force_global = getenv("CRANE_QOS_TABLES_GLOBAL") != nullptr;  // tests: the path of tables that do not fit
    const uint32_t in_smem = !force_global && table_bytes + 40 * 1024 <= h->v2_budget ? 1u : 0u;
    const size_t dyn = in_smem ? table_bytes : 0;
    CU(cudaFuncSetAttribute(k_qos_chain, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)dyn));
    CRANE_LAUNCH(k_qos_chain, Q, kQosThreads, dyn, h->stream, q, h->layout.dict, list, h->d_q_off.p, in_smem);
    CU(cudaGetLastError());
    CU(cudaEventRecord(h->ev[kEvQosEnd], h->stream));
    h->timing.kernel_launches += 3;
  }
  if (N) CU(cudaMemcpyAsync(reason, h->outputs.d_reason.p, N, cudaMemcpyDeviceToHost, h->stream));
  if ((size_t)U * Q) CU(cudaMemcpyAsync(qt->user_usage, h->d_q_user_usage.p, (size_t)U * Q * sizeof(crane_meta_resource_t), cudaMemcpyDeviceToHost, h->stream));
  if ((size_t)A * Q) CU(cudaMemcpyAsync(qt->account_usage, h->d_q_acct_usage.p, (size_t)A * Q * sizeof(crane_meta_resource_t), cudaMemcpyDeviceToHost, h->stream));
  CU(cudaMemcpyAsync(qt->qos_usage, h->d_q_qos_usage.p, (size_t)Q * sizeof(crane_meta_resource_t), cudaMemcpyDeviceToHost, h->stream));
  CU(cudaStreamSynchronize(h->stream));
  h->timing.qos_ms = N ? elapsed_ms(h, kEvQosBegin, kEvQosEnd) : 0.f;
  return CRANE_OK;
}

int crane_sched_schedule_steps(crane_sched_t* h, const crane_step_jobs_t* jb, const crane_steps_t* st,
                               crane_step_placements_t* out, float* device_ms) {
  if (!h || !jb || !st || !out) return CRANE_EINVAL;
  TRY(require(h, kCluster, "schedule_steps"));
  const uint32_t J = jb->n_jobs;
  TRY(check_step_jobs(h, jb));
  TRY(check_offsets(h, "step jobs: step_off", jb->step_off, J));
  const uint32_t E = jb->node_off[J], S = jb->step_off[J];
  if (st->n != S) return fail(h, CRANE_EINVAL, "steps: n (%u) != step_off[n_jobs] (%u)", st->n, S);
  uint64_t nrows = 0, trows = 0;
  TRY(check_steps(h, st, &nrows, &trows));
  if ((J && !out->placed) || (S && (!out->scheduled || !out->node_off || !out->task_off)) || !out->node_off || !out->task_off ||
      (nrows && (!out->alloc_node || !out->alloc_ntasks || !out->alloc_res)) || (trows && (!out->task_node || !out->task_res)))
    return fail(h, CRANE_EINVAL, "step placements: null column");
  CU(cudaSetDevice(h->device));
  (void)cudaGetLastError();
  cudaStream_t sm = h->stream;

  // one u32 table, one row table, one view table: three copies in, five out
  std::vector<uint32_t> u;
  u.reserve((size_t)3 * J + E + 8 * (size_t)S + 8);
  auto put = [&](const uint32_t* p, size_t n) { size_t at = u.size(); u.insert(u.end(), p, p + n); return at; };
  const size_t o_noff = put(jb->node_off, (size_t)J + 1);
  const size_t o_node = put(jb->node, E);
  const size_t o_soff = put(jb->step_off, (size_t)J + 1);
  const size_t o_nn = put(st->node_num, S), o_nt = put(st->ntasks, S);
  const size_t o_t0 = put(st->ntasks_per_node_min, S), o_t1 = put(st->ntasks_per_node_max, S);
  size_t o_io = 0, o_in = 0, o_eo = 0, o_en = 0;
  if (st->incl_off) { o_io = put(st->incl_off, (size_t)S + 1); o_in = put(st->incl_nodes, st->incl_off[S]); }
  if (st->excl_off) { o_eo = put(st->excl_off, (size_t)S + 1); o_en = put(st->excl_nodes, st->excl_off[S]); }
  out->node_off[0] = 0;
  out->task_off[0] = 0;
  for (uint32_t s = 0; s < S; ++s) {
    out->node_off[s + 1] = out->node_off[s] + st->node_num[s];
    out->task_off[s + 1] = out->task_off[s] + st->ntasks[s];
  }
  const size_t o_ooff = put(out->node_off, (size_t)S + 1), o_toff = put(out->task_off, (size_t)S + 1);
  const size_t n_in = u.size();
  const size_t o_placed = n_in, o_anode = o_placed + J, o_antasks = o_anode + nrows, o_tnode = o_antasks + nrows;
  const size_t n_u32 = o_tnode + trows;
  CU(h->d_steps_u32.ensure(std::max<size_t>(n_u32, 1)));
  CU(h->d_steps_rows.ensure(std::max<size_t>(E + nrows + trows, 1)));
  CU(h->d_steps_views.ensure(std::max<size_t>(2 * (size_t)S, 1)));
  CU(h->d_steps_sched.ensure(std::max<size_t>(S, 1)));
  uint32_t* du = h->d_steps_u32.p;
  Row* dr = h->d_steps_rows.p;
  View* dv = h->d_steps_views.p;
  CU(cudaMemcpyAsync(du, u.data(), n_in * sizeof(uint32_t), cudaMemcpyHostToDevice, sm));
  if (n_u32 > n_in) CU(cudaMemsetAsync(du + n_in, 0, (n_u32 - n_in) * sizeof(uint32_t), sm));
  if (E) CU(cudaMemcpyAsync(dr, jb->avail, E * sizeof(Row), cudaMemcpyHostToDevice, sm));
  if (nrows + trows) CU(cudaMemsetAsync(dr + E, 0, (nrows + trows) * sizeof(Row), sm));
  if (S) {
    CU(cudaMemcpyAsync(dv, st->req_node, S * sizeof(View), cudaMemcpyHostToDevice, sm));
    CU(cudaMemcpyAsync(dv + S, st->req_task, S * sizeof(View), cudaMemcpyHostToDevice, sm));
    CU(cudaMemsetAsync(h->d_steps_sched.p, 0, S, sm));
  }
  StepJobsDev dj{J, du + o_noff, du + o_node, dr, du + o_soff};
  StepsDev ds{du + o_nn, du + o_nt, du + o_t0, du + o_t1, dv, dv + S,
              st->incl_off ? du + o_io : nullptr, du + o_in, st->excl_off ? du + o_eo : nullptr, du + o_en};
  StepOutDev dout{du + o_placed, h->d_steps_sched.p, du + o_ooff, du + o_anode, du + o_antasks, dr + E,
                  du + o_toff, du + o_tnode, dr + E + nrows};
  CU(cudaEventRecord(h->ev[kEvStepsBegin], sm));
  if (J) {
    launch_steps(h, dj, ds, dout);
    CU(cudaGetLastError());
  }
  CU(cudaEventRecord(h->ev[kEvStepsEnd], sm));
  if (J) CU(cudaMemcpyAsync(out->placed, du + o_placed, J * sizeof(uint32_t), cudaMemcpyDeviceToHost, sm));
  if (S) CU(cudaMemcpyAsync(out->scheduled, h->d_steps_sched.p, S, cudaMemcpyDeviceToHost, sm));
  if (nrows) {
    CU(cudaMemcpyAsync(out->alloc_node, du + o_anode, nrows * sizeof(uint32_t), cudaMemcpyDeviceToHost, sm));
    CU(cudaMemcpyAsync(out->alloc_ntasks, du + o_antasks, nrows * sizeof(uint32_t), cudaMemcpyDeviceToHost, sm));
    CU(cudaMemcpyAsync(out->alloc_res, dr + E, nrows * sizeof(Row), cudaMemcpyDeviceToHost, sm));
  }
  if (trows) {
    CU(cudaMemcpyAsync(out->task_node, du + o_tnode, trows * sizeof(uint32_t), cudaMemcpyDeviceToHost, sm));
    CU(cudaMemcpyAsync(out->task_res, dr + E + nrows, trows * sizeof(Row), cudaMemcpyDeviceToHost, sm));
  }
  if (E) CU(cudaMemcpyAsync(jb->avail, dr, E * sizeof(Row), cudaMemcpyDeviceToHost, sm));
  CU(cudaStreamSynchronize(sm));
  CU(cudaGetLastError());
  if (device_ms) *device_ms = elapsed_ms(h, kEvStepsBegin, kEvStepsEnd);
  return CRANE_OK;
}

int crane_sched_step_jobs_reset(crane_sched_t* h) {
  if (!h) return CRANE_EINVAL;
  TRY(require(h, kCluster, "step_jobs_reset"));
  h->sj.reset();
  h->sp.reset();
  h->sr.valid = false;
  return CRANE_OK;
}

int crane_sched_step_jobs_start(crane_sched_t* h, const uint32_t* rows, uint32_t n, uint32_t* first) {
  if (!h) return CRANE_EINVAL;
  TRY(require(h, kCluster, "step_jobs_start"));
  TRY(check_rows(h, "step_jobs_start", rows, n, h->rr.n, [&](uint32_t r) { return h->rr.h_dead[r] != 0; }));
  CU(cudaSetDevice(h->device));
  h->sr.valid = false;
  cudaStream_t st = h->stream;
  const uint32_t base = h->sj.n, eb = h->sj.h_node_off.back();
  std::vector<uint32_t> off(n + 1, eb);
  for (uint32_t k = 0; k < n; ++k) {
    const uint64_t e = (uint64_t)off[k] + (h->rr.h_rr_alloc_off[rows[k] + 1] - h->rr.h_rr_alloc_off[rows[k]]);
    if (e > 0xfffffff0ull || (uint64_t)base + n > 0xfffffff0ull) return fail(h, CRANE_EINVAL, "step_jobs_start: too many rows");
    off[k + 1] = (uint32_t)e;
  }
  if (n) {
    CU(h->sj.d_node.grow(off[n], eb, st));
    CU(h->sj.d_avail.grow(off[n], eb, st));
    H2D_AT(h->sj.d_node_off, off.data(), base, (size_t)n + 1);
    H2D(h->d_sp_call, rows, n);
    CU(h->d_flag.ensure(1));
    CU(cudaMemsetAsync(h->d_flag.p, 0, sizeof(uint32_t), st));
    CRANE_LAUNCH(k_sj_seed, warp_grid(h, n), 256, 0, st, h->rr.d_rr_alloc_off.p, h->rr.d_rr_alloc_node.p, h->rr.d_rr_alloc_res.p,
                 h->d_sp_call.p, n, h->sj.d_node_off.p + base, h->sj.d_node.p, h->sj.d_avail.p, h->d_flag.p);
    uint32_t bad = 0;
    CU(cudaMemcpyAsync(&bad, h->d_flag.p, sizeof(uint32_t), cudaMemcpyDeviceToHost, st));
    CU(cudaStreamSynchronize(st));
    CU(cudaGetLastError());
    if (bad) return fail(h, CRANE_EINVAL, "step_jobs_start: a running row's allocation nodes are not ascending and distinct");
  }
  h->sj.commit(off);
  if (first) *first = base;
  return CRANE_OK;
}

int crane_sched_step_jobs_append(crane_sched_t* h, const crane_step_jobs_t* jb, uint32_t* first) {
  if (!h || !jb) return CRANE_EINVAL;
  TRY(require(h, kCluster, "step_jobs_append"));
  if (jb->step_off) return fail(h, CRANE_EINVAL, "step_jobs_append: step_off must be NULL (steps come with steps_append)");
  TRY(check_step_jobs(h, jb));
  const uint32_t J = jb->n_jobs, E = jb->node_off[J];
  const uint32_t base = h->sj.n, eb = h->sj.h_node_off.back();
  if ((uint64_t)eb + E > 0xfffffff0ull || (uint64_t)base + J > 0xfffffff0ull)
    return fail(h, CRANE_EINVAL, "step_jobs_append: too many rows");
  CU(cudaSetDevice(h->device));
  h->sr.valid = false;
  std::vector<uint32_t> off(J + 1);
  for (uint32_t j = 0; j <= J; ++j) off[j] = eb + jb->node_off[j];
  H2D_AT(h->sj.d_node_off, off.data(), base, (size_t)J + 1);
  H2D_AT(h->sj.d_node, jb->node, eb, E);
  H2D_AT(h->sj.d_avail, reinterpret_cast<const Row*>(jb->avail), eb, E);
  CU(cudaStreamSynchronize(h->stream));  // (the staging vector is pageable)
  h->sj.commit(off);
  if (first) *first = base;
  return CRANE_OK;
}

int crane_sched_step_jobs_erase(crane_sched_t* h, const uint32_t* rows, uint32_t n) {
  if (!h) return CRANE_EINVAL;
  TRY(require(h, kCluster, "step_jobs_erase"));
  TRY(check_rows(h, "step_jobs_erase", rows, n, h->sj.n, [&](uint32_t r) { return h->sj.h_dead[r] != 0; }));
  h->sr.valid = false;
  for (uint32_t k = 0; k < n; ++k) {  // its step rows go with it: every check looks at the job
    h->sj.h_dead[rows[k]] = 1;
    std::vector<uint32_t>().swap(h->sj.h_queue[rows[k]]);
  }
  return CRANE_OK;
}

int crane_sched_steps_append(crane_sched_t* h, const crane_steps_t* st, const uint32_t* job_row, uint32_t* first) {
  if (!h || !st) return CRANE_EINVAL;
  TRY(require(h, kCluster, "steps_append"));
  const uint32_t S = st->n;
  uint64_t nrows = 0, trows = 0;
  TRY(check_steps(h, st, &nrows, &trows));
  if (S && !job_row) return fail(h, CRANE_EINVAL, "steps_append: null job_row");
  for (uint32_t s = 0; s < S; ++s) {
    if (job_row[s] >= h->sj.n) return fail(h, CRANE_EINVAL, "steps_append[%u]: job row %u out of range", s, job_row[s]);
    if (h->sj.h_dead[job_row[s]]) return fail(h, CRANE_EINVAL, "steps_append[%u]: job row %u was erased", s, job_row[s]);
  }
  const uint32_t base = h->sp.n, ib = h->sp.h_incl_off.back(), xb = h->sp.h_excl_off.back();
  const uint32_t ni = st->incl_off ? st->incl_off[S] : 0, nx = st->excl_off ? st->excl_off[S] : 0;
  if ((uint64_t)base + S > 0xfffffff0ull || (uint64_t)ib + ni > 0xfffffff0ull || (uint64_t)xb + nx > 0xfffffff0ull)
    return fail(h, CRANE_EINVAL, "steps_append: too many rows");
  CU(cudaSetDevice(h->device));
  h->sr.valid = false;
  std::vector<uint32_t> io(S + 1), xo(S + 1);
  for (uint32_t s = 0; s <= S; ++s) {
    io[s] = ib + (st->incl_off ? st->incl_off[s] : 0);
    xo[s] = xb + (st->excl_off ? st->excl_off[s] : 0);
  }
  H2D_AT(h->sp.d_job, job_row, base, S);
  H2D_AT(h->sp.d_nn, st->node_num, base, S);
  H2D_AT(h->sp.d_nt, st->ntasks, base, S);
  H2D_AT(h->sp.d_t0, st->ntasks_per_node_min, base, S);
  H2D_AT(h->sp.d_t1, st->ntasks_per_node_max, base, S);
  H2D_AT(h->sp.d_req_node, reinterpret_cast<const View*>(st->req_node), base, S);
  H2D_AT(h->sp.d_req_task, reinterpret_cast<const View*>(st->req_task), base, S);
  H2D_AT(h->sp.d_incl_off, io.data(), base, (size_t)S + 1);
  H2D_AT(h->sp.d_excl_off, xo.data(), base, (size_t)S + 1);
  H2D_AT(h->sp.d_incl, st->incl_nodes, ib, ni);
  H2D_AT(h->sp.d_excl, st->excl_nodes, xb, nx);
  CU(h->sp.d_alloc_at.grow(std::max<size_t>((size_t)base + S, 1), base, h->stream));
  CU(cudaStreamSynchronize(h->stream));  // (the staging vectors are pageable)
  for (uint32_t s = 0; s < S; ++s) {
    h->sp.h_job.push_back(job_row[s]);
    h->sp.h_nn.push_back(st->node_num[s]);
    h->sp.h_nt.push_back(st->ntasks[s]);
    h->sp.h_state.push_back(kSpPending);
    h->sp.h_incl_off.push_back(io[s + 1]);
    h->sp.h_excl_off.push_back(xo[s + 1]);
    h->sj.h_queue[job_row[s]].push_back(base + s);
    h->sj.mark_dirty(job_row[s]);
  }
  h->sp.n = base + S;
  if (first) *first = base;
  return CRANE_OK;
}

int crane_sched_steps_erase(crane_sched_t* h, const uint32_t* rows, uint32_t n) {
  if (!h) return CRANE_EINVAL;
  TRY(require(h, kCluster, "steps_erase"));
  TRY(check_rows(h, "steps_erase", rows, n, h->sp.n, [&](uint32_t r) {
    return h->sp.h_state[r] == kSpErased || h->sj.h_dead[h->sp.h_job[r]];
  }));
  CU(cudaSetDevice(h->device));
  h->sr.valid = false;
  // scheduled rows give their node rows back, job by job, in row order
  std::vector<std::pair<uint32_t, uint32_t>> rel;  // (job, step row)
  for (uint32_t k = 0; k < n; ++k) {
    const uint32_t s = rows[k], j = h->sp.h_job[s];
    if (h->sp.h_state[s] == kSpScheduled) {
      rel.emplace_back(j, s);
    } else {
      auto& q = h->sj.h_queue[j];
      q.erase(std::find(q.begin(), q.end(), s));
    }
    h->sp.h_state[s] = kSpErased;
    h->sj.mark_dirty(j);
  }
  if (rel.empty()) return CRANE_OK;
  std::sort(rel.begin(), rel.end());
  std::vector<uint32_t> jobs, off{0}, steps;  // uploaded as one table: jobs | off | steps
  for (size_t q = 0; q < rel.size(); ++q) {
    if (q == 0 || rel[q].first != rel[q - 1].first) {
      if (q) off.push_back((uint32_t)q);
      jobs.push_back(rel[q].first);
    }
    steps.push_back(rel[q].second);
  }
  off.push_back((uint32_t)rel.size());
  const uint32_t m = (uint32_t)jobs.size();
  std::vector<uint32_t> u(jobs);
  u.insert(u.end(), off.begin(), off.end());
  u.insert(u.end(), steps.begin(), steps.end());
  H2D(h->d_sp_call, u.data(), u.size());
  const uint32_t* du = h->d_sp_call.p;
  CRANE_LAUNCH(k_sp_release, warp_grid(h, m), 256, 0, h->stream, step_pool(h->sj, h->sp), du, du + m, du + 2 * m + 1, m);
  CU(cudaGetLastError());
  CU(cudaStreamSynchronize(h->stream));
  return CRANE_OK;
}

int crane_sched_steps_run(crane_sched_t* h, uint32_t* n_scheduled, uint32_t* n_node_rows, uint32_t* n_task_rows,
                          float* device_ms) {
  if (!h) return CRANE_EINVAL;
  TRY(require(h, kCluster, "steps_run"));
  CU(cudaSetDevice(h->device));
  (void)cudaGetLastError();
  cudaStream_t sm = h->stream;
  h->sr.clear();
  h->sr.sa_base = h->sp.n_alloc;
  // the pass visits the dirty jobs with a live pending step, ascending, each with its queue
  std::sort(h->sj.h_dirty_rows.begin(), h->sj.h_dirty_rows.end());
  std::vector<uint32_t> u;  // jl | sl
  for (uint32_t j : h->sj.h_dirty_rows) {
    h->sj.h_dirty[j] = 0;
    if (!h->sj.h_dead[j] && !h->sj.h_queue[j].empty()) u.push_back(j);
  }
  h->sj.h_dirty_rows.clear();
  const uint32_t J = (uint32_t)u.size();
  uint64_t E = 0, Li = 0, Le = 0, N = 0, T = 0;
  for (uint32_t w = 0; w < J; ++w) {
    const uint32_t j = u[w];
    E += h->sj.h_node_off[j + 1] - h->sj.h_node_off[j];
    for (uint32_t s : h->sj.h_queue[j]) {
      u.push_back(s);
      Li += h->sp.h_incl_off[s + 1] - h->sp.h_incl_off[s];
      Le += h->sp.h_excl_off[s + 1] - h->sp.h_excl_off[s];
      N += h->sp.h_nn[s];
      T += h->sp.h_nt[s];
    }
  }
  const uint32_t S = (uint32_t)(u.size() - J);
  if (N > 0xfffffff0ull || T > 0xfffffff0ull || (uint64_t)h->sp.n_alloc + N > 0xfffffff0ull)
    return fail(h, CRANE_EINVAL, "steps_run: too many node / task rows");
  float ms = 0.f;
  if (J) {
    // dense u32 columns: jl | sl | node_off | node | step_off | nn | nt | t0 | t1 | incl_off | incl | excl_off | excl |
    //                    out node_off | out task_off | placed | alloc_node | alloc_ntasks | task_node | pos
    size_t at = 0;
    auto take = [&](uint64_t n) { const size_t a = at; at += n; return a; };
    const size_t o_jl = take(J), o_sl = take(S), o_noff = take(J + 1), o_node = take(E), o_soff = take(J + 1);
    const size_t o_nn = take(S), o_nt = take(S), o_t0 = take(S), o_t1 = take(S);
    const size_t o_io = take(S + 1), o_in = take(Li), o_xo = take(S + 1), o_xn = take(Le);
    const size_t o_ooff = take(S + 1), o_toff = take(S + 1), o_placed = take(J);
    const size_t o_anode = take(N), o_antasks = take(N), o_tnode = take(T), o_pos = take(2 * (uint64_t)S);
    CU(h->d_steps_u32.ensure(at));
    CU(h->d_steps_rows.ensure(std::max<uint64_t>(E + N + T, 1)));
    CU(h->d_steps_views.ensure(2 * (size_t)S));
    CU(h->d_steps_sched.ensure(S));
    uint32_t* du = h->d_steps_u32.p;
    Row* dr = h->d_steps_rows.p;
    StepPassDev d{};
    d.n_jobs = J;
    d.n_steps = S;
    d.jl = du + o_jl;
    d.sl = du + o_sl;
    d.node_off = du + o_noff;
    d.node = du + o_node;
    d.avail = dr;
    d.step_off = du + o_soff;
    d.node_num = du + o_nn;
    d.ntasks = du + o_nt;
    d.ntpn_min = du + o_t0;
    d.ntpn_max = du + o_t1;
    d.req_node = h->d_steps_views.p;
    d.req_task = h->d_steps_views.p + S;
    d.incl_off = du + o_io;
    d.incl_nodes = du + o_in;
    d.excl_off = du + o_xo;
    d.excl_nodes = du + o_xn;
    d.out_node_off = du + o_ooff;
    d.out_task_off = du + o_toff;
    d.placed = du + o_placed;
    d.scheduled = h->d_steps_sched.p;
    d.alloc_node = du + o_anode;
    d.alloc_ntasks = du + o_antasks;
    d.task_node = du + o_tnode;
    d.alloc_res = dr + E;
    d.task_res = dr + E + N;
    CU(cudaMemcpyAsync(du, u.data(), u.size() * sizeof(uint32_t), cudaMemcpyHostToDevice, sm));
    CU(cudaEventRecord(h->ev[kEvSpBegin], sm));
    const uint32_t mx = std::max(J, S) + 1;
    CRANE_LAUNCH(k_sp_pass_cols, std::min<uint32_t>((mx + 255) / 256, 8 * h->n_sm), 256, 0, sm, step_pool(h->sj, h->sp), d);
    ScanSegs sg{{d.node_off, d.incl_off, d.excl_off, d.out_node_off, d.out_task_off}, {J + 1, S + 1, S + 1, S + 1, S + 1}};
    CRANE_LAUNCH(k_sp_scan, 1, 1024, 0, sm, sg);
    CRANE_LAUNCH(k_sp_pass_rows, warp_grid(h, (uint64_t)J + S), 256, 0, sm, step_pool(h->sj, h->sp), d);
    StepJobsDev dj{J, d.node_off, d.node, d.avail, d.step_off};
    StepsDev ds{d.node_num, d.ntasks, d.ntpn_min, d.ntpn_max, d.req_node, d.req_task,
                d.incl_off, d.incl_nodes, d.excl_off, d.excl_nodes};
    StepOutDev dout{d.placed, d.scheduled, d.out_node_off, d.alloc_node, d.alloc_ntasks, d.alloc_res,
                    d.out_task_off, d.task_node, d.task_res};
    launch_steps(h, dj, ds, dout);
    CU(cudaEventRecord(h->ev[kEvSpMid], sm));
    std::vector<uint8_t> sched(S);
    CU(cudaMemcpyAsync(sched.data(), d.scheduled, S, cudaMemcpyDeviceToHost, sm));
    CU(cudaStreamSynchronize(sm));
    CU(cudaGetLastError());
    // the results are the scheduled steps in ascending step-row order: their row positions
    std::vector<std::pair<uint32_t, uint32_t>> got;  // (step row, pass index)
    for (uint32_t i = 0; i < S; ++i)
      if (sched[i]) got.emplace_back(u[J + i], i);
    std::sort(got.begin(), got.end());
    std::vector<uint32_t> pos(2 * (size_t)S, 0);
    for (const auto& g : got) {
      const uint32_t s = g.first;
      pos[2 * (size_t)g.second] = h->sr.h_node_off.back();
      pos[2 * (size_t)g.second + 1] = h->sr.h_task_off.back();
      h->sr.h_rows.push_back(s);
      h->sr.h_node_off.push_back(h->sr.h_node_off.back() + h->sp.h_nn[s]);
      h->sr.h_task_off.push_back(h->sr.h_task_off.back() + h->sp.h_nt[s]);
    }
    const uint32_t Nr = h->sr.h_node_off.back(), Tr = h->sr.h_task_off.back();
    if (!got.empty()) {
      CU(h->sp.d_sa_node.grow((size_t)h->sp.n_alloc + Nr, h->sp.n_alloc, sm));
      CU(h->sp.d_sa_res.grow((size_t)h->sp.n_alloc + Nr, h->sp.n_alloc, sm));
      CU(h->sr.d_u32.ensure((size_t)Nr + Tr));
      CU(h->sr.d_rows.ensure(std::max<uint32_t>(Tr, 1)));
      CU(cudaMemcpyAsync(du + o_pos, pos.data(), pos.size() * sizeof(uint32_t), cudaMemcpyHostToDevice, sm));
      CU(cudaEventRecord(h->ev[kEvSpScatter], sm));
      CRANE_LAUNCH(k_sp_scatter, warp_grid(h, (uint64_t)J + S), 256, 0, sm, step_pool(h->sj, h->sp), d, du + o_pos,
                   h->sp.n_alloc, h->sr.d_u32.p, h->sr.d_u32.p + Nr, h->sr.d_rows.p);
      CU(cudaEventRecord(h->ev[kEvSpEnd], sm));
      CU(cudaStreamSynchronize(sm));
      CU(cudaGetLastError());
      ms = elapsed_ms(h, kEvSpScatter, kEvSpEnd);
    }
    ms += elapsed_ms(h, kEvSpBegin, kEvSpMid);
    // mirrors: the scheduled steps are the head of their job's queue
    uint32_t i = 0;
    for (uint32_t w = 0; w < J; ++w) {
      auto& q = h->sj.h_queue[u[w]];
      size_t k = 0;
      for (const size_t len = q.size(); k < len && sched[i + k]; ++k) h->sp.h_state[q[k]] = kSpScheduled;
      i += (uint32_t)q.size();
      q.erase(q.begin(), q.begin() + k);
    }
    h->sp.n_alloc += Nr;
  }
  if (n_scheduled) *n_scheduled = (uint32_t)h->sr.h_rows.size();
  if (n_node_rows) *n_node_rows = h->sr.h_node_off.back();
  if (n_task_rows) *n_task_rows = h->sr.h_task_off.back();
  if (device_ms) *device_ms = ms;
  h->sr.valid = true;
  return CRANE_OK;
}

int crane_sched_steps_fetch(crane_sched_t* h, crane_step_results_t* out) {
  if (!h || !out) return CRANE_EINVAL;
  if (!h->sr.valid) return fail(h, CRANE_EINVAL, "steps_fetch: steps_run first");
  const size_t Ns = h->sr.h_rows.size(), N = h->sr.h_node_off.back(), T = h->sr.h_task_off.back();
  if (!out->node_off || !out->task_off || (Ns && !out->step_row) ||
      (N && (!out->alloc_node || !out->alloc_ntasks || !out->alloc_res)) || (T && (!out->task_node || !out->task_res)))
    return fail(h, CRANE_EINVAL, "step results: null column");
  CU(cudaSetDevice(h->device));
  cudaStream_t sm = h->stream;
  if (Ns) memcpy(out->step_row, h->sr.h_rows.data(), Ns * sizeof(uint32_t));
  memcpy(out->node_off, h->sr.h_node_off.data(), (Ns + 1) * sizeof(uint32_t));
  memcpy(out->task_off, h->sr.h_task_off.data(), (Ns + 1) * sizeof(uint32_t));
  if (N) {
    CU(cudaMemcpyAsync(out->alloc_node, h->sp.d_sa_node.p + h->sr.sa_base, N * sizeof(uint32_t), cudaMemcpyDeviceToHost, sm));
    CU(cudaMemcpyAsync(out->alloc_res, h->sp.d_sa_res.p + h->sr.sa_base, N * sizeof(Row), cudaMemcpyDeviceToHost, sm));
    CU(cudaMemcpyAsync(out->alloc_ntasks, h->sr.d_u32.p, N * sizeof(uint32_t), cudaMemcpyDeviceToHost, sm));
  }
  if (T) {
    CU(cudaMemcpyAsync(out->task_node, h->sr.d_u32.p + N, T * sizeof(uint32_t), cudaMemcpyDeviceToHost, sm));
    CU(cudaMemcpyAsync(out->task_res, h->sr.d_rows.p, T * sizeof(Row), cudaMemcpyDeviceToHost, sm));
  }
  CU(cudaStreamSynchronize(sm));
  return CRANE_OK;
}

int crane_sched_step_jobs_avail(crane_sched_t* h, const uint32_t* rows, uint32_t n, crane_res_in_node_t* dst,
                                uint32_t* n_node_rows) {
  if (!h) return CRANE_EINVAL;
  TRY(require(h, kCluster, "step_jobs_avail"));
  TRY(check_rows(h, "step_jobs_avail", rows, n, h->sj.n, [&](uint32_t r) { return h->sj.h_dead[r] != 0; }));
  std::vector<uint32_t> u(rows, rows + n);  // rows | dst_off
  u.push_back(0);
  for (uint32_t k = 0; k < n; ++k) u.push_back(u.back() + h->sj.h_node_off[rows[k] + 1] - h->sj.h_node_off[rows[k]]);
  const uint32_t E = u.back();
  if (n_node_rows) *n_node_rows = E;
  CU(cudaSetDevice(h->device));
  h->sr.valid = false;
  if (!E || !dst) return CRANE_OK;
  H2D(h->d_sp_call, u.data(), u.size());
  CU(h->d_steps_rows.ensure(E));
  CRANE_LAUNCH(k_sj_avail_gather, warp_grid(h, n), 256, 0, h->stream, h->sj.d_node_off.p, h->sj.d_avail.p,
               h->d_sp_call.p, h->d_sp_call.p + n, n, h->d_steps_rows.p);
  CU(cudaMemcpyAsync(dst, h->d_steps_rows.p, (size_t)E * sizeof(Row), cudaMemcpyDeviceToHost, h->stream));
  CU(cudaStreamSynchronize(h->stream));
  CU(cudaGetLastError());
  return CRANE_OK;
}

int crane_sched_step_rows(const crane_sched_t* h, uint32_t* step_jobs, uint32_t* steps, uint32_t* alloc_rows) {
  if (!h) return CRANE_EINVAL;
  if (step_jobs) *step_jobs = h->sj.n;
  if (steps) *steps = h->sp.n;
  if (alloc_rows) *alloc_rows = h->sp.n_alloc;
  return CRANE_OK;
}

int crane_sched_steps_compact(crane_sched_t* h, uint32_t* step_job_map, uint32_t* step_map) {
  if (!h) return CRANE_EINVAL;
  TRY(require(h, kCluster, "steps_compact"));
  CU(cudaSetDevice(h->device));
  h->sr.valid = false;
  cudaStream_t st = h->stream;
  const StepsKept kp(h->sj, h->sp);
  const uint32_t J = h->sj.n, S = h->sp.n;
  if (kp.Jl < J || kp.Sl < S) {
    // ---- every new buffer before the first gather: CRANE_ENOMEM leaves the tables as they were ----
    StepJobTable sj;
    StepTable sp;
    TRY(steps_fresh(h, kp, sj, sp));
    H2D(h->d_sp_call, kp.u.data(), kp.u.size());
    // ---- gathers, then the new tables replace the old ones (whose buffers go with the locals) ----
    TRY(steps_copy(h, kp, sj, sp, h->d_sp_call.p));
    CU(cudaGetLastError());
    CU(cudaStreamSynchronize(st));
    std::swap(h->sj, sj);
    std::swap(h->sp, sp);
  }
  // (identity maps when nothing was erased)
  if (step_job_map) std::copy(kp.jmap.begin(), kp.jmap.end(), step_job_map);
  if (step_map) std::copy(kp.smap.begin(), kp.smap.end(), step_map);
  return CRANE_OK;
}

int crane_sched_get_timing(const crane_sched_t* h, crane_sched_timing_t* t) {
  if (!h || !t) return CRANE_EINVAL;
  *t = h->timing;
  return CRANE_OK;
}

int crane_sched_debug_bitmap(crane_sched_t* h, uint32_t* dst, size_t cap_words, uint32_t* rows,
                             uint32_t* words_per_row) {
  if (!h) return CRANE_EINVAL;
  TRY(require(h, kRan, "debug_bitmap"));
  CU(cudaSetDevice(h->device));
  uint32_t nq = 0;
  CU(cudaMemcpy(&nq, h->layout.d_part_job_off.p + h->layout.n_vparts, sizeof(uint32_t), cudaMemcpyDeviceToHost));
  if (rows) *rows = nq;
  if (words_per_row) *words_per_row = h->layout.words_per_row;
  size_t n = std::min(cap_words, (size_t)nq * h->layout.words_per_row);
  if (dst && n) CU(cudaMemcpy(dst, h->work.d_bitmap.p, n * sizeof(uint32_t), cudaMemcpyDeviceToHost));
  return CRANE_OK;
}

}  // extern "C"
