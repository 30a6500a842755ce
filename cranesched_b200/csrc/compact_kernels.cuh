// compact_kernels.cuh — sm_90a kernels of crane_sched_compact.
//
// The resident pending and running tables keep a row's index until the table is
// replaced, so erased rows stay behind as tombstones and resolved dependency entries
// stay behind retired. Compaction rewrites the tables with only their live rows and
// open entries, on the device, where the gate state lives:
//   live rows   k_rt_live_keys + the stable LSD radix sort (the regroup's): the live rows
//               first, in row order; k_cp_map scatters their ranks into the old -> new map
//   columns     one gather per table (k_cp_pending, k_cp_running): new row c = c-th live row
//   CSR tables  lengths of the live rows, their exclusive scan (k_sort_scan) and one warp
//               per row copying its entries (k_cp_csr)
//   entries     k_cp_ent_keys flags the open entries of live rows, the same sort lists them
//               in entry order, k_cp_entries copies them with dependent and dependee mapped
// Live rows and kept entries keep their order, so every order-sensitive step of a run
// (the stable priority sort, FIFO, the regroup's sorts and fp64 sums, account grouping)
// sees the same sequence as on the uncompacted tables.
#pragma once

#include "sched_kernels.cuh"
#include "running_kernels.cuh"
#include "gate_kernels.cuh"

namespace crane {

constexpr uint32_t kRowNone = 0xffffffffu;  // CRANE_ROW_NONE

// map[live[c]] = c; the other entries of map were set to kRowNone
__global__ void k_cp_map(const uint32_t* live, uint32_t n_live, uint32_t* map) {
  const uint32_t c = blockIdx.x * blockDim.x + threadIdx.x;
  if (c < n_live) map[live[c]] = c;
}

// The fixed-width columns of the pending table; optional columns are null when the table
// has none. Gate columns are copied for the new rows [0, gate_n).
struct PendingCols {
  uint32_t* partition;
  int64_t* time_limit;
  int64_t* submit_time;
  uint32_t* node_num;
  uint32_t* ntpn_min;
  uint32_t* ntpn_max;
  uint32_t* ntasks;
  uint8_t* exclusive;
  uint32_t* partition_priority;
  uint32_t* qos_priority;
  uint32_t* account;
  uint32_t* qos;
  uint32_t* user;
  double* mandated;
  uint32_t* reservation;
  View* req_node;
  View* req_task;
  View* req_total;
  uint8_t* held;
  int64_t* begin;
  uint8_t* is_or;
  uint32_t* open;
  long long* ready;
};

__global__ void k_cp_pending(PendingCols s, PendingCols d, const uint32_t* live, uint32_t n_live, uint32_t gate_n) {
  const uint32_t c = blockIdx.x * blockDim.x + threadIdx.x;
  if (c >= n_live) return;
  const uint32_t r = live[c];
  d.partition[c] = s.partition[r];
  d.time_limit[c] = s.time_limit[r];
  d.submit_time[c] = s.submit_time[r];
  d.node_num[c] = s.node_num[r];
  d.ntpn_min[c] = s.ntpn_min[r];
  d.ntpn_max[c] = s.ntpn_max[r];
  d.ntasks[c] = s.ntasks[r];
  d.exclusive[c] = s.exclusive[r];
  d.partition_priority[c] = s.partition_priority[r];
  d.qos_priority[c] = s.qos_priority[r];
  d.account[c] = s.account[r];
  if (d.qos) {
    d.qos[c] = s.qos[r];
    d.user[c] = s.user[r];
  }
  if (d.mandated) d.mandated[c] = s.mandated[r];
  if (d.reservation) d.reservation[c] = s.reservation[r];
  d.req_node[c] = s.req_node[r];
  d.req_task[c] = s.req_task[r];
  d.req_total[c] = s.req_total[r];
  if (c < gate_n) {
    d.held[c] = s.held[r];
    d.begin[c] = s.begin[r];
    d.is_or[c] = s.is_or[r];
    d.open[c] = s.open[r];
    d.ready[c] = s.ready[r];
  }
}

// The fixed-width columns of the running table (alloc_off, alloc_node, alloc_res and dead
// are not read: the CSR goes through k_cp_csr, the new rows are all live)
__global__ void k_cp_running(RunTableDev s, RunTableDev d, const uint32_t* live, uint32_t n_live) {
  const uint32_t c = blockIdx.x * blockDim.x + threadIdx.x;
  if (c >= n_live) return;
  const uint32_t r = live[c];
  d.start_time[c] = s.start_time[r];
  d.end_time[c] = s.end_time[r];
  d.node_num[c] = s.node_num[r];
  d.partition_priority[c] = s.partition_priority[r];
  d.qos_priority[c] = s.qos_priority[r];
  d.account[c] = s.account[r];
  d.reservation[c] = s.reservation[r];
  d.view_cpu_raw[c] = s.view_cpu_raw[r];
  d.view_mem[c] = s.view_mem[r];
}

// len[c] = entries of the c-th live row of a CSR table, len[n_live] = 0: the exclusive
// scan of len[0, n_live] is the new offsets
__global__ void k_cp_lengths(const uint32_t* off, const uint32_t* live, uint32_t n_live, uint32_t* len) {
  const uint32_t c = blockIdx.x * blockDim.x + threadIdx.x;
  if (c < n_live) len[c] = off[live[c] + 1] - off[live[c]];
  else if (c == n_live) len[c] = 0;
}

// One warp per live row: its entries of a CSR table at their new offsets
template <class T>
__global__ void k_cp_csr(const uint32_t* off, const T* src, const uint32_t* live, uint32_t n_live,
                         const uint32_t* new_off, T* dst) {
  const int lane = lane_id();
  const uint32_t warps = blockDim.x >> 5;
  for (uint32_t c = blockIdx.x * warps + warp_id(); c < n_live; c += gridDim.x * warps) {
    const uint32_t r = live[c], s0 = off[r], n = off[r + 1] - s0, d0 = new_off[c];
    for (uint32_t k = lane; k < n; k += 32) dst[d0 + k] = src[s0 + k];
  }
}

// keys = 1 for an entry that goes (retired, or its dependent row erased), vals = entry;
// *n_keep counts the others
__global__ void k_cp_ent_keys(GateDev g, const uint8_t* pd_dead, uint64_t* keys, uint32_t* vals, uint32_t* n_keep) {
  const uint32_t e = blockIdx.x * blockDim.x + threadIdx.x;
  bool keep = false;
  if (e < g.n_ent) {
    keep = g.live[e] && !(pd_dead && pd_dead[g.dependent[e]]);
    keys[e] = keep ? 0u : 1u;
    vals[e] = e;
  }
  const unsigned b = __ballot_sync(kFullMask, keep);
  if (lane_id() == 0 && b) atomicAdd(n_keep, (uint32_t)__popc(b));
}

// The kept entries in entry order: dependent through the pending map, dependee through
// the pending or the running map by kind (an erased dependee becomes kRowNone, which no
// event row matches); a null map is the identity. `delay` is the new delay column
// (GateDev's is read-only).
__global__ void k_cp_entries(GateDev s, GateDev d, uint64_t* delay, const uint32_t* keep, uint32_t n_keep,
                             const uint32_t* pd_map, const uint32_t* rr_map) {
  const uint32_t c = blockIdx.x * blockDim.x + threadIdx.x;
  if (c >= n_keep) return;
  const uint32_t e = keep[c];
  const uint8_t kind = s.kind[e];
  const uint32_t dependent = s.dependent[e];
  uint32_t q = s.dependee[e];
  const uint32_t* map = kind == kDepPending ? pd_map : kind == kDepRunning ? rr_map : nullptr;
  if (map && q != kRowNone) q = map[q];
  d.dependent[c] = pd_map ? pd_map[dependent] : dependent;
  d.dependee[c] = q;
  d.kind[c] = kind;
  d.type[c] = s.type[e];
  d.live[c] = 1;
  delay[c] = s.delay[e];
}

}  // namespace crane
