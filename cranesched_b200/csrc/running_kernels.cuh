// running_kernels.cuh — sm_90a kernels of the device-resident running table.
//
// The running table is a table of rows that keep their index until the table is
// replaced; an ended job's row becomes a tombstone. Jobs started by a run move into
// it on the device (k_start, the commit loop of JobScheduler.cpp:1273-1305), and
// before a run the regroup kernels build the tick's RunningDev view from the live
// rows: the dense per-job columns (k_bounds, k_service), the allocations grouped by
// node state (k_node_init) and the jobs grouped by account (k_service).
//
// The groupings are stable (a stable LSD radix sort): k_node_init sums the initial
// cost in fp64 in the order of a node state's entries and k_service the service
// value in the order of an account's jobs (deviation D6), so the view must list them
// in row order, exactly as the host regroup of a host running table did.
#pragma once

#include "sched_kernels.cuh"

namespace crane {

// The resident rows, tombstones included
struct RunTableDev {
  uint32_t n;
  int64_t* start_time;
  int64_t* end_time;
  uint32_t* node_num;
  uint32_t* partition_priority;
  uint32_t* qos_priority;
  uint32_t* account;
  uint32_t* reservation;    // 0xffffffff = none
  int64_t* view_cpu_raw;
  uint64_t* view_mem;
  uint32_t* alloc_off;      // [n+1] CSR over (node, res) entries
  uint32_t* alloc_node;
  Row* alloc_res;
  const uint8_t* dead;      // [n] tombstones
};

// What a running job's allocation on a node is looked up in: the node states of the
// partitions and of the reservations (crane_sched::build_layout)
struct NodeStateMap {
  uint32_t n_nodes, n_slots, n_comp, n_resv;
  const uint32_t* node_slot;   // [n_nodes] node -> slot of its partition, or 0xffffffff
  const uint32_t* part_base;   // [n_vparts+1]
  const uint32_t* r_node_off;  // [n_resv+1] nodes of each reservation, ascending
  const uint32_t* r_node;
};

// Node state a running job's allocation on `node` counts against: the node's own, or —
// for a job inside a reservation — the reservation's state of that node
// (JobScheduler.cpp:5715-5741); 0xffffffff = none (the reference skips it, :5719)
__device__ __forceinline__ uint32_t running_slot(const NodeStateMap& m, uint32_t rv, uint32_t node) {
  if (rv == 0xffffffffu) return m.node_slot[node];
  if (rv >= m.n_resv) return 0xffffffffu;  // the reference logs an error and skips the job
  uint32_t lo = m.r_node_off[rv], hi = m.r_node_off[rv + 1];
  const uint32_t first = lo;
  while (lo < hi) {  // lower_bound
    const uint32_t mid = lo + (hi - lo) / 2;
    if (m.r_node[mid] < node) lo = mid + 1;
    else hi = mid;
  }
  if (lo == m.r_node_off[rv + 1] || m.r_node[lo] != node) return 0xffffffffu;
  return m.part_base[m.n_comp + rv] + (lo - first);
}

// ------------------------------------------------------------------------
// crane_sched_start: the listed pending rows must hold a start-now placement
// ------------------------------------------------------------------------
__global__ void k_start_check(const uint32_t* rows, uint32_t n, const uint8_t* reason, uint32_t* bad) {
  const uint32_t k = blockIdx.x * blockDim.x + threadIdx.x;
  if (k < n && reason[rows[k]] != CRANE_REASON_NONE) atomicOr(bad, 1u);
}

// One warp per started job: its placement rows become the new running row base + i
// (allocated_res, JobScheduler.cpp:1276-1281); the view is the sum of the rows.
__global__ void k_start(PendingDev pd, PlaceDev out, const uint32_t* rows, uint32_t n, uint32_t base, RunTableDev rt) {
  const int lane = lane_id();
  const uint32_t warps = blockDim.x >> 5;
  for (uint32_t i = blockIdx.x * warps + warp_id(); i < n; i += gridDim.x * warps) {
    const uint32_t r = rows[i], dst = base + i;
    const uint32_t nn = pd.node_num[r], src = pd.alloc_off[r], d0 = rt.alloc_off[dst];
    long long cpu = 0;
    unsigned long long mem = 0;
    for (uint32_t k = lane; k < nn; k += 32) {
      const Row res = out.alloc_res[src + k];
      rt.alloc_node[d0 + k] = out.alloc_node[src + k];
      rt.alloc_res[d0 + k] = res;
      cpu += res.cpu_raw;
      mem += res.mem;
    }
    for (int o = 16; o > 0; o >>= 1) {
      cpu += __shfl_xor_sync(kFullMask, cpu, o);
      mem += __shfl_xor_sync(kFullMask, mem, o);
    }
    if (lane == 0) {
      rt.start_time[dst] = out.start_time[r];
      rt.end_time[dst] = out.end_time[r];
      rt.node_num[dst] = nn;
      rt.partition_priority[dst] = pd.partition_priority[r];
      rt.qos_priority[dst] = pd.qos_priority[r];
      rt.account[dst] = pd.account[r];
      rt.reservation[dst] = pd.reservation ? pd.reservation[r] : 0xffffffffu;
      rt.view_cpu_raw[dst] = (int64_t)cpu;
      rt.view_mem[dst] = (uint64_t)mem;
    }
  }
}

// ------------------------------------------------------------------------
// Regroup (crane_sched_keep_running)
// ------------------------------------------------------------------------
// keys = tombstone flag, vals = row: the stable sort puts the live rows first, in row order
__global__ void k_rt_live_keys(const uint8_t* dead, uint32_t n, uint64_t* keys, uint32_t* vals) {
  const uint32_t r = blockIdx.x * blockDim.x + threadIdx.x;
  if (r < n) {
    keys[r] = dead[r] ? 1u : 0u;
    vals[r] = r;
  }
}

// One warp per row: key of every allocation entry = its node state in bits 0-31 (n_slots
// for a tombstone or a node outside the node states, which sorts them last) and its row
// in bits 32-63; vals = the entry. A live entry on a node >= n_nodes raises *bad.
__global__ void k_rt_entry_keys(RunTableDev rt, NodeStateMap m, uint64_t* keys, uint32_t* vals, uint32_t* bad) {
  const int lane = lane_id();
  const uint32_t warps = blockDim.x >> 5;
  for (uint32_t r = blockIdx.x * warps + warp_id(); r < rt.n; r += gridDim.x * warps) {
    const bool dead = rt.dead[r] != 0;
    const uint32_t rv = rt.reservation[r];
    for (uint32_t k = rt.alloc_off[r] + lane; k < rt.alloc_off[r + 1]; k += 32) {
      uint32_t g = m.n_slots;
      if (!dead) {
        const uint32_t node = rt.alloc_node[k];
        if (node >= m.n_nodes) {
          atomicOr(bad, 1u);
        } else {
          const uint32_t s = running_slot(m, rv, node);
          if (s != 0xffffffffu) g = s;
        }
      }
      keys[k] = (uint64_t)r << 32 | g;
      vals[k] = k;
    }
  }
}

// off[i] = the first position whose key (bits 0-31) is >= i, for i in [0, m]; keys ascending
__global__ void k_rt_offsets(const uint64_t* keys, uint32_t n, uint32_t m, uint32_t* off) {
  const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i > m) return;
  uint32_t lo = 0, hi = n;
  while (lo < hi) {
    const uint32_t mid = lo + (hi - lo) / 2;
    if ((uint32_t)keys[mid] < i) lo = mid + 1;
    else hi = mid;
  }
  off[i] = lo;
}

// The allocations grouped by node state: end time of the owning job, allocated row
__global__ void k_rt_slot_gather(RunTableDev rt, const uint64_t* keys, const uint32_t* vals, uint32_t n,
                                 const uint32_t* n_valid_ptr, int64_t* slot_end, Row* slot_res) {
  const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n || i >= *n_valid_ptr) return;
  slot_end[i] = rt.end_time[(uint32_t)(keys[i] >> 32)];
  slot_res[i] = rt.alloc_res[vals[i]];
}

// keys = account, vals = job of the view: the stable sort groups the jobs by account
__global__ void k_rt_acc_keys(const uint32_t* account, uint32_t n, uint64_t* keys, uint32_t* vals) {
  const uint32_t c = blockIdx.x * blockDim.x + threadIdx.x;
  if (c < n) {
    keys[c] = account[c];
    vals[c] = c;
  }
}

// The accounts that appear in the live pending rows or the running jobs
__global__ void k_acc_present(const uint32_t* pd_account, const uint8_t* pd_dead, uint32_t n_pending,
                              const uint32_t* rn_account, uint32_t n_running, uint8_t* present) {
  const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n_pending) {
    if (!pd_dead || !pd_dead[i]) present[pd_account[i]] = 1;
  } else if (i < n_pending + n_running) {
    present[rn_account[i - n_pending]] = 1;
  }
}

}  // namespace crane
