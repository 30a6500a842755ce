// step_resident_kernels.cuh — sm_90a kernels of the device-resident step state of running
// jobs (JobInCtld::step_res_avail_ and pending_step_ids_, CtldPublicDefs.h:984-1009).
//
// Two resident tables whose rows keep their index until crane_sched_steps_compact
// (compact_kernels.cuh) or crane_sched_step_jobs_reset:
//   step jobs  one row per running job that can get steps: its nodes (ascending) and one
//              step_res_avail_ row per node, in a node pool (CSR sj_node_off);
//   steps      one row per step: its crane_steps_t columns, and once scheduled the offset
//              of its node rows in the allocation pool (the node rows stay there so that
//              EraseStep can give them back).
// A pass gathers the dense StepJobsDev / StepsDev tables of the jobs it visits from the
// resident ones, runs the unchanged k_steps on them and scatters its results back:
//   k_sp_pass_cols   per visited job its node count, per visited step its columns and
//                    the counts the prefix sums turn into offsets;
//   k_sp_scan        those prefix sums (one block, one segment after another);
//   k_sp_pass_rows   nodes, avail rows and include / exclude lists into the dense tables;
//   k_steps          (step_kernels.cuh)
//   k_sp_scatter     avail back into the pool, node rows of the scheduled steps into the
//                    allocation pool, their ntasks and task rows into the pass's results.
// k_sj_seed copies started jobs' allocations out of the resident running table, and
// k_sp_release adds the node rows of ended steps back to their jobs' avail.
#pragma once

#include "step_kernels.cuh"

namespace crane {

// ------------------------------------------------------------------------
// crane_sched_step_jobs_start: avail = the running row's allocation
// (JobInCtld::SetStepResAvail(allocated_res), JobScheduler.cpp:1277)
// ------------------------------------------------------------------------
// One warp per started row; *bad is set when a row's nodes are not ascending and distinct.
__global__ void k_sj_seed(const uint32_t* rr_alloc_off, const uint32_t* rr_alloc_node, const Row* rr_alloc_res,
                          const uint32_t* rows, uint32_t n, const uint32_t* sj_node_off, uint32_t* sj_node,
                          Row* sj_avail, uint32_t* bad) {
  const uint32_t lane = threadIdx.x & 31u;
  const uint32_t n_warps = gridDim.x * (blockDim.x >> 5);
  for (uint32_t k = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5); k < n; k += n_warps) {
    const uint32_t src = rr_alloc_off[rows[k]], cnt = rr_alloc_off[rows[k] + 1] - src, dst = sj_node_off[k];
    for (uint32_t i = lane; i < cnt; i += 32) {
      const uint32_t node = rr_alloc_node[src + i];
      if (i && rr_alloc_node[src + i - 1] >= node) *bad = 1;
      sj_node[dst + i] = node;
      sj_avail[dst + i] = rr_alloc_res[src + i];
    }
  }
}

// ------------------------------------------------------------------------
// one pass (crane_sched_steps_run)
// ------------------------------------------------------------------------
// The resident tables, tombstones included
struct StepPoolDev {
  const uint32_t* sj_node_off;  // [step jobs + 1] CSR into the node pool
  const uint32_t* sj_node;
  Row* sj_avail;
  const uint32_t* job, *node_num, *ntasks, *ntpn_min, *ntpn_max;  // [steps]
  const View* req_node;
  const View* req_task;
  const uint32_t* incl_off;     // [steps + 1] CSR into the include pool
  const uint32_t* incl_nodes;
  const uint32_t* excl_off;
  const uint32_t* excl_nodes;
  uint32_t* alloc_at;           // [steps] a scheduled step's first row in the allocation pool
  uint32_t* sa_node;            // allocation pool: node rows of scheduled steps
  Row* sa_res;
};

// The visited jobs (ascending rows) and their live pending steps (job by job, FIFO), and
// the dense tables k_steps runs on
struct StepPassDev {
  uint32_t n_jobs, n_steps;
  const uint32_t* jl;      // [n_jobs] step-job rows
  const uint32_t* sl;      // [n_steps] step rows
  uint32_t* node_off;      // [n_jobs + 1]
  uint32_t* node;
  Row* avail;
  uint32_t* step_off;      // [n_jobs + 1]
  uint32_t* node_num, *ntasks, *ntpn_min, *ntpn_max;
  View* req_node;
  View* req_task;
  uint32_t* incl_off;      // [n_steps + 1]
  uint32_t* incl_nodes;
  uint32_t* excl_off;      // [n_steps + 1]
  uint32_t* excl_nodes;
  uint32_t* out_node_off;  // [n_steps + 1]
  uint32_t* out_task_off;  // [n_steps + 1]
  uint32_t* placed;        // [n_jobs]
  uint8_t* scheduled;      // [n_steps]
  uint32_t* alloc_node, *alloc_ntasks, *task_node;
  Row* alloc_res;
  Row* task_res;
};

// Per visited job: its node count; per visited step: its columns, the counts the scan
// turns into offsets, and where its job's steps start (the steps come job by job, in the
// order of jl, so a step whose job differs from its predecessor's starts the next job).
// The [n] entries of the counted columns are 0 placeholders for the totals.
__global__ void k_sp_pass_cols(StepPoolDev p, StepPassDev d) {
  const uint32_t stride = gridDim.x * blockDim.x;
  const uint32_t m = d.n_jobs > d.n_steps ? d.n_jobs : d.n_steps;
  for (uint32_t i = blockIdx.x * blockDim.x + threadIdx.x; i <= m; i += stride) {
    if (i < d.n_jobs) {
      const uint32_t j = d.jl[i];
      d.node_off[i] = p.sj_node_off[j + 1] - p.sj_node_off[j];
      d.placed[i] = 0;
    } else if (i == d.n_jobs) {
      d.node_off[i] = 0;
      d.step_off[i] = d.n_steps;
    }
    if (i < d.n_steps) {
      const uint32_t s = d.sl[i];
      d.node_num[i] = p.node_num[s];
      d.ntasks[i] = p.ntasks[s];
      d.ntpn_min[i] = p.ntpn_min[s];
      d.ntpn_max[i] = p.ntpn_max[s];
      d.req_node[i] = p.req_node[s];
      d.req_task[i] = p.req_task[s];
      d.out_node_off[i] = p.node_num[s];
      d.out_task_off[i] = p.ntasks[s];
      d.incl_off[i] = p.incl_off[s + 1] - p.incl_off[s];
      d.excl_off[i] = p.excl_off[s + 1] - p.excl_off[s];
      d.scheduled[i] = 0;
      const uint32_t job = p.job[s];
      if (i == 0 || p.job[d.sl[i - 1]] != job) {
        uint32_t lo = 0, hi = d.n_jobs;  // lower_bound of job in jl
        while (lo < hi) {
          const uint32_t mid = lo + (hi - lo) / 2;
          if (d.jl[mid] < job) lo = mid + 1;
          else hi = mid;
        }
        d.step_off[lo] = i;
      }
    } else if (i == d.n_steps) {
      d.out_node_off[i] = d.out_task_off[i] = d.incl_off[i] = d.excl_off[i] = 0;
    }
  }
}

// Exclusive prefix sum of each segment in place, by one block (segments of n + 1 entries
// whose last is 0 end with their total)
constexpr int kScanSegs = 5;
struct ScanSegs {
  uint32_t* p[kScanSegs];
  uint32_t n[kScanSegs];
};
__global__ void __launch_bounds__(1024) k_sp_scan(ScanSegs sg) {
  __shared__ uint32_t s_part[1024];
  __shared__ uint32_t s_carry;
  for (int g = 0; g < kScanSegs; ++g) {
    uint32_t* a = sg.p[g];
    const uint32_t total = sg.n[g];
    if (threadIdx.x == 0) s_carry = 0;
    __syncthreads();
    for (uint32_t base = 0; base < total; base += blockDim.x) {
      const uint32_t i = base + threadIdx.x;
      const uint32_t v = i < total ? a[i] : 0;
      s_part[threadIdx.x] = v;
      __syncthreads();
      for (uint32_t o = 1; o < blockDim.x; o <<= 1) {
        const uint32_t add = threadIdx.x >= o ? s_part[threadIdx.x - o] : 0;
        __syncthreads();
        s_part[threadIdx.x] += add;
        __syncthreads();
      }
      const uint32_t incl = s_part[threadIdx.x], carry = s_carry;
      if (i < total) a[i] = carry + incl - v;
      __syncthreads();
      if (threadIdx.x == blockDim.x - 1) s_carry = carry + incl;
      __syncthreads();
    }
  }
}

// One warp per visited job (its nodes and avail rows) and per visited step (its lists)
__global__ void k_sp_pass_rows(StepPoolDev p, StepPassDev d) {
  const uint32_t lane = threadIdx.x & 31u;
  const uint32_t n_warps = gridDim.x * (blockDim.x >> 5);
  for (uint32_t w = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5); w < d.n_jobs + d.n_steps; w += n_warps) {
    if (w < d.n_jobs) {
      const uint32_t j = d.jl[w], src = p.sj_node_off[j], cnt = p.sj_node_off[j + 1] - src, dst = d.node_off[w];
      for (uint32_t i = lane; i < cnt; i += 32) {
        d.node[dst + i] = p.sj_node[src + i];
        d.avail[dst + i] = p.sj_avail[src + i];
      }
    } else {
      const uint32_t i = w - d.n_jobs, s = d.sl[i];
      for (uint32_t k = lane; k < d.incl_off[i + 1] - d.incl_off[i]; k += 32)
        d.incl_nodes[d.incl_off[i] + k] = p.incl_nodes[p.incl_off[s] + k];
      for (uint32_t k = lane; k < d.excl_off[i + 1] - d.excl_off[i]; k += 32)
        d.excl_nodes[d.excl_off[i] + k] = p.excl_nodes[p.excl_off[s] + k];
    }
  }
}

// One warp per visited job (avail back into the pool when it placed a step) and per
// visited step; a scheduled one has its result rows at pos[2i] (node rows) and pos[2i+1]
// (task rows): rows of the pass's scheduled steps in ascending step-row order. Its node
// rows go to the allocation pool at sa_base + pos[2i], ntasks and task rows to the results.
__global__ void k_sp_scatter(StepPoolDev p, StepPassDev d, const uint32_t* pos, uint32_t sa_base,
                             uint32_t* res_ntasks, uint32_t* res_task_node, Row* res_task_res) {
  const uint32_t lane = threadIdx.x & 31u;
  const uint32_t n_warps = gridDim.x * (blockDim.x >> 5);
  for (uint32_t w = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5); w < d.n_jobs + d.n_steps; w += n_warps) {
    if (w < d.n_jobs) {
      if (d.placed[w] == 0) continue;
      const uint32_t j = d.jl[w], dst = p.sj_node_off[j], cnt = p.sj_node_off[j + 1] - dst, src = d.node_off[w];
      for (uint32_t i = lane; i < cnt; i += 32) p.sj_avail[dst + i] = d.avail[src + i];
    } else {
      const uint32_t i = w - d.n_jobs;
      if (!d.scheduled[i]) continue;
      const uint32_t nr = pos[2 * i], tr = pos[2 * i + 1];
      const uint32_t n0 = d.out_node_off[i], nn = d.out_node_off[i + 1] - n0;
      const uint32_t t0 = d.out_task_off[i], nt = d.out_task_off[i + 1] - t0;
      for (uint32_t k = lane; k < nn; k += 32) {
        p.sa_node[sa_base + nr + k] = d.alloc_node[n0 + k];
        p.sa_res[sa_base + nr + k] = d.alloc_res[n0 + k];
        res_ntasks[nr + k] = d.alloc_ntasks[n0 + k];
      }
      for (uint32_t k = lane; k < nt; k += 32) {
        res_task_node[tr + k] = d.task_node[t0 + k];
        res_task_res[tr + k] = d.task_res[t0 + k];
      }
      if (lane == 0) p.alloc_at[d.sl[i]] = sa_base + nr;
    }
  }
}

// ------------------------------------------------------------------------
// crane_sched_steps_erase of scheduled steps: step_res_avail_ += AllocatedRes()
// (JobInCtld::EraseStep, CtldPublicDefs.h:1000-1009)
// ------------------------------------------------------------------------
// One warp per affected job (jobs[w]); its released steps are steps[off[w] .. off[w+1])
// in row order, the lanes over a step's node rows (distinct nodes), each finding its
// node's entry by binary search over the job's ascending nodes.
__global__ void k_sp_release(StepPoolDev p, const uint32_t* jobs, const uint32_t* off, const uint32_t* steps,
                             uint32_t n) {
  const uint32_t lane = threadIdx.x & 31u;
  const uint32_t n_warps = gridDim.x * (blockDim.x >> 5);
  for (uint32_t w = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5); w < n; w += n_warps) {
    const uint32_t j = jobs[w], k0 = p.sj_node_off[j], k1 = p.sj_node_off[j + 1];
    for (uint32_t q = off[w]; q < off[w + 1]; ++q) {
      const uint32_t s = steps[q], a0 = p.alloc_at[s];
      for (uint32_t i = lane; i < p.node_num[s]; i += 32) {
        const uint32_t node = p.sa_node[a0 + i];
        uint32_t lo = k0, hi = k1;
        while (lo < hi) {
          const uint32_t mid = lo + (hi - lo) / 2;
          if (p.sj_node[mid] < node) lo = mid + 1;
          else hi = mid;
        }
        if (lo < k1 && p.sj_node[lo] == node) row_add(p.sj_avail[lo], p.sa_res[a0 + i]);
      }
      __syncwarp();
    }
  }
}

// crane_sched_step_jobs_avail: the avail rows of jobs rows[k], one after another (dst_off)
__global__ void k_sj_avail_gather(const uint32_t* sj_node_off, const Row* sj_avail, const uint32_t* rows,
                                  const uint32_t* dst_off, uint32_t n, Row* dst) {
  const uint32_t lane = threadIdx.x & 31u;
  const uint32_t n_warps = gridDim.x * (blockDim.x >> 5);
  for (uint32_t k = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5); k < n; k += n_warps) {
    const uint32_t src = sj_node_off[rows[k]], cnt = sj_node_off[rows[k] + 1] - src;
    for (uint32_t i = lane; i < cnt; i += 32) dst[dst_off[k] + i] = sj_avail[src + i];
  }
}

}  // namespace crane
