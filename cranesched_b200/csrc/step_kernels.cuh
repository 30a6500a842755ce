// step_kernels.cuh — the step scheduler of running jobs (JobInCtld::SchedulePendingSteps,
// reference src/CraneCtld/CtldPublicDefs.cpp:1877-1998).
//
// Every running job owns step_res_avail_, a ResourceV3 over its own nodes, so jobs are
// independent; only the FIFO steps inside one job form a chain (a step that does not fit
// blocks itself and every later step of the job). k_steps gives every job one warp:
//   candidates  the lanes count, for 32 nodes at a time, the tasks `c` each node could take
//               (req_node once, then req_task while c < ntpn_max and it fits — NOT
//               NodeSelect's get_max_tasks, which counts from ntpn_min upwards). The counts
//               are exact in parallel: avail does not change during this phase. Lane 0 then
//               feeds them, in node-index order (deviation D8: the reference walks an
//               unordered_map), into a std::priority_queue restatement whose top is the node
//               with the fewest tasks, and stops where the reference breaks.
//   hand-out    lane 0 pops the heap: per node n = min(rest, c - 1) + 1 tasks and the first
//               task id; the lanes then place the popped nodes in parallel (one lane per
//               node): req_node, then n successive req_task allocations, each subtracted
//               from avail.
// The heap lives in shared memory, one per warp; node_num <= kStepHeapMax - 1.
#pragma once

#include "algebra.cuh"

namespace crane {

constexpr int kStepHeapMax = 128;      // = kHeapMax of commit_v2.cuh: steps of up to 127 nodes
constexpr int kStepWarps = 4;          // warps (jobs in flight) per CTA

struct StepJobsDev {
  uint32_t n_jobs;
  const uint32_t* node_off;  // [n_jobs + 1] CSR over (job, node) pairs
  const uint32_t* node;      // node index, ascending within a job
  Row* avail;                // step_res_avail_, updated in place
  const uint32_t* step_off;  // [n_jobs + 1] the job's pending steps are rows [step_off[j], step_off[j+1])
};
struct StepsDev {
  const uint32_t* node_num;
  const uint32_t* ntasks;
  const uint32_t* ntpn_min;
  const uint32_t* ntpn_max;
  const View* req_node;
  const View* req_task;
  const uint32_t* incl_off;  // NULL = no include lists
  const uint32_t* incl_nodes;
  const uint32_t* excl_off;  // NULL = no exclude lists
  const uint32_t* excl_nodes;
};
struct StepOutDev {
  uint32_t* placed;          // [n_jobs]
  uint8_t* scheduled;        // [n_steps]
  const uint32_t* node_off;  // [n_steps + 1] prefix sum of node_num
  uint32_t* alloc_node;
  uint32_t* alloc_ntasks;
  Row* alloc_res;
  const uint32_t* task_off;  // [n_steps + 1] prefix sum of ntasks
  uint32_t* task_node;
  Row* task_res;
};

// std::priority_queue<NodeInfo> of SchedulePendingSteps: NodeInfo::operator< is "has more
// tasks", so the top has the fewest. push / pop are libstdc++'s __push_heap / __adjust_heap,
// as heap_push2 / heap_pop2 in commit_v2.cuh (that copy keeps 16-bit fields in its own
// layout; this one holds 32-bit counts and job-local node positions).
struct StepHeap {
  uint32_t nt[kStepHeapMax];
  uint32_t k[kStepHeapMax];
  uint32_t size, sum;
};
__device__ __forceinline__ bool step_heap_less(uint32_t a_nt, uint32_t b_nt) { return a_nt > b_nt; }
__device__ inline void step_heap_push(StepHeap& h, uint32_t nt, uint32_t k) {
  uint32_t hole = h.size++;
  while (hole > 0) {
    const uint32_t parent = (hole - 1) / 2;
    if (!step_heap_less(h.nt[parent], nt)) break;
    h.nt[hole] = h.nt[parent]; h.k[hole] = h.k[parent];
    hole = parent;
  }
  h.nt[hole] = nt; h.k[hole] = k;
}
__device__ inline void step_heap_pop(StepHeap& h) {
  const uint32_t len = h.size - 1;
  if (len == 0) { h.size = 0; return; }
  const uint32_t vnt = h.nt[len], vk = h.k[len];
  uint32_t hole = 0, second = 0;
  while ((int32_t)second < ((int32_t)len - 1) / 2) {  // __adjust_heap
    second = 2 * (second + 1);
    if (step_heap_less(h.nt[second], h.nt[second - 1])) --second;
    h.nt[hole] = h.nt[second]; h.k[hole] = h.k[second];
    hole = second;
  }
  if ((len & 1u) == 0 && (int32_t)second == ((int32_t)len - 2) / 2) {
    second = 2 * (second + 1);
    h.nt[hole] = h.nt[second - 1]; h.k[hole] = h.k[second - 1];
    hole = second - 1;
  }
  while (hole > 0) {  // __push_heap(first, hole, 0, value)
    const uint32_t parent = (hole - 1) / 2;
    if (!step_heap_less(h.nt[parent], vnt)) break;
    h.nt[hole] = h.nt[parent]; h.k[hole] = h.k[parent];
    hole = parent;
  }
  h.nt[hole] = vnt; h.k[hole] = vk;
  h.size = len;
}

struct StepWarp {
  StepHeap heap;
  uint32_t c[32];                 // tasks of the 32 nodes of the current round, 0xFFFFFFFF = not a candidate
  uint32_t pop_k[kStepHeapMax];   // hand-out, in pop order: job-local node position,
  uint32_t pop_n[kStepHeapMax];   //   tasks on it,
  uint32_t pop_t[kStepHeapMax];   //   its first task id
  uint32_t done, ok;
};
__shared__ StepWarp s_step[kStepWarps];

__device__ __forceinline__ bool step_list_has(const uint32_t* off, const uint32_t* nodes, uint32_t s, uint32_t n) {
  for (uint32_t i = off[s]; i < off[s + 1]; ++i)
    if (nodes[i] == n) return true;
  return false;
}

// tasks node `n` with availability `a` can take for step s (CtldPublicDefs.cpp:1907-1930),
// 0xFFFFFFFF if it is not a candidate
__device__ __noinline__ uint32_t step_node_tasks(const StepsDev& st, uint32_t s, uint32_t n, const Row& a0,
                                                 const GresDict& d) {
  if (st.excl_off && step_list_has(st.excl_off, st.excl_nodes, s, n)) return 0xFFFFFFFFu;
  if (st.incl_off && st.incl_off[s + 1] > st.incl_off[s] && !step_list_has(st.incl_off, st.incl_nodes, s, n))
    return 0xFFFFFFFFu;
  Row a = a0, got;
  if (!feasible<true>(st.req_node[s], a, d, &got)) return 0xFFFFFFFFu;
  row_sub(a, got);
  const View rt = st.req_task[s];
  const uint32_t tmax = st.ntpn_max[s];
  uint32_t c = 0;
  while (c < tmax && feasible<true>(rt, a, d, &got)) {
    ++c;
    row_sub(a, got);
  }
  return c < st.ntpn_min[s] ? 0xFFFFFFFFu : c;
}

__global__ void __launch_bounds__(32 * kStepWarps) k_steps(StepJobsDev jb, StepsDev st, StepOutDev out, uint32_t dslot) {
  const GresDict& d = c_dicts[dslot];
  const uint32_t lane = threadIdx.x & 31u, w = threadIdx.x >> 5;
  StepWarp& sw = s_step[w];
  const uint32_t n_warps = gridDim.x * kStepWarps;
  for (uint32_t j = blockIdx.x * kStepWarps + w; j < jb.n_jobs; j += n_warps) {
    const uint32_t k0 = jb.node_off[j], nk = jb.node_off[j + 1] - k0;
    const uint32_t s0 = jb.step_off[j], s1 = jb.step_off[j + 1];
    const uint32_t* nodes = jb.node + k0;
    Row* avail = jb.avail + k0;
    uint32_t s = s0;
    for (; s < s1; ++s) {
      const uint32_t node_num = st.node_num[s], ntasks = st.ntasks[s];
      // ---- candidates --------------------------------------------------------------
      if (lane == 0) { sw.heap.size = 0; sw.heap.sum = 0; sw.done = 0; }
      __syncwarp();
      for (uint32_t base = 0; base < nk; base += 32) {
        const uint32_t k = base + lane;
        sw.c[lane] = k < nk ? step_node_tasks(st, s, nodes[k], avail[k], d) : 0xFFFFFFFFu;
        __syncwarp();
        if (lane == 0) {
          const uint32_t m = nk - base < 32u ? nk - base : 32u;
          for (uint32_t i = 0; i < m; ++i) {
            const uint32_t c = sw.c[i];
            if (c == 0xFFFFFFFFu) continue;
            step_heap_push(sw.heap, c, base + i);
            sw.heap.sum += c;
            if (sw.heap.size > node_num) {
              sw.heap.sum -= sw.heap.nt[0];
              step_heap_pop(sw.heap);
            }
            if (sw.heap.size == node_num && sw.heap.sum >= ntasks) { sw.done = 1; break; }
          }
        }
        __syncwarp();
        if (sw.done) break;
      }
      // ---- blocking (head of line) + hand-out order ------------------------------------
      if (lane == 0) {
        sw.ok = sw.heap.size == node_num && sw.heap.sum >= ntasks;
        if (sw.ok) {
          uint32_t rest = ntasks - node_num, tid = 0;
          for (uint32_t i = 0; i < node_num; ++i) {
            const uint32_t c = sw.heap.nt[0];
            const uint32_t n = (rest < c - 1 ? rest : c - 1) + 1;
            sw.pop_k[i] = sw.heap.k[0];
            sw.pop_n[i] = n;
            sw.pop_t[i] = tid;
            tid += n;
            rest -= n - 1;
            step_heap_pop(sw.heap);
          }
        }
      }
      __syncwarp();
      if (!sw.ok) break;
      // ---- placement: one lane per popped node -----------------------------------------
      const uint32_t noff = out.node_off[s], toff = out.task_off[s];
      for (uint32_t i = lane; i < node_num; i += 32) {
        const uint32_t k = sw.pop_k[i];
        uint32_t rank = 0;  // node rows are in node-index order = job-local position order
        for (uint32_t i2 = 0; i2 < node_num; ++i2) rank += sw.pop_k[i2] < k;
        Row a = avail[k], got, acc;
        feasible<true>(st.req_node[s], a, d, &got);
        row_sub(a, got);
        acc = got;
        const View rt = st.req_task[s];
        const uint32_t n = sw.pop_n[i], t0 = toff + sw.pop_t[i];
        for (uint32_t t = 0; t < n; ++t) {
          feasible<true>(rt, a, d, &got);
          row_sub(a, got);
          row_add(acc, got);
          out.task_node[t0 + t] = nodes[k];
          out.task_res[t0 + t] = got;
        }
        avail[k] = a;
        out.alloc_node[noff + rank] = nodes[k];
        out.alloc_ntasks[noff + rank] = n;
        out.alloc_res[noff + rank] = acc;
      }
      if (lane == 0) out.scheduled[s] = 1;
      __syncwarp();  // avail of this step is visible to every lane before the next one
    }
    if (lane == 0) out.placed[j] = s - s0;
    __syncwarp();
  }
}

}  // namespace crane
