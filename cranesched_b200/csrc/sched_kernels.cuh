// sched_kernels.cuh — sm_90a (H100) kernels of the CraneCtld scheduling hot path.
//
// Reference functions restated here (SURVEY.md §8a):
//   R3  NodeState::InitTimeAvailResMap           JobScheduler.h:295-332
//   R4  MinCpuTimeRatioFirst / NodeSelector cost JobScheduler.h:40-54,492-532
//   R5  BasicPriority                            JobScheduler.h:177-195
//   R6  MultiFactorPriority                      JobScheduler.cpp:6526-6739
//   R7  LocalScheduler::GetNodesAndTrySchedule_  JobScheduler.cpp:5185-5405
//   R8  ResourceView::GetFeasibleResourceInNode  PublicHeader.cpp:519-599 (algebra.cuh)
//   R9  EarliestStartSubsetSelector              JobScheduler.h:786-859
//   R10 NodeState::UpdateResourceInNode          JobScheduler.h:334-453
//   R11 SchedulerAlgo::NodeSelect job loop       JobScheduler.cpp:5777-5867
//
// Data layout in HBM (all per tick, see DESIGN.md):
//   node slot g = compact index of an alive && !drain node inside its
//   partition's contiguous range [part_base[p], part_base[p+1]).
//   tl_ent[g][CAP] = {int64 t; Row seg} (80 B), tl_n[g]; CAP = max_jobs_per_node + 1.
#pragma once

#include "algebra.cuh"

#ifndef CRANE_EMU
#define CRANE_DYN_SMEM(T, name) extern __shared__ __align__(16) unsigned char name##_raw[]; T* name = reinterpret_cast<T*>(name##_raw)
#define CRANE_LAUNCH(kernel, grid, block, smem, stream, ...) kernel<<<(grid), (block), (smem), (stream)>>>(__VA_ARGS__)
#endif

namespace crane {

constexpr int64_t kInf = INT64_MAX;
constexpr uint32_t kFullMask = 0xffffffffu;

// gres dictionaries in constant memory, one slot per live handle of this device
// (a cluster's (name,type) layout belongs to its handle, never to the module)
constexpr int kDictSlots = 16;
__constant__ GresDict c_dicts[kDictSlots];

// ------------------------------------------------------------------------
// device-side tables
// ------------------------------------------------------------------------
struct PendingDev {  // SoA mirror of crane_pending_t
  uint32_t n;
  const uint32_t* partition;
  const int64_t* time_limit;
  const int64_t* submit_time;
  const uint32_t* node_num;
  const uint32_t* ntasks_per_node_min;
  const uint32_t* ntasks_per_node_max;
  const uint32_t* ntasks;
  const uint8_t* exclusive;
  const uint32_t* partition_priority;
  const uint32_t* qos_priority;
  const uint32_t* account;
  const double* mandated_priority;
  const View* req_node;
  const View* req_task;
  const View* req_total;
  const uint32_t* incl_off;
  const uint32_t* incl_nodes;
  const uint32_t* excl_off;
  const uint32_t* excl_nodes;
  const uint32_t* alloc_off;  // exclusive prefix sum of node_num
  const uint32_t* reservation;  // or null
  const uint8_t* dead;          // erased rows of the device-resident table (or null): not in the queue; in a
                                // gated run the row's exclusion code (ERASED or a gate reason)
};

struct RunningDev {
  uint32_t n;
  const int64_t* start_time;
  const int64_t* end_time;
  const uint32_t* node_num;
  const uint32_t* partition_priority;
  const uint32_t* qos_priority;
  const uint32_t* account;
  const int64_t* view_cpu_raw;
  const uint64_t* view_mem;
  // running allocations regrouped by node slot (input order kept)
  const uint32_t* slot_off;   // [n_slots+1]
  const int64_t* slot_end;    // end_time of the owning job (unclamped)
  const Row* slot_res;
  // running jobs regrouped by account (input order kept)
  uint32_t n_accounts;
  const uint32_t* acc_off;    // [n_accounts+1]
  const uint32_t* acc_job;
  const uint8_t* acc_present; // account appears in pending or running
};

constexpr int kMaxClasses = 16;  // distinct res_total rows cached per partition

struct ClusterDev {
  uint32_t n_slots;           // node states: usable nodes of the partitions, then the nodes of every reservation
  uint32_t n_parts;           // partitions of the cluster
  uint32_t n_comp;            // schedulers of partitions: one per connected group of overlapping partitions
  uint32_t n_vparts;          // schedulers: n_comp + one per reservation (JobScheduler.cpp:5757-5766)
  const uint32_t* part_comp;  // [n_parts] scheduler of a partition
  const uint32_t* part_cidx;  // [n_parts] index of the partition inside its scheduler
  const uint8_t* slot_memb;   // [n_slots] bit i: the node is in partition i of its scheduler (null: no overlap)
  uint32_t n_resv;
  uint32_t max_part_slots;
  const uint32_t* part_base;  // [n_vparts+1] slot ranges
  // reservations (JobScheduler.cpp:5655-5713)
  const int64_t* resv_start;  // [n_resv]
  const int64_t* resv_end;
  const uint32_t* slot_resv;  // [n_slots] reservation whose node state this is, 0xffffffff = a partition's node
  const uint32_t* rsv_off;    // [n_slots+1] reservations holding resources of a partition's node, ascending id
  const uint32_t* rsv_id;
  const Row* rsv_res;
  const uint32_t* slot_node;  // slot -> global node index
  const uint32_t* node_slot;  // global node -> slot or 0xffffffff
  const Row* slot_total;      // res_total per slot
  const uint8_t* slot_class;  // per slot: index into its partition's class rows, 0xff = none
  const Row* class_rows;      // [n_parts][kMaxClasses]
};

// one timeline breakpoint: from time t on, `seg` is available on the node
// (an entry of NodeState::time_avail_res_map, JobScheduler.h:239,285)
struct __align__(16) TlEntry {
  int64_t t;
  Row seg;
};
static_assert(sizeof(TlEntry) == 80, "TlEntry layout");

struct TimelineDev {
  uint32_t cap;               // entries per slot
  uint32_t* n;                // [n_slots]
  TlEntry* ent;               // [n_slots][cap]
  Row* avail0;                // [n_slots] tick-start res_avail (NodeState::res_avail)
  double* cost0;              // [n_slots] initial cost (NodeRater)
  uint8_t* skip;              // [n_slots] timeline size >= max_jobs_per_node
  int64_t* first_resv;        // [n_slots] craned_id_first_resv_map: earliest start of a reservation on the node, kInf = none
};

// per-job record in final queue order (partition-major, priority order inside)
struct __align__(16) JobQ {
  View req;            // req_node + req_task * ntasks_per_node (min_res_view)
  int64_t time_limit;
  uint32_t job;        // index into the pending table
  uint32_t node_num;
  uint32_t alloc_off;
  uint32_t ntasks_per_node;
  uint32_t flags;      // kJq* below
  uint32_t ntpn_max;   // ntasks_per_node_max
  uint64_t spec8;      // per-entry typed counts, one byte each (clamped to 127)
  uint8_t name_need[CRANE_GRES_NAMES];  // per name max(total, sum typed), clamped to 255
  uint32_t ntasks;     // total task count of the job
  uint32_t vpart;      // scheduler of the job: partition, or n_parts + reservation
};
static_assert(sizeof(JobQ) == 112, "JobQ layout");
// JobQ::flags
constexpr uint32_t kJqExclusive = 1u << 0;  // exclusive node allocation
constexpr uint32_t kJqHasGres = 1u << 1;    // the request names gres
constexpr uint32_t kJqGeneral = 1u << 2;    // general task distribution (a ntasks_per_node range or an uneven ntasks)
constexpr uint32_t kJqNamesShift = 8;       // bits 8-15: gres names requested (bit per name)
constexpr uint32_t kJqPartShift = 16;       // bits 16-18: partition inside a scheduler of overlapping partitions
__device__ __forceinline__ bool jq_exclusive(const JobQ& q) { return (q.flags & kJqExclusive) != 0; }
__device__ __forceinline__ bool jq_has_gres(const JobQ& q) { return (q.flags & kJqHasGres) != 0; }
__device__ __forceinline__ bool jq_general(const JobQ& q) { return (q.flags & kJqGeneral) != 0; }
__device__ __forceinline__ uint32_t jq_gnames(const JobQ& q) { return (q.flags >> kJqNamesShift) & 0xffu; }
__device__ __forceinline__ uint32_t jq_part(const JobQ& q) { return (q.flags >> kJqPartShift) & 7u; }

struct PlaceDev {
  uint8_t* reason;
  double* priority;
  int64_t* start_time;
  int64_t* end_time;
  uint32_t* n_alloc;
  uint32_t* alloc_node;
  uint32_t* alloc_ntasks;
  Row* alloc_res;
};

struct Bounds {  // MultiFactorPriority::FactorBound, JobScheduler.h:206-216
  unsigned long long age_max, age_min;
  unsigned long long qos_max, qos_min;
  unsigned long long part_max, part_min;
  unsigned long long nodes_max, nodes_min;
  unsigned long long mem_max, mem_min;
  unsigned long long cpus_max, cpus_min;  // raw cpu_t (monotone in the double)
  unsigned long long svc_max_bits, svc_min_bits;  // non-negative doubles as bits
};

// ------------------------------------------------------------------------
// warp helpers
// ------------------------------------------------------------------------
__device__ __forceinline__ int lane_id() { return threadIdx.x & 31; }
__device__ __forceinline__ int warp_id() { return threadIdx.x >> 5; }

__device__ __forceinline__ uint64_t shfl_u64(uint64_t v, int src) {
  return (uint64_t)__shfl_sync(kFullMask, (unsigned long long)v, src);
}
__device__ __forceinline__ int64_t shfl_i64(int64_t v, int src) {
  return (int64_t)__shfl_sync(kFullMask, (long long)v, src);
}
// packed per-entry slot counts of a row (8 x u8) for the cheap pre-filter
__device__ __forceinline__ uint64_t pack_gres_counts(const Row& r) {
  uint64_t p = 0;
#pragma unroll
  for (uint32_t e = 0; e < CRANE_GRES_ENTRIES; ++e) p |= (uint64_t)popc32(field16(r.g, e)) << (8 * e);
  return p;
}
// count-only gres verdict against packed per-entry slot counts (all < 128):
// every typed count fits its entry (byte-wise >= without borrows) and each
// requested name has max(total, sum typed) slots over its entries (byte sum by
// multiply). Same verdict as feasible_gres<false> on a row with these counts.
__device__ __forceinline__ bool gres_counts_ok(uint64_t packed, uint64_t spec8, uint32_t names, const uint8_t* name_need, const GresDict& dict) {
  const uint64_t H = 0x8080808080808080ull;
  if ((((packed | H) - spec8) & H) != H) return false;
  while (names) {
    const uint32_t g = (uint32_t)__ffs((int)names) - 1u;
    names &= names - 1u;
    const uint32_t have = (uint32_t)(((packed & dict.name_mask8[g]) * 0x0101010101010101ull) >> 56);
    if (have < name_need[g]) return false;
  }
  return true;
}

// ------------------------------------------------------------------------
// K-prio part 1: factor bounds (JobScheduler.cpp:6553-6633)
// ------------------------------------------------------------------------
__global__ void k_bounds_init(Bounds* b) {
  if (threadIdx.x == 0 && blockIdx.x == 0) {
    b->age_max = 0; b->age_min = ~0ull;
    b->qos_max = 0; b->qos_min = 0xffffffffull;
    b->part_max = 0; b->part_min = 0xffffffffull;
    b->nodes_max = 0; b->nodes_min = 0xffffffffull;
    b->mem_max = 0; b->mem_min = ~0ull;
    b->cpus_max = 0; b->cpus_min = ~0ull;  // "double max" sentinel handled at use
    b->svc_max_bits = 0;                               // 0.0
    b->svc_min_bits = 0x41EFFFFFFFE00000ull;           // 4294967295.0
  }
}

__device__ __forceinline__ void warp_minmax_commit(unsigned long long mn, unsigned long long mx,
                                                   unsigned long long* gmin, unsigned long long* gmax) {
  for (int o = 16; o > 0; o >>= 1) {
    unsigned long long a = __shfl_xor_sync(kFullMask, mn, o);
    unsigned long long c = __shfl_xor_sync(kFullMask, mx, o);
    mn = a < mn ? a : mn;
    mx = c > mx ? c : mx;
  }
  if (lane_id() == 0) {
    atomicMin(gmin, mn);
    atomicMax(gmax, mx);
  }
}

__global__ void k_bounds(PendingDev pd, RunningDev rn, int64_t now, uint64_t max_age, Bounds* b) {
  const uint32_t total = pd.n + rn.n;
  unsigned long long age_mn = ~0ull, age_mx = 0, qos_mn = ~0ull, qos_mx = 0, part_mn = ~0ull, part_mx = 0,
                     nod_mn = ~0ull, nod_mx = 0, mem_mn = ~0ull, mem_mx = 0, cpu_mn = ~0ull, cpu_mx = 0;
  for (uint32_t i = blockIdx.x * blockDim.x + threadIdx.x; i < total; i += gridDim.x * blockDim.x) {
    unsigned long long qos, part, nodes, mem, cpu;
    if (i < pd.n && pd.dead && pd.dead[i]) continue;
    if (i < pd.n) {
      unsigned long long age = (unsigned long long)(now - pd.submit_time[i]);
      if (age > max_age) age = max_age;
      age_mn = age < age_mn ? age : age_mn;
      age_mx = age > age_mx ? age : age_mx;
      qos = pd.qos_priority[i];
      part = pd.partition_priority[i];
      nodes = pd.node_num[i];
      mem = pd.req_total[i].mem;
      cpu = (unsigned long long)pd.req_total[i].cpu_raw;
    } else {
      uint32_t k = i - pd.n;
      qos = rn.qos_priority[k];
      part = rn.partition_priority[k];
      nodes = rn.node_num[k];
      mem = rn.view_mem[k];
      cpu = (unsigned long long)rn.view_cpu_raw[k];
    }
    qos_mn = qos < qos_mn ? qos : qos_mn; qos_mx = qos > qos_mx ? qos : qos_mx;
    part_mn = part < part_mn ? part : part_mn; part_mx = part > part_mx ? part : part_mx;
    nod_mn = nodes < nod_mn ? nodes : nod_mn; nod_mx = nodes > nod_mx ? nodes : nod_mx;
    mem_mn = mem < mem_mn ? mem : mem_mn; mem_mx = mem > mem_mx ? mem : mem_mx;
    cpu_mn = cpu < cpu_mn ? cpu : cpu_mn; cpu_mx = cpu > cpu_mx ? cpu : cpu_mx;
  }
  warp_minmax_commit(age_mn, age_mx, &b->age_min, &b->age_max);
  warp_minmax_commit(qos_mn, qos_mx, &b->qos_min, &b->qos_max);
  warp_minmax_commit(part_mn, part_mx, &b->part_min, &b->part_max);
  warp_minmax_commit(nod_mn, nod_mx, &b->nodes_min, &b->nodes_max);
  warp_minmax_commit(mem_mn, mem_mx, &b->mem_min, &b->mem_max);
  warp_minmax_commit(cpu_mn, cpu_mx, &b->cpus_min, &b->cpus_max);
}

__device__ __forceinline__ double cpu_raw_to_double(unsigned long long raw) {
  return __ddiv_rn(__ll2double_rn((long long)raw), 256.0);
}
// cpus_alloc_min starts at numeric_limits<double>::max(), cpus_alloc_max at 0
// (JobScheduler.cpp:6575-6576); with no job at all the raw sentinel is kept.
__device__ __forceinline__ double cpus_min_double(const Bounds& b) {
  return b.cpus_min == ~0ull ? 1.7976931348623157e308 : cpu_raw_to_double(b.cpus_min);
}

// per-account service value (JobScheduler.cpp:6635-6671); one thread per
// account walks that account's running jobs in input order (deviation D6).
__global__ void k_service(RunningDev rn, int64_t now, Bounds* b, double* acc_service) {
  uint32_t a = blockIdx.x * blockDim.x + threadIdx.x;
  bool present = a < rn.n_accounts && rn.acc_present[a];
  double sum = 0.0;
  if (present) {
    const double cmin = cpus_min_double(*b), cmax = cpu_raw_to_double(b->cpus_max);
    for (uint32_t k = rn.acc_off[a]; k < rn.acc_off[a + 1]; ++k) {
      uint32_t j = rn.acc_job[k];
      double sv = 0.0;
      if (cmax > cmin)
        sv = __dadd_rn(sv, __ddiv_rn(__dmul_rn(1.0, __dsub_rn(cpu_raw_to_double((unsigned long long)rn.view_cpu_raw[j]), cmin)),
                                     __dsub_rn(cmax, cmin)));
      else
        sv = __dadd_rn(sv, 1.0);
      if (b->nodes_max > b->nodes_min)
        sv = __dadd_rn(sv, __ddiv_rn(__dmul_rn(1.0, __uint2double_rn(rn.node_num[j] - (uint32_t)b->nodes_min)),
                                     __uint2double_rn((uint32_t)b->nodes_max - (uint32_t)b->nodes_min)));
      else
        sv = __dadd_rn(sv, 1.0);
      if (b->mem_max > b->mem_min)
        sv = __dadd_rn(sv, __ddiv_rn(__dmul_rn(1.0, __ull2double_rn(rn.view_mem[j] - b->mem_min)),
                                     __ull2double_rn(b->mem_max - b->mem_min)));
      else
        sv = __dadd_rn(sv, 1.0);
      unsigned long long run_time = (unsigned long long)(now - rn.start_time[j]);
      sum = __dadd_rn(sum, __dmul_rn(sv, __ull2double_rn(run_time)));
    }
    acc_service[a] = sum;
    unsigned long long bits = (unsigned long long)__double_as_longlong(sum);  // sum >= 0
    atomicMin(&b->svc_min_bits, bits);
    atomicMax(&b->svc_max_bits, bits);
  }
}

// ------------------------------------------------------------------------
// K-prio part 2: priority value and sort key (JobScheduler.cpp:6674-6739)
// ------------------------------------------------------------------------
struct PrioCfg {
  uint32_t type, favor_small, w_age, w_fs, w_size, w_part, w_qos;
  uint64_t max_age;
};

__global__ void k_priority(PendingDev pd, PrioCfg cfg, int64_t now, const Bounds* bp,
                           const double* acc_service, double* prio_out, uint64_t* key_out,
                           uint32_t* idx_out) {
  uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= pd.n) return;
  double p = pd.mandated_priority ? pd.mandated_priority[i] : 0.0;
  if (cfg.type != 0 && p == 0.0) {
    const Bounds b = *bp;
    unsigned long long age = (unsigned long long)(now - pd.submit_time[i]);
    if (age > cfg.max_age) age = cfg.max_age;
    double f_age = 0, f_qos = 0, f_part = 0, f_size = 0, f_fs = 0;
    if (b.age_max > b.age_min)
      f_age = __ddiv_rn(__dmul_rn(1.0, __ull2double_rn(age - b.age_min)), __ull2double_rn(b.age_max - b.age_min));
    if (b.qos_max > b.qos_min)
      f_qos = __ddiv_rn(__dmul_rn(1.0, __uint2double_rn(pd.qos_priority[i] - (uint32_t)b.qos_min)),
                        __uint2double_rn((uint32_t)b.qos_max - (uint32_t)b.qos_min));
    if (b.part_max > b.part_min)
      f_part = __ddiv_rn(__dmul_rn(1.0, __uint2double_rn(pd.partition_priority[i] - (uint32_t)b.part_min)),
                         __uint2double_rn((uint32_t)b.part_max - (uint32_t)b.part_min));
    const double cmin = cpus_min_double(b), cmax = cpu_raw_to_double(b.cpus_max);
    if (cmax > cmin)
      f_size = __dadd_rn(f_size, __ddiv_rn(__dmul_rn(1.0, __dsub_rn(cpu_raw_to_double((unsigned long long)pd.req_total[i].cpu_raw), cmin)),
                                           __dsub_rn(cmax, cmin)));
    if (b.nodes_max > b.nodes_min)
      f_size = __dadd_rn(f_size, __ddiv_rn(__dmul_rn(1.0, __uint2double_rn(pd.node_num[i] - (uint32_t)b.nodes_min)),
                                           __uint2double_rn((uint32_t)b.nodes_max - (uint32_t)b.nodes_min)));
    if (b.mem_max > b.mem_min)
      f_size = __dadd_rn(f_size, __ddiv_rn(__dmul_rn(1.0, __ull2double_rn(pd.req_total[i].mem - b.mem_min)),
                                           __ull2double_rn(b.mem_max - b.mem_min)));
    if (cfg.favor_small)
      f_size = __dsub_rn(1.0, __ddiv_rn(f_size, 3.0));
    else
      f_size = __ddiv_rn(f_size, 3.0);
    double smin = __longlong_as_double((long long)b.svc_min_bits);
    double smax = __longlong_as_double((long long)b.svc_max_bits);
    if (smax > smin)
      f_fs = __dsub_rn(1.0, __ddiv_rn(__dsub_rn(acc_service[pd.account[i]], smin), __dsub_rn(smax, smin)));
    p = __dmul_rn(__uint2double_rn(cfg.w_age), f_age);
    p = __dadd_rn(p, __dmul_rn(__uint2double_rn(cfg.w_part), f_part));
    p = __dadd_rn(p, __dmul_rn(__uint2double_rn(cfg.w_size), f_size));
    p = __dadd_rn(p, __dmul_rn(__uint2double_rn(cfg.w_fs), f_fs));
    p = __dadd_rn(p, __dmul_rn(__uint2double_rn(cfg.w_qos), f_qos));
  }
  prio_out[i] = p;
  // ascending radix order of the key == descending priority; ties keep input
  // order because the LSD sort is stable (deviation D2). BasicPriority: key 0.
  uint64_t bits = (uint64_t)__double_as_longlong(p);
  uint64_t orderable = (bits >> 63) ? ~bits : (bits | 0x8000000000000000ull);
  key_out[i] = (pd.dead && pd.dead[i]) ? (cfg.type == 0 ? 1ull : ~0ull) : (cfg.type == 0 ? 0ull : ~orderable);  // erased rows sort last
  idx_out[i] = i;
}

// ------------------------------------------------------------------------
// stable LSD radix sort, 8-bit digits, (u64 key, u32 value)
// one warp per block walks its tile row by row, so equal digits keep order.
// ------------------------------------------------------------------------
constexpr int kSortTile = 2048;

__device__ __forceinline__ unsigned match_any_u32(unsigned v) {
#ifdef CRANE_EMU
  unsigned m = 0;
  for (int l = 0; l < 32; ++l) {
    unsigned o = __shfl_sync(kFullMask, v, l);
    if (o == v) m |= 1u << l;
  }
  return m;
#else
  return __match_any_sync(kFullMask, v);
#endif
}

__global__ void k_sort_hist(const uint64_t* keys, uint32_t n, int shift, uint32_t* hist, uint32_t nblocks) {
  __shared__ uint32_t s_cnt[256];
  for (int i = threadIdx.x; i < 256; i += blockDim.x) s_cnt[i] = 0;
  __syncthreads();
  uint32_t base = blockIdx.x * kSortTile;
  for (uint32_t off = threadIdx.x; off < (uint32_t)kSortTile; off += blockDim.x) {
    uint32_t i = base + off;
    if (i < n) atomicAdd(&s_cnt[(keys[i] >> shift) & 0xff], 1u);
  }
  __syncthreads();
  for (int d = threadIdx.x; d < 256; d += blockDim.x) hist[(size_t)d * nblocks + blockIdx.x] = s_cnt[d];
}

// exclusive scan of hist[256*nblocks] (digit-major) by one block
__global__ void k_sort_scan(uint32_t* hist, uint32_t total) {
  __shared__ uint32_t s_part[1024];
  __shared__ uint32_t s_carry;
  if (threadIdx.x == 0) s_carry = 0;
  __syncthreads();
  for (uint32_t base = 0; base < total; base += blockDim.x) {
    uint32_t i = base + threadIdx.x;
    uint32_t v = i < total ? hist[i] : 0;
    // block inclusive scan (Hillis-Steele in shared memory)
    s_part[threadIdx.x] = v;
    __syncthreads();
    for (uint32_t o = 1; o < blockDim.x; o <<= 1) {
      uint32_t add = threadIdx.x >= o ? s_part[threadIdx.x - o] : 0;
      __syncthreads();
      s_part[threadIdx.x] += add;
      __syncthreads();
    }
    uint32_t incl = s_part[threadIdx.x];
    uint32_t carry = s_carry;
    if (i < total) hist[i] = carry + incl - v;
    __syncthreads();
    if (threadIdx.x == blockDim.x - 1) s_carry = carry + incl;
    __syncthreads();
  }
}

__global__ void k_sort_scatter(const uint64_t* keys_in, const uint32_t* vals_in, uint64_t* keys_out,
                               uint32_t* vals_out, uint32_t n, int shift, const uint32_t* hist,
                               uint32_t nblocks) {
  // blockDim.x == 32
  __shared__ uint32_t s_off[256];
  for (int d = threadIdx.x; d < 256; d += 32) s_off[d] = hist[(size_t)d * nblocks + blockIdx.x];
  __syncwarp();
  uint32_t base = blockIdx.x * kSortTile;
  const int lane = threadIdx.x;
  for (int row = 0; row < kSortTile / 32; ++row) {
    uint32_t i = base + row * 32 + lane;
    bool valid = i < n;
    uint64_t k = valid ? keys_in[i] : 0;
    unsigned d = valid ? (unsigned)((k >> shift) & 0xff) : 0x100u;  // invalid lanes share a fake digit
    unsigned peers = match_any_u32(d);
    int rank = __popc(peers & ((1u << lane) - 1u));
    uint32_t dst = 0;
    if (valid) dst = s_off[d] + rank;
    __syncwarp();
    if (valid && rank == 0) s_off[d] += __popc(peers);
    __syncwarp();
    if (valid) {
      keys_out[dst] = k;
      vals_out[dst] = vals_in[i];
    }
  }
}

// ------------------------------------------------------------------------
// queue build: after the priority sort, order[r] is the job at rank r.
// Ranks >= limit get "Priority" (JobScheduler.cpp:6545-6550 / JS.h:191-193);
// unknown partitions get "Partition Not Found" (JobScheduler.cpp:5783-5786).
// The remaining ranks are stably re-sorted by partition id (key2).
// ------------------------------------------------------------------------
__global__ void k_queue_keys(PendingDev pd, const uint32_t* order, const double* prio, uint32_t limit,
                             ClusterDev cl, int64_t now, uint64_t* key2, PlaceDev out, uint32_t* part_count, uint32_t* vpart) {
  uint32_t r = blockIdx.x * blockDim.x + threadIdx.x;
  if (r >= pd.n) return;
  uint32_t j = order[r];
  out.priority[j] = prio[j];
  out.start_time[j] = 0;
  out.end_time[j] = 0;
  out.n_alloc[j] = 0;
  // the scheduler of the job: its reservation's (if it has started and not ended,
  // JobScheduler.cpp:5665, 5676, 5788-5795) or its partition's
  uint32_t p = pd.partition[j];
  const uint32_t rv = pd.reservation ? pd.reservation[j] : 0xffffffffu;
  uint8_t reason = CRANE_REASON_NONE;
  bool found = p < cl.n_parts;
  uint8_t miss = CRANE_REASON_PART_NOT_FOUND;
  if (rv != 0xffffffffu) {
    miss = CRANE_REASON_RESV_NOT_FOUND;
    found = rv < cl.n_resv && now >= cl.resv_start[rv] && now < cl.resv_end[rv];
    p = cl.n_comp + rv;
  } else if (found) {
    p = cl.part_comp[p];
  }
  uint64_t k = 0;
  if (pd.dead && pd.dead[j]) {  // a tombstone (1) or the gate's code of the row (gate_kernels.cuh)
    reason = pd.dead[j] == 1 ? (uint8_t)CRANE_REASON_ERASED : pd.dead[j];
    found = false;
    k = (uint64_t)cl.n_vparts + 1;
  } else if (r >= limit) {
    reason = CRANE_REASON_PRIORITY;
    k = (uint64_t)cl.n_vparts + 1;
  } else if (!found) {
    reason = miss;
    k = (uint64_t)cl.n_vparts;
  } else {
    k = p;
    atomicAdd(&part_count[p], 1u);
  }
  vpart[j] = found ? p : 0xffffffffu;
  out.reason[j] = reason;
  key2[r] = k;
}

__global__ void k_part_offsets(const uint32_t* part_count, uint32_t n_parts, uint32_t* part_job_off) {
  if (threadIdx.x == 0 && blockIdx.x == 0) {
    uint32_t acc = 0;
    for (uint32_t p = 0; p < n_parts; ++p) {
      part_job_off[p] = acc;
      acc += part_count[p];
    }
    part_job_off[n_parts] = acc;
  }
}

// JobQ records in final queue order (coalesced 96-byte records for the commit
// kernel); min_res_view of JobScheduler.cpp:5190-5192.
__global__ void k_build_jobq(PendingDev pd, const uint32_t* queue, const uint32_t* n_queued_ptr, JobQ* jobq, uint32_t dslot, const uint32_t* vpart,
                             uint32_t cl_n_comp, const uint32_t* part_cidx) {
  const GresDict& c_dict = c_dicts[dslot];
  uint32_t r = blockIdx.x * blockDim.x + threadIdx.x;
  if (r >= *n_queued_ptr) return;
  uint32_t j = queue[r];
  JobQ q;
  uint32_t t = pd.ntasks_per_node_min[j];
  view_node_plus_tasks(q.req, pd.req_node[j], pd.req_task[j], t);
  q.time_limit = pd.time_limit[j];
  q.job = j;
  q.node_num = pd.node_num[j];
  q.alloc_off = pd.alloc_off[j];
  q.ntasks_per_node = t;
  q.flags = (pd.exclusive[j] ? kJqExclusive : 0u) | (view_has_gres(q.req) ? kJqHasGres : 0u);
  q.ntpn_max = pd.ntasks_per_node_max[j];
  q.ntasks = pd.ntasks[j];
  q.vpart = vpart[j];
  // partition inside a scheduler of overlapping partitions
  if (q.vpart < cl_n_comp && part_cidx) q.flags |= (part_cidx[pd.partition[j]] & 7u) << kJqPartShift;
  // anything but "exactly ntasks_per_node tasks on each of node_num nodes" takes the general
  // task distribution (JobScheduler.cpp:5193-5222, 5340-5361)
  if (q.ntpn_max != t || (uint64_t)t * q.node_num != q.ntasks) q.flags |= kJqGeneral;
  q.spec8 = 0;
  for (uint32_t g = 0; g < CRANE_GRES_NAMES; ++g) {
    uint32_t typed = 0;
    for (uint32_t e = c_dict.name_first[g]; e < (uint32_t)c_dict.name_first[g] + c_dict.name_count[g]; ++e) {
      const uint32_t sp = field16(q.req.gspec, e);
      typed += sp;
      q.spec8 |= (uint64_t)(sp > 127 ? 127 : sp) << (8 * e);
    }
    const uint32_t tot = field16(q.req.gtot, g);
    const uint32_t need = tot > typed ? tot : typed;
    q.name_need[g] = (uint8_t)(need > 255 ? 255 : need);
    if (need) q.flags |= 1u << (kJqNamesShift + g);
  }
  jobq[r] = q;
}

// ------------------------------------------------------------------------
// K-init: per node slot, NodeState + timeline + initial cost
// (JobScheduler.cpp:5715-5753, JobScheduler.h:295-332, 492-505)
// ------------------------------------------------------------------------
__global__ void k_node_init(ClusterDev cl, RunningDev rn, TimelineDev tl, int64_t now, uint32_t max_jobs, uint32_t cost_policy) {
  uint32_t g = blockIdx.x * blockDim.x + threadIdx.x;
  if (g >= cl.n_slots) return;
  const Row total = cl.slot_total[g];
  Row avail = total;
  // a reservation's own node state lives from the reservation's start to its end;
  // before and after, nothing is scheduled into it (JobScheduler.cpp:5665, 5676, 5790-5795)
  const uint32_t myresv = cl.slot_resv ? cl.slot_resv[g] : 0xffffffffu;
  int64_t horizon = kInf;
  bool dead = false;
  if (myresv != 0xffffffffu) {
    horizon = cl.resv_end[myresv];
    dead = now >= horizon || now < cl.resv_start[myresv];
  }
  // NodeRater (JobScheduler.h:492-505): later reservations, then allocated_res — the
  // reservations that have started (JobScheduler.cpp:5676-5683) and the running jobs
  double cost = cost_policy == 1 ? __ll2double_rn(total.cpu_raw) : 0.0;  // (BestFit: seeded with the cpu count)
  const uint32_t r_lo = cl.rsv_off ? cl.rsv_off[g] : 0, r_hi = cl.rsv_off ? cl.rsv_off[g + 1] : 0;
  int64_t first = kInf;
  for (uint32_t k = r_lo; k < r_hi; ++k) {
    const uint32_t r = cl.rsv_id[k];
    const int64_t rs = cl.resv_start[r], re = cl.resv_end[r];
    if (now >= re) continue;  // expired but not cleaned up (:5665)
    first = rs < first ? rs : first;
    if (now < rs) cost = __dadd_rn(cost, cost_step(cost_policy, re - rs, cl.rsv_res[k].cpu_raw, total.cpu_raw));
  }
  for (uint32_t k = r_lo; k < r_hi; ++k) {
    const uint32_t r = cl.rsv_id[k];
    const int64_t rs = cl.resv_start[r], re = cl.resv_end[r];
    if (now >= re || now < rs) continue;
    row_sub(avail, cl.rsv_res[k]);
    cost = __dadd_rn(cost, cost_step(cost_policy, re - now, cl.rsv_res[k].cpu_raw, total.cpu_raw));
  }
  uint32_t lo = rn.n ? rn.slot_off[g] : 0, hi = rn.n ? rn.slot_off[g + 1] : 0;
  for (uint32_t k = lo; k < hi; ++k) {  // allocated_res in input order
    int64_t end = rn.slot_end[k];
    if (end < now + 1) end = now + 1;   // JobScheduler.cpp:5547-5548
    const Row res = rn.slot_res[k];
    row_sub(avail, res);
    cost = __dadd_rn(cost, cost_step(cost_policy, end - now, res.cpu_raw, total.cpu_raw));
  }
  tl.avail0[g] = avail;
  tl.cost0[g] = cost;
  tl.first_resv[g] = first;
  // InitTimeAvailResMap (JobScheduler.h:295-332): every change time is a breakpoint;
  // a segment starts from the one before it, then takes the releases of its time,
  // then the reservations that start at its time (release before allocate).
  TlEntry* E = tl.ent + (size_t)g * tl.cap;
  uint32_t n = 1;
  E[0].t = now;
  bool overflow = false;
  auto add_time = [&](int64_t t) {  // sorted, distinct
    if (overflow || t <= now) return;  // (a change at `now` itself belongs to the first segment)
    uint32_t idx = 1;
    while (idx < n && E[idx].t < t) ++idx;
    if (idx < n && E[idx].t == t) return;
    if (n + 2 > tl.cap) { overflow = true; return; }  // + sentinel would not fit
    for (uint32_t m = n; m > idx; --m) E[m].t = E[m - 1].t;
    E[idx].t = t;
    ++n;
  };
  for (uint32_t k = r_lo; k < r_hi; ++k) {
    const uint32_t r = cl.rsv_id[k];
    if (now >= cl.resv_end[r]) continue;
    if (now < cl.resv_start[r]) add_time(cl.resv_start[r]);
    add_time(cl.resv_end[r]);
  }
  for (uint32_t k = lo; k < hi; ++k) {
    int64_t end = rn.slot_end[k];
    add_time(end < now + 1 ? now + 1 : end);
  }
  E[0].seg = avail;
  for (uint32_t i = 1; i < n; ++i) {
    const int64_t t = E[i].t;
    Row seg = E[i - 1].seg;
    for (uint32_t k = r_lo; k < r_hi; ++k)
      if (now < cl.resv_end[cl.rsv_id[k]] && cl.resv_end[cl.rsv_id[k]] == t) row_add(seg, cl.rsv_res[k]);
    for (uint32_t k = lo; k < hi; ++k) {
      int64_t end = rn.slot_end[k];
      if (end < now + 1) end = now + 1;
      if (end == t) row_add(seg, rn.slot_res[k]);
    }
    for (uint32_t k = r_lo; k < r_hi; ++k)
      if (now < cl.resv_start[cl.rsv_id[k]] && cl.resv_start[cl.rsv_id[k]] == t) row_sub(seg, cl.rsv_res[k]);
    E[i].seg = seg;
  }
  // the zero sentinel: time_avail_res_map[end].SetToZero() (JobScheduler.h:331). For a
  // reservation's node state `end` is the reservation's end: entries at or after it go
  uint32_t keep = n;
  if (horizon != kInf) {
    keep = 1;
    while (keep < n && E[keep].t < horizon) ++keep;
  }
  E[keep].t = horizon;
  row_zero(E[keep].seg);
  n = keep + 1;
  tl.n[g] = n;
  tl.skip[g] = (overflow || dead || n >= max_jobs) ? 1 : 0;  // JobScheduler.cpp:5230
}

// ------------------------------------------------------------------------
// K-feas: jobs x nodes capability bitmap.
// bit(r, q) = node q of job r's partition passes the node-list filters
// (JobScheduler.cpp:5238-5256) and get_max_tasks(res_total) > 0 (:5258).
// One warp per queue rank; lane l evaluates node 32*w + l; __ballot_sync
// packs the word. Rows are `words_per_row` (a multiple of 4) words apart so
// the commit kernel can fetch a row with one 16-byte-aligned bulk copy.
// ------------------------------------------------------------------------
__global__ void k_feas_bitmap(ClusterDev cl, PendingDev pd, const JobQ* jobq, const uint32_t* n_queued_ptr,
                              uint32_t words_per_row, uint32_t* bitmap, const uint32_t* part_owner, uint32_t rank, uint32_t dslot) {
  const GresDict& c_dict = c_dicts[dslot];
  const int lane = lane_id();
  const uint32_t n_queued = *n_queued_ptr;
  uint32_t warps_per_block = blockDim.x >> 5;
  for (uint32_t r = blockIdx.x * warps_per_block + warp_id(); r < n_queued; r += gridDim.x * warps_per_block) {
    JobQ jq = jobq[r];
    uint32_t p = jq.vpart;
    if (part_owner && part_owner[p] != rank) continue;  // another GPU commits this scheduler
    const uint32_t cidx = jq_part(jq);
    uint32_t base = cl.part_base[p], mp = cl.part_base[p + 1] - base;
    const uint32_t row_words = (mp + 31) / 32;          // words beyond the job's own partition are never read
    uint32_t il = 0, ih = 0, el = 0, eh = 0;
    if (pd.incl_off) { il = pd.incl_off[jq.job]; ih = pd.incl_off[jq.job + 1]; }
    if (pd.excl_off) { el = pd.excl_off[jq.job]; eh = pd.excl_off[jq.job + 1]; }
    for (uint32_t w = 0; w < row_words; ++w) {
      uint32_t q = w * 32 + lane;
      bool ok = false;
      if (q < mp) {
        uint32_t node = cl.slot_node[base + q];
        ok = !cl.slot_memb || ((cl.slot_memb[base + q] >> cidx) & 1u);  // overlapping partitions: a member of the job's own
        if (ok && ih > il) {  // included_nodes non-empty: node must be listed
          ok = false;
          for (uint32_t k = il; k < ih; ++k) ok |= pd.incl_nodes[k] == node;
        }
        for (uint32_t k = el; k < eh && ok; ++k) ok = pd.excl_nodes[k] != node;
        if (ok) ok = feasible<false>(jq.req, cl.slot_total[base + q], c_dict, nullptr);
      }
      unsigned word = __ballot_sync(kFullMask, ok);
      if (lane == 0) bitmap[(size_t)r * words_per_row + w] = word;
    }
  }
}

__global__ void k_mark_dead(const uint32_t* rows, uint32_t n, uint8_t* dead) {
  const uint32_t k = blockIdx.x * blockDim.x + threadIdx.x;
  if (k < n) dead[rows[k]] = 1;
}

// One queue over several GPUs: the placement columns of jobs another rank owns
// go to zero, so the union over ranks is a sum (crane_sched_set_shard).
__global__ void k_shard_mask(PendingDev pd, PlaceDev out, const uint32_t* part_owner, uint32_t n_parts, uint32_t rank) {
  const uint32_t j = blockIdx.x * blockDim.x + threadIdx.x;
  if (j >= pd.n) return;
  const uint32_t p = pd.partition[j];
  const bool resv = pd.reservation && pd.reservation[j] != 0xffffffffu;  // reservations are committed by rank 0
  const uint32_t owner = (!resv && p < n_parts) ? part_owner[p] : 0u;
  if (owner != rank) {
    out.reason[j] = 0;
    out.start_time[j] = 0;
    out.end_time[j] = 0;
    out.n_alloc[j] = 0;
  }
}

// ------------------------------------------------------------------------
// Helpers of K-commit (commit_v2.cuh): phase profiling, TMA bulk copies, named
// barriers, the out-of-line allocation, order keys.
// ------------------------------------------------------------------------
// optional phase profiling (-DCRANE_PROFILE builds only; never in the product .so)
#ifdef CRANE_PROFILE
#define PROF_DECL long long prof_last = clock64(); unsigned long long prof_acc[16] = {0}
#define PROF(i) do { if (threadIdx.x == 0) { long long t__ = clock64(); prof_acc[i] += (unsigned long long)(t__ - prof_last); prof_last = t__; } } while (0)
#define PROF_CNT(i, v) do { if (threadIdx.x == 0) prof_acc[i] += (v); } while (0)
#define PROF_FLUSH(dst) do { if (threadIdx.x == 0 && (dst)) for (int i__ = 0; i__ < 16; ++i__) (dst)[blockIdx.x * 16 + i__] = prof_acc[i__]; } while (0)
#else
#define PROF_DECL
#define PROF(i)
#define PROF_CNT(i, v)
#define PROF_FLUSH(dst)
#endif

// ---- TMA 1-D bulk copy + mbarrier (sm_90a) ----------------------------------
#ifdef CRANE_EMU
__device__ __forceinline__ void mbar_init(uint64_t*, uint32_t) {}
__device__ __forceinline__ void mbar_expect_tx(uint64_t*, uint32_t) {}
__device__ __forceinline__ void mbar_wait(uint64_t*, uint32_t) {}
__device__ __forceinline__ void tma_load_1d(void* dst, const void* src, uint32_t bytes, uint64_t*) { memcpy(dst, src, bytes); }
__device__ __forceinline__ void fence_mbar_init() {}
#else
__device__ __forceinline__ uint32_t smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }
__device__ __forceinline__ void mbar_init(uint64_t* bar, uint32_t count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count) : "memory");
}
__device__ __forceinline__ void fence_mbar_init() {
  asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
}
__device__ __forceinline__ void mbar_expect_tx(uint64_t* bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes) : "memory");
}
__device__ __forceinline__ void mbar_wait(uint64_t* bar, uint32_t parity) {
  uint32_t done = 0;
  const uint32_t addr = smem_u32(bar);
  while (!done) {
    asm volatile(
        "{\n"
        ".reg .pred p;\n"
        "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n"
        "selp.u32 %0, 1, 0, p;\n"
        "}\n"
        : "=r"(done)
        : "r"(addr), "r"(parity)
        : "memory");
  }
}
__device__ __forceinline__ void tma_load_1d(void* dst, const void* src, uint32_t bytes, uint64_t* bar) {
  asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(smem_u32(dst)),
               "l"(src), "r"(bytes), "r"(smem_u32(bar))
               : "memory");
}
#endif

// named barrier among `nthreads` threads (whole warps) of the CTA; id 1..15 (0 is __syncthreads)
__device__ __forceinline__ void named_bar_sync(uint32_t id, uint32_t nthreads) {
#ifdef CRANE_EMU
  emu_named_bar((int)id, (int)nthreads, true);
#else
  asm volatile("bar.sync %0, %1;" ::"r"(id), "r"(nthreads) : "memory");
#endif
}

// ResourceView::GetFeasibleResourceInNode with the concrete pick, one shared
// out-of-line instance for the cold paths
__device__ __noinline__ bool feasible_alloc(const View& req, const Row& avail, Row& alloc, uint32_t dslot) {
  return feasible<true>(req, avail, c_dicts[dslot], &alloc);
}

__device__ __forceinline__ bool key_lt(double c, uint32_t o, double kc, uint32_t ko) {
  return (c < kc) || (c == kc && o < ko);
}
__device__ __forceinline__ unsigned long long vmax8(unsigned long long a, unsigned long long b) {
  return (unsigned long long)__vmaxu4((unsigned)a, (unsigned)b) |
         (unsigned long long)__vmaxu4((unsigned)(a >> 32), (unsigned)(b >> 32)) << 32;
}


}  // namespace crane
