// commit_v2.cuh — K-commit, second design: the sequential job loop of
// SchedulerAlgo::NodeSelect (JobScheduler.cpp:5777-5867) as batches of up to
// 32 consecutive jobs, every phase data-parallel over the whole CTA.
//
// One persistent CTA per partition (the reference's LocalScheduler,
// JobScheduler.cpp:5757-5766). The CTA's 256 threads are 32 GROUPS of 8 lanes.
// A batch is a run of consecutive jobs (<= 32 jobs, <= 32 nodes in total):
//
//   select    group t lists, for job t, the first candidates in (cost, node)
//             order (JobScheduler.cpp:5224-5266): nodes that are capable
//             (bitmap bit, timeline below the size cap) and pass a pre-filter
//             on the first timeline segment — a necessary condition for the
//             window test because availability only shrinks inside a tick;
//             with fewer than node_num of them, the first capable nodes,
//             which is where a backfill goes (JobScheduler.cpp:5269-5278);
//   validate  (for a few batches after a pick failed the exact test) every listed
//             candidate of the immediate-start jobs is tested exactly, at once;
//             the lists keep the passing ones (validate2);
//   resolve   in job order every job takes its first node_num free candidates:
//             warp 0 walks the jobs (lane = list entry, a taken node is marked
//             in its scratch word, the next job's list is prefetched). A job
//             that could use a node taken by an earlier job of the batch at
//             that node's NEW place in the order ends the batch: it needs the
//             updated timeline (a node the earlier job filled is no candidate). Warps 1-7 meanwhile test every slot's first
//             guess (the entry taken if the jobs before take the entries before);
//   evaluate  group w runs the exact test of task w = (job, node) without
//             touching state: window minimum (JobScheduler.cpp:5285-5334) or
//             allocation against res_total + earliest common start
//             (JobScheduler.h:806-849; the nodes of a job iterate T <- max of
//             their earliest fits to the fixed point);
//   commit    the jobs before the first failing one are placed: concrete
//             cores/slots (PublicHeader.cpp:519-599), timeline update
//             (JobScheduler.h:334-453), outputs, reason label
//             (JobScheduler.cpp:5829-5848);
//   re-key    UpdateCost (JobScheduler.h:520-532) for all placed nodes at once:
//             the order is a flat array; a surviving entry's shift is constant
//             between the sorted places where nodes leave or arrive, so the
//             affected range is copied segment by segment (warps 0-3, while
//             warps 4-7 commit, when the batch has at most 16 tasks).
//
// The job at which a batch stops (its pick failed the exact test, so the walk
// has to continue past it), jobs wider than a batch, jobs with a general task
// distribution and tiny partitions take the ONE-JOB PATH (single2): the same
// walk in windows of 256 order positions, up to 32 candidates of a window tested
// exactly at once, the first node_num passing ones taken.
//
// Why the result equals the sequential loop: a job's pick is "the first K nodes
// in the order that pass". Candidates of the batch-start state are a superset
// of the passing nodes of any later state (monotonicity), nodes not touched by
// the batch look the same in every state, and a touched node only matters for
// job t if it sorts before t's last pick at its new key — exactly the case
// that ends the batch. Every phase boundary is a CTA barrier; there are no
// polled words and no warp-specialised barrier sites in this kernel.
#pragma once

namespace crane {

constexpr int kT2 = 256;           // threads per CTA
constexpr int kGL = 8;             // lanes per group
constexpr int kNG = kT2 / kGL;     // 32 groups
constexpr int kMaxJ = 32;          // jobs per batch
constexpr int kMaxT = kNG;         // (job, node) tasks per batch: one group each
constexpr int kBlk = 32;           // order positions per bounds block
constexpr int kRingMax = 64;       // prefetch ring depth (jobs)
constexpr int kValidateFor = 8;    // batches with up-front validation after a pick failed the exact test
constexpr int kSpare = 12;         // ... during which every job lists this many candidates more than it needs
constexpr int kRK = 64;            // nodes re-keyed by one event-based rebuild (more: full sort)
constexpr int kHeapMax = 128;      // general task distribution: top-K heaps of up to 127 nodes
constexpr int kDeltaClasses = 4;   // res_total classes with a pre-computed cost delta per batch job
static_assert(kMaxT <= 32 && kMaxJ <= 32, "resolve lays a batch over one warp's ballots");

struct Smem2 {
  double* cost;                 // [mp]  NodeRater::cost
  long long* cpu0;              // [mp]  cpu of the first timeline segment
  unsigned long long* gcnt;     // [mp]  packed gres slot counts of the first segment
  long long* bmax_cpu;          // [nblk] max cpu0 over the block
  long long* bmax_cpug;         // [nblk] max cpu0 over the block's nodes with a free gres slot
  unsigned long long* bmax_g;   // [nblk] per-byte max of gcnt over the block
  uint32_t* scratch;            // [mp+1] claim words (resolve) / shift marks (re-key) / list2 (one-job path)
  uint32_t* bits_ring;          // [ring][words]
  uint16_t* ord;                // [mp]  node at order position p: ascending (cost, node), NodeSelector's std::set (JobScheduler.h:588)
  uint16_t* tmp;                // [mp]  re-key scratch
  uint16_t* posn;               // [mp]  position of a node
  uint16_t* nseg;               // [mp]  timeline entry count
  uint16_t* list;               // = tmp: picks of the one-job path
  uint8_t* skip;                // [mp]  timeline at the size cap (JobScheduler.cpp:5230)
  uint8_t* cls;                 // [mp]  res_total class
  uint8_t* memb;                // [mp]  bit p: the node belongs to partition p of this scheduler (only with several)
  uint32_t nblk, ring;
};
constexpr int kMaxCompParts = 8;   // partitions of one scheduler that share nodes (one NodeState, several LocalSchedulers)
// shared memory of the order of one MORE partition over the same nodes: cost, bounds, ord, tmp, posn
__host__ __device__ inline size_t commit2_extra_bytes(uint32_t mp) {
  const size_t nblk = (mp + kBlk - 1) / kBlk;
  return (((size_t)mp * 8 + nblk * 8 * 3 + (size_t)mp * 2 * 3) + 15) & ~(size_t)15;
}
__host__ __device__ inline size_t commit2_fixed_bytes(uint32_t mp, bool gres, uint32_t nparts = 1) {
  const size_t nblk = (mp + kBlk - 1) / kBlk;
  size_t b = (size_t)mp * 8 * (gres ? 3 : 2) + nblk * 8 * 3 + ((size_t)mp + 4) * 4 + (size_t)mp * 2 * 4 + (size_t)mp * 2 + 256;
  if (nparts > 1) b += 16 + (nparts - 1) * commit2_extra_bytes(mp) + mp;  // + membership byte per node
  return b;
}
// ring slots that fit next to a partition of mp nodes (0 = the partition does not fit)
__host__ __device__ inline uint32_t commit2_ring_slots(uint32_t mp, uint32_t words, bool gres, size_t budget, uint32_t nparts = 1) {
  const size_t fixed = commit2_fixed_bytes(mp, gres, nparts);
  if (fixed >= budget) return 0;
  size_t r = (budget - fixed) / ((size_t)words * 4);
  if (r > (size_t)kRingMax) r = kRingMax;
  return r >= (size_t)kMaxJ + 4 ? (uint32_t)r : 0u;
}
__host__ __device__ inline size_t commit2_smem_bytes(uint32_t mp, uint32_t words, bool gres, uint32_t ring, uint32_t nparts = 1) {
  return commit2_fixed_bytes(mp, gres, nparts) + (size_t)ring * words * 4;
}

// ---- groups of 8 lanes ---------------------------------------------------------
// All 32 lanes of a warp execute every collective below (4 groups in lock-step);
// a group without work passes act = false and follows the loops.
__device__ __forceinline__ uint32_t g_lane() { return threadIdx.x & (kGL - 1); }
__device__ __forceinline__ uint32_t g_index() { return threadIdx.x / kGL; }
__device__ __forceinline__ uint32_t g_shift() { return (uint32_t)lane_id() & ~(uint32_t)(kGL - 1); }
__device__ __forceinline__ uint32_t g_ballot(bool p) { return (__ballot_sync(kFullMask, p) >> g_shift()) & ((1u << kGL) - 1u); }
__device__ __forceinline__ int64_t g_bcast_i64(int64_t v, uint32_t src) { return shfl_i64(v, (int)(g_shift() + src)); }
__device__ __forceinline__ uint64_t g_and64(uint64_t v) {
#pragma unroll
  for (int o = 1; o < kGL; o <<= 1) v &= shfl_u64(v, lane_id() ^ o);
  return v;
}

// ---- a node's timeline worked on by one group ------------------------------------
struct Win2 {            // window minimum of one node (JobScheduler.cpp:5314-5319)
  uint64_t c0, c1, c2, c3, g0, g1;
  int64_t cpu;           // cpu/mem/mem_sw minima (g_window<true> only)
  uint64_t mem, mem_sw;
  bool ok;               // cpu/mem (or, exclusive: res_total) hold in every segment of the window
};

// Segments that start before w_end: cpu/mem tested per segment, core and gres
// masks AND-reduced ("the window minimum", algebra.cuh). Exclusive jobs: every
// segment must still hold res_total (JobScheduler.cpp:5285-5293). kMinima: the
// cpu/mem/mem_sw minima over the window too (general task distribution, which
// counts tasks on the window minimum row itself).
template <bool kMinima = false>
__device__ __forceinline__ void g_window(const TlEntry* E, uint32_t n, int64_t w_end, int64_t req_cpu, uint64_t req_mem,
                                         bool exclusive, bool with_gres, const Row& tot, bool act, Win2& w) {
  const uint32_t gl = g_lane();
  const uint64_t ones = ~0ull;
  uint64_t c0 = ones, c1 = ones, c2 = ones, c3 = ones, g0 = ones, g1 = ones;
  int64_t mcpu = INT64_MAX;
  uint64_t mmem = ones, msw = ones;
  bool ok = true, more = act;
  for (uint32_t base = 0; __any_sync(kFullMask, more); base += kGL) {
    const uint32_t i0 = base + gl;
    const bool ld0 = more && i0 < n;
    TlEntry e0;
    e0.t = kInf;
    if (ld0) e0 = E[i0];
    const bool in0 = ld0 && e0.t < w_end;
    if (in0) {
      if constexpr (kMinima) {
        mcpu = e0.seg.cpu_raw < mcpu ? e0.seg.cpu_raw : mcpu;
        mmem = e0.seg.mem < mmem ? e0.seg.mem : mmem;
        msw = e0.seg.mem_sw < msw ? e0.seg.mem_sw : msw;
      }
      if (exclusive) ok = ok && row_le(tot, e0.seg);
      else {
        ok = ok && e0.seg.cpu_raw >= req_cpu && e0.seg.mem >= req_mem;
        if (!core_empty(e0.seg)) { c0 &= e0.seg.core[0]; c1 &= e0.seg.core[1]; c2 &= e0.seg.core[2]; c3 &= e0.seg.core[3]; }
        g0 &= e0.seg.g[0];
        g1 &= e0.seg.g[1];
      }
    }
    const uint32_t gb = g_ballot(in0);
    if (gb != (1u << kGL) - 1u) more = false;  // entries are time-sorted: the window (or the timeline) ends in this chunk
  }
  w.ok = g_ballot(!ok) == 0;
  w.c0 = ones; w.c1 = ones; w.c2 = ones; w.c3 = ones; w.g0 = ones; w.g1 = ones;
  if (__any_sync(kFullMask, act && !exclusive)) {
    w.c0 = g_and64(c0); w.c1 = g_and64(c1); w.c2 = g_and64(c2); w.c3 = g_and64(c3);
    if (__any_sync(kFullMask, act && with_gres)) { w.g0 = g_and64(g0); w.g1 = g_and64(g1); }
  }
  if constexpr (kMinima) {
#pragma unroll
    for (int o = 1; o < kGL; o <<= 1) {
      const int64_t oc = shfl_i64(mcpu, lane_id() ^ o);
      const uint64_t om = shfl_u64(mmem, lane_id() ^ o), os = shfl_u64(msw, lane_id() ^ o);
      mcpu = oc < mcpu ? oc : mcpu;
      mmem = om < mmem ? om : mmem;
      msw = os < msw ? os : msw;
    }
    w.cpu = mcpu; w.mem = mmem; w.mem_sw = msw;
  }
}
// the row GetFeasibleResourceInNode sees for an immediate start: res_avail
// Ckmin'ed with the window (cpu/mem already verified segment by segment)
__device__ __forceinline__ void win_row(const Win2& w, const Row& a0, const View& req, Row& wr) {
  wr.cpu_raw = req.cpu_raw;
  wr.mem = req.mem;
  wr.mem_sw = 0;
  wr.core[0] = a0.core[0] & w.c0; wr.core[1] = a0.core[1] & w.c1;
  wr.core[2] = a0.core[2] & w.c2; wr.core[3] = a0.core[3] & w.c3;
  wr.g[0] = a0.g[0] & w.g0; wr.g[1] = a0.g[1] & w.g1;
}
// the same with cpu/mem/mem_sw Ckmin'ed as well (w from g_window<true>): the row
// the general task distribution counts tasks on
__device__ __forceinline__ void win_row_min(const Win2& w, const Row& a0, const View& req, Row& wr) {
  win_row(w, a0, req, wr);
  wr.cpu_raw = a0.cpu_raw < w.cpu ? a0.cpu_raw : w.cpu;
  wr.mem = a0.mem < w.mem ? a0.mem : w.mem;
  wr.mem_sw = a0.mem_sw < w.mem_sw ? a0.mem_sw : w.mem_sw;
}

// earliest t >= T0 such that `alloc` <= every segment overlapping [t, t+limit)
// on this node, kInf if none (per-node half of EarliestStartSubsetSelector,
// JobScheduler.h:731-784, 806-849). Run starts come from the ballot of breakers.
__device__ __forceinline__ int64_t g_earliest(const TlEntry* E, uint32_t n, const Row& alloc, int64_t T0, int64_t limit, bool act) {
  const uint32_t gl = g_lane();
  int64_t carry = -1, result = kInf;
  bool more = act;
  for (uint32_t base = 0; __any_sync(kFullMask, more); base += kGL) {
    const uint32_t i = base + gl;
    int64_t t = kInf, tend = kInf;
    bool sat = false;
    if (more && i < n) {
      const TlEntry e = E[i];
      t = e.t;
      tend = (i + 1 < n) ? E[i + 1].t : kInf;
      sat = tend > T0 && row_le(alloc, e.seg);
    }
    const uint32_t bm = g_ballot(!sat);
    const uint32_t below = bm & ((1u << gl) - 1u);
    const uint32_t r = below ? 32u - (uint32_t)__clz((int)below) : 0u;  // first lane of my run in this chunk
    int64_t rs = g_bcast_i64(t, r);
    rs = rs > T0 ? rs : T0;
    if (!below && carry >= 0) rs = carry;  // the run started in an earlier chunk
    const bool ok = sat && (tend == kInf || tend - rs >= limit);
    const uint32_t okm = g_ballot(ok);
    const int64_t first_ok = g_bcast_i64(rs, okm ? (uint32_t)__ffs((int)okm) - 1u : 0u);
    const int64_t last = g_bcast_i64(rs, kGL - 1);
    if (more) {
      if (okm) { result = first_ok; more = false; }
      else {
        carry = ((bm >> (kGL - 1)) & 1u) ? -1 : last;
        if (base + kGL >= n) more = false;
      }
    }
  }
  return result;
}

// NodeState::UpdateResourceInNode (JobScheduler.h:334-453, allocation
// direction): breakpoints at start/end, subtract inside [start, end); in place,
// entries above the start move upward top chunk first. Returns the new entry
// count; seg0 = the (new) first segment.
__device__ __forceinline__ uint32_t g_update(TlEntry* E, uint32_t n, int64_t start, int64_t end, const Row& alloc, bool act, Row& seg0) {
  const uint32_t gl = g_lane();
  uint32_t cnt_s = 0, cnt_e = 0;
  bool has_s = false, has_e = false, more = act;
  for (uint32_t base = 0; __any_sync(kFullMask, more); base += kGL) {
    const uint32_t i = base + gl;
    const int64_t t = (more && i < n) ? E[i].t : kInf;
    const uint32_t ms = g_ballot(t <= start), me = g_ballot(t <= end);
    const uint32_t hs = g_ballot(t == start), he = g_ballot(t == end);
    if (more) {
      cnt_s += (uint32_t)__popc(ms);
      cnt_e += (uint32_t)__popc(me);
      has_s = has_s || hs != 0;
      has_e = has_e || he != 0;
      if (me != (1u << kGL) - 1u) more = false;
    }
  }
  uint32_t i_s = 0, i_e = 0, ins_s = 0, ins_e = 0;
  if (act) {
    i_s = cnt_s - 1; i_e = cnt_e - 1;
    ins_s = has_s ? 0u : 1u; ins_e = has_e ? 0u : 1u;
  }
  // entries (i_s, hi] move/subtract; above i_e nothing changes unless a breakpoint
  // is inserted. The lane that moves entry i_e also writes the new breakpoint at
  // `end`, which keeps the un-subtracted value.
  int32_t hi = act ? ((ins_s + ins_e) ? (int32_t)n - 1 : (int32_t)i_e) : -1;
  const int32_t lo = (int32_t)i_s + 1;
  more = act && hi >= lo;
  while (__any_sync(kFullMask, more)) {
    const int32_t j = hi - (int32_t)gl;
    const bool a = more && j >= lo;
    TlEntry e;
    e.t = 0;
    if (a) e = E[j];
    __syncwarp();
    if (a) {
      if ((uint32_t)j == i_e && ins_e) {
        TlEntry f;
        f.t = end;
        f.seg = e.seg;
        E[i_e + ins_s + 1] = f;
      }
      if (e.t < end) row_sub(e.seg, alloc);
      E[(uint32_t)j + ins_s + ((uint32_t)j > i_e ? ins_e : 0u)] = e;
    }
    __syncwarp();
    hi -= kGL;
    if (hi < lo) more = false;
  }
  if (act && gl == 0) {  // the entry covering `start`: never moved
    TlEntry e = E[i_s];
    if (i_e == i_s && ins_e) {
      TlEntry f;
      f.t = end;
      f.seg = e.seg;
      E[i_e + ins_s + 1] = f;
    }
    row_sub(e.seg, alloc);
    if (ins_s) { e.t = start; E[i_s + 1] = e; } else { E[i_s] = e; }  // cases #3 / #4 of JobScheduler.h:343-412
  }
  __syncwarp();
  if (act) seg0 = E[0].seg;
  return n + ins_s + ins_e;
}

// The dynamic shared memory of k_commit2 and its carve-up. Every function derives
// the pointers from the array itself (never loads them from memory), so the
// compiler keeps the accesses in the shared address space (LDS/STS, not generic).
#ifdef CRANE_EMU
#define CRANE_DYN_BASE() (reinterpret_cast<unsigned char*>((reinterpret_cast<uintptr_t>(emu::tctx.block->dyn_smem.data()) + 15) & ~uintptr_t(15)))
#else
extern __shared__ __align__(16) unsigned char crane_dyn_smem2[];
#define CRANE_DYN_BASE() (crane_dyn_smem2)
#endif
__device__ __forceinline__ Smem2 smem2_layout(uint32_t mp, uint32_t words, uint32_t ring, bool gres, uint32_t nparts = 1, uint32_t part = 0) {
  Smem2 sm;
  sm.nblk = (mp + kBlk - 1) / kBlk;
  sm.ring = ring;
  unsigned char* ptr = CRANE_DYN_BASE();  // 16-byte aligned; widest element types first
  sm.cost = reinterpret_cast<double*>(ptr); ptr += (size_t)mp * 8;
  sm.cpu0 = reinterpret_cast<long long*>(ptr); ptr += (size_t)mp * 8;
  sm.gcnt = gres ? reinterpret_cast<unsigned long long*>(ptr) : nullptr;  // a cluster without gres keeps no slot counts
  if (gres) ptr += (size_t)mp * 8;
  sm.bmax_cpu = reinterpret_cast<long long*>(ptr); ptr += (size_t)sm.nblk * 8;
  sm.bmax_cpug = reinterpret_cast<long long*>(ptr); ptr += (size_t)sm.nblk * 8;
  sm.bmax_g = reinterpret_cast<unsigned long long*>(ptr); ptr += (size_t)sm.nblk * 8;
  ptr += (16u - (uint32_t)(((size_t)mp * (gres ? 24 : 16) + (size_t)sm.nblk * 24) & 15u)) & 15u;
  sm.bits_ring = reinterpret_cast<uint32_t*>(ptr); ptr += (size_t)ring * words * 4;
  sm.scratch = reinterpret_cast<uint32_t*>(ptr); ptr += ((size_t)mp + 4) * 4;
  sm.ord = reinterpret_cast<uint16_t*>(ptr); ptr += (size_t)mp * 2;
  sm.tmp = reinterpret_cast<uint16_t*>(ptr); ptr += (size_t)mp * 2;
  sm.posn = reinterpret_cast<uint16_t*>(ptr); ptr += (size_t)mp * 2;
  sm.nseg = reinterpret_cast<uint16_t*>(ptr); ptr += (size_t)mp * 2;
  sm.list = sm.tmp;  // the one-job path's picks: consumed before the re-key writes tmp
  sm.skip = ptr; ptr += mp;
  sm.cls = ptr; ptr += mp;
  sm.memb = nullptr;
  if (nparts > 1) {
    // overlapping partitions: one order per partition over the same node states
    // (NodeSelector per LocalScheduler, JobScheduler.cpp:5757-5762); partition 0 uses
    // the arrays above, every further one a block of its own
    ptr += (16u - (uint32_t)(reinterpret_cast<uintptr_t>(ptr) & 15u)) & 15u;
    if (part > 0) {
      unsigned char* x = ptr + (size_t)(part - 1) * commit2_extra_bytes(mp);
      sm.cost = reinterpret_cast<double*>(x); x += (size_t)mp * 8;
      sm.bmax_cpu = reinterpret_cast<long long*>(x); x += (size_t)sm.nblk * 8;
      sm.bmax_cpug = reinterpret_cast<long long*>(x); x += (size_t)sm.nblk * 8;
      sm.bmax_g = reinterpret_cast<unsigned long long*>(x); x += (size_t)sm.nblk * 8;
      sm.ord = reinterpret_cast<uint16_t*>(x); x += (size_t)mp * 2;
      sm.tmp = reinterpret_cast<uint16_t*>(x); x += (size_t)mp * 2;
      sm.posn = reinterpret_cast<uint16_t*>(x);
      sm.list = sm.tmp;
    }
    sm.memb = ptr + (size_t)(nparts - 1) * commit2_extra_bytes(mp);
  }
  return sm;
}

// ---- per-CTA state in static shared memory (file scope: every function of this
// kernel reaches it without pointer chasing) ----------------------------------------
struct BJob2 {          // one job of the batch
  uint32_t slot;        // ring slot
  uint32_t K;           // node_num
  uint32_t need;        // nodes of this job and of the jobs before it: candidates worth listing
  uint32_t tfirst;      // need - K: its tasks are [tfirst, need)
  uint32_t n0, n1;      // candidates listed: pre-filter (immediate start) / capable (backfill)
  uint32_t mode;        // 0 immediate start, 1 backfill
  uint32_t state;       // 0 resolved, 1 candidates taken by earlier jobs (wait), 2 fewer than K capable nodes ("Resource"), 3 clash with a re-keyed node (wait)
};
struct BTask2 {         // one (job, node) pair
  uint32_t q;           // node (partition-local)
  uint32_t job;         // index in the batch, 0xffffffff = void slot
  double nc;            // cost of the node once the job is placed
};

struct Commit2Args {
  ClusterDev cl;
  TimelineDev tl;
  const JobQ* jobq;
  const uint32_t* part_job_off;
  const uint32_t* bitmap;
  uint32_t words_per_row;
  uint32_t ring;
  PlaceDev out;
  int64_t now;
  int64_t max_window;
  uint32_t max_jobs;
  uint32_t cost_policy;
  uint32_t gres;              // the cluster has gres entries
  uint32_t dslot;             // the handle's gres dictionary: c_dicts[dslot]
  const View* req_node;       // pending.req_node / req_task (general task distribution only)
  const View* req_task;
  const uint32_t* part_list;  // partitions this launch commits (one CTA each), or null = all
  const uint32_t* sched_nparts;  // [n_vparts] partitions per scheduler
  const uint8_t* slot_memb;      // [n_slots] bit p: the node is in partition p of its scheduler
  unsigned long long* prof;
};

struct Ctx2 {           // per-CTA constants
  ClusterDev cl;
  TimelineDev tl;
  PlaceDev out;
  int64_t now, max_window;
  uint32_t base, mp, words, max_jobs, ring, gres, dslot, cost_policy, part;
  uint32_t ncp;   // partitions of this scheduler (1, or the partitions of a connected component of overlapping ones)
  uint32_t npos;  // positions of the current partition's order (= mp with one partition)
  const View* req_node;
  const View* req_task;
};
#define C_DICT2 (c_dicts[s2_cx.dslot])
#define SM2() smem2_layout(s2_cx.mp, s2_cx.words, s2_cx.ring, s2_cx.gres != 0, s2_cx.ncp, s2_cx.ncp > 1 ? s2_curp : 0u)
// the arrays every partition of a scheduler shares (node summaries), and all arrays of a scheduler with one partition
#define SM2S() smem2_layout(s2_cx.mp, s2_cx.words, s2_cx.ring, s2_cx.gres != 0)

__shared__ Ctx2 s2_cx;
__shared__ uint32_t s2_curp;                   // partition of the job in hand (schedulers with several)
__shared__ uint32_t s2_mcount[kMaxCompParts];  // members per partition
__shared__ JobQ s2_jobs[kRingMax];
__shared__ __align__(8) uint64_t s2_bar[kRingMax];
__shared__ Row s2_classrow[kMaxClasses];
__shared__ BJob2 s2_bj[kMaxJ];
__shared__ BTask2 s2_task[kMaxT];
__shared__ uint32_t s2_tjob[kMaxT + 1];   // job of task slot w, void slots included
__shared__ uint16_t s2_cl[2][kMaxJ][kMaxT];  // [0] pre-filter candidates (immediate start), [1] capable nodes (backfill)
__shared__ uint32_t s2_rk_node[kRK];
__shared__ double s2_rk_nc[kRK];
__shared__ uint32_t s2_ip[kRK], s2_rp[kRK], s2_np[kRK];
__shared__ uint32_t s2_w[kT2 / 32];
__shared__ uint32_t s2_ev_a[2 * kRK];  // re-key: sorted places where the survivors' shift changes (bit 31: a removal)
__shared__ int s2_ev_d[2 * kRK];       // shift behind the event
__shared__ uint16_t s2_long[2 * kRK];  // re-key: the segments copied by all threads
__shared__ uint32_t s2_nlong;
constexpr int kShortSeg = 12;          // longest segment its own thread copies
__shared__ long long s2_e[2][kNG];        // earliest fits: per task (batch) / per group max (one-job path)
__shared__ long long s2_e2[2][kNG];       // per group min (one-job path)
__shared__ long long s2_T0[kMaxJ];
__shared__ uint32_t s2_jst[kMaxJ];        // backfill iteration of a batch job: 0 active, 1 found, 2 failed, 3 not a backfill
__shared__ uint32_t s2_ok[kNG];
__shared__ uint32_t s2_joblabel[kMaxJ];
__shared__ uint16_t s2_chunk[kNG];
__shared__ uint32_t s2_jw[kMaxJ];       // K | tfirst << 8 | mode << 16 | state << 17 | list length << 24
__shared__ double s2_jdelta[kMaxJ][kDeltaClasses];  // cost a node of class c gains when the job is placed on it
__shared__ unsigned long long s2_prof_windows, s2_prof_tests, s2_prof_singles;  // one-job path statistics (profiling builds)
__shared__ uint32_t s2_nj, s2_njr, s2_nbf, s2_cut, s2_pmin, s2_pmax, s2_cutpos, s2_nsel, s2_label;
__shared__ long long s2_gmax_cpu, s2_gmax_cpug;  // maxima over all blocks
__shared__ unsigned long long s2_gmax_g;

__device__ __forceinline__ Row node_total2(uint32_t q) {
  const uint8_t c = SM2S().cls[q];
  if (c != 0xff) return s2_classrow[c];
  return s2_cx.cl.slot_total[s2_cx.base + q];
}
__device__ __forceinline__ int64_t node_total_cpu2(uint32_t q) {
  const uint8_t c = SM2S().cls[q];
  if (c != 0xff) return s2_classrow[c].cpu_raw;
  return s2_cx.cl.slot_total[s2_cx.base + q].cpu_raw;
}

// what the selection needs to know about a job
struct JSel2 {
  const uint32_t* bits;
  int64_t req_cpu;
  uint64_t spec8;
  const uint8_t* name_need;
  uint32_t gnames;
  bool exclusive, has_gres;
};
__device__ __forceinline__ void jsel_load(const JobQ& jq, const uint32_t* bits, JSel2& js) {
  js.bits = bits;
  js.req_cpu = jq.req.cpu_raw;
  js.spec8 = jq.spec8;
  js.name_need = jq.name_need;
  js.gnames = jq_gnames(jq);
  js.exclusive = jq_exclusive(jq);
  js.has_gres = jq_has_gres(jq);
}
__device__ __forceinline__ bool capable2(const Smem2& sm, const JSel2& js, uint32_t q) {
  return ((js.bits[q >> 5] >> (q & 31)) & 1u) && !sm.skip[q];
}
// necessary condition of the window test, on the first segment's counts (cpu0: its
// cpu, which a job of the batch that starts now on the node lowers)
__device__ __forceinline__ bool prefilter_cpu2(const Smem2& sm, const JSel2& js, uint32_t q, int64_t cpu0) {
  if (js.exclusive) return true;
  if (cpu0 < js.req_cpu) return false;
  return !js.has_gres || (sm.gcnt && gres_counts_ok(sm.gcnt[q], js.spec8, js.gnames, js.name_need, C_DICT2));
}
__device__ __forceinline__ bool prefilter2(const Smem2& sm, const JSel2& js, uint32_t q) {
  return prefilter_cpu2(sm, js, q, sm.cpu0[q]);
}
__device__ __forceinline__ bool bounds_admit2(const JSel2& js, long long mcpu, long long mcpug, unsigned long long mg) {
  if (js.exclusive) return true;
  if (js.has_gres) return mcpug >= js.req_cpu && gres_counts_ok(mg, js.spec8, js.gnames, js.name_need, C_DICT2);
  return mcpu >= js.req_cpu;
}
__device__ __forceinline__ bool block_promising2(const Smem2& sm, const JSel2& js, uint32_t b) {
  return bounds_admit2(js, sm.bmax_cpu[b], sm.bmax_cpug[b], sm.bmax_g[b]);
}

// Candidate lists of one batch job, by one group (all groups of the warp in
// lock-step). c0: first `need` nodes in order passing capability + pre-filter;
// c1 (only if c0 came up short): first `need` capable nodes.
__device__ __forceinline__ void select2(const Smem2& sm, uint32_t mp, const JSel2& js, uint32_t need, bool act, uint16_t* c0,
                                        uint16_t* c1, uint32_t& n0_out, uint32_t& n1_out) {
  const uint32_t gl = g_lane();
  const uint16_t* ord = sm.ord;
  uint32_t c = 0, pos = 0;
  bool probed = false;
  // no block at all admits a candidate: only the capable list is needed
  bool more = act && need > 0 && bounds_admit2(js, s2_gmax_cpu, s2_gmax_cpug, s2_gmax_g);
  while (__any_sync(kFullMask, more)) {
    bool pred = false;
    uint32_t q = 0;
    const bool probe = more && !probed;
    if (probe) {  // bounds of the next 8 blocks
      const uint32_t b = pos / kBlk + gl;
      pred = b < sm.nblk && block_promising2(sm, js, b);
    } else if (more) {
      const uint32_t p = pos + gl;
      if (p < mp) {
        q = ord[p];
        pred = capable2(sm, js, q) && prefilter2(sm, js, q);
      }
    }
    const uint32_t gb = g_ballot(pred);
    if (probe) {
      if (gb == 0) pos += kBlk * kGL;
      else { pos += kBlk * ((uint32_t)__ffs((int)gb) - 1u); probed = true; }
      if (pos >= mp) more = false;
    } else if (more) {
      const uint32_t rank = c + (uint32_t)__popc(gb & ((1u << gl) - 1u));
      if (pred && rank < need) c0[rank] = (uint16_t)q;
      c += (uint32_t)__popc(gb);
      pos += kGL;
      if (pos % kBlk == 0) probed = false;
      if (c >= need || pos >= mp) more = false;
    }
  }
  const uint32_t n0 = c < need ? c : need;
  uint32_t cum = 0;
  pos = 0;
  more = act && n0 < need;
  while (__any_sync(kFullMask, more)) {
    bool cap = false;
    uint32_t q = 0;
    const uint32_t p = pos + gl;
    if (more && p < mp) {
      q = ord[p];
      cap = capable2(sm, js, q);
    }
    const uint32_t gb = g_ballot(cap);
    if (more) {
      const uint32_t rank = cum + (uint32_t)__popc(gb & ((1u << gl) - 1u));
      if (cap && rank < need) c1[rank] = (uint16_t)q;
      cum += (uint32_t)__popc(gb);
      pos += kGL;
      if (cum >= need || pos >= mp) more = false;
    }
  }
  n0_out = n0;
  n1_out = cum < need ? cum : need;
}

// MinCpuTimeRatioFirst::UpdateCost (JobScheduler.h:46-52): cost the node gets
// when the job is placed on it
__device__ __forceinline__ double new_cost2(const JobQ& jq, uint32_t q, const double* cost) {
  const int64_t tot_cpu = node_total_cpu2(q);
  return __dadd_rn(cost[q], cost_step(s2_cx.cost_policy, jq.time_limit, jq_exclusive(jq) ? tot_cpu : jq.req.cpu_raw, tot_cpu));
}

// block-wide exclusive prefix over one value per thread (kT2 threads)
__device__ __forceinline__ uint32_t block_excl_scan(uint32_t v, uint32_t& total) {
  const uint32_t lane = lane_id(), wid = warp_id();
  uint32_t inc = v;
#pragma unroll
  for (int o = 1; o < 32; o <<= 1) {
    const uint32_t up = __shfl_up_sync(kFullMask, inc, o);
    if ((int)lane >= o) inc += up;
  }
  if (lane == 31) s2_w[wid] = inc;
  __syncthreads();
  uint32_t off = 0, tot = 0;
#pragma unroll
  for (int w = 0; w < kT2 / 32; ++w) {
    const uint32_t x = s2_w[w];
    if ((uint32_t)w < wid) off += x;
    tot += x;
  }
  __syncthreads();
  total = tot;
  return off + inc - v;
}

// exact bounds of the blocks [b_first, b_last] of the order (one group per
// block), then the maxima over all blocks
__device__ __noinline__ void bounds_recompute2(uint32_t b_first, uint32_t b_last) {
  const Smem2 sm = SM2();
  const uint32_t mp = s2_cx.npos, gl = g_lane();  // positions of the current order
  const uint32_t nb = b_last >= sm.nblk ? sm.nblk : b_last + 1;
  for (uint32_t b0 = b_first; b0 < nb; b0 += kNG) {  // uniform trip count over the CTA
    const uint32_t b = b0 + g_index();
    long long mc = INT64_MIN, mcg = INT64_MIN;
    unsigned long long mg = 0;
    if (b < nb) {
#pragma unroll
      for (uint32_t k = 0; k < kBlk / kGL; ++k) {
        const uint32_t p = b * kBlk + k * kGL + gl;
        if (p < mp) {
          const uint32_t q = sm.ord[p];
          const long long c = sm.cpu0[q];
          const unsigned long long g = sm.gcnt ? sm.gcnt[q] : 0ull;
          mc = c > mc ? c : mc;
          if (g && c > mcg) mcg = c;
          mg = vmax8(mg, g);
        }
      }
    }
#pragma unroll
    for (int o = 1; o < kGL; o <<= 1) {
      const long long oc = __shfl_xor_sync(kFullMask, mc, o), ocg = __shfl_xor_sync(kFullMask, mcg, o);
      mc = oc > mc ? oc : mc;
      mcg = ocg > mcg ? ocg : mcg;
      mg = vmax8(mg, __shfl_xor_sync(kFullMask, mg, o));
    }
    if (b < nb && gl == 0) { sm.bmax_cpu[b] = mc; sm.bmax_cpug[b] = mcg; sm.bmax_g[b] = mg; }
  }
  __syncthreads();
  if (warp_id() == 0) {
    long long mc = INT64_MIN, mcg = INT64_MIN;
    unsigned long long mg = 0;
    for (uint32_t b = lane_id(); b < sm.nblk; b += 32) {
      mc = sm.bmax_cpu[b] > mc ? sm.bmax_cpu[b] : mc;
      mcg = sm.bmax_cpug[b] > mcg ? sm.bmax_cpug[b] : mcg;
      mg = vmax8(mg, sm.bmax_g[b]);
    }
    for (int o = 16; o > 0; o >>= 1) {
      const long long oc = __shfl_xor_sync(kFullMask, mc, o), ocg = __shfl_xor_sync(kFullMask, mcg, o);
      mc = oc > mc ? oc : mc;
      mcg = ocg > mcg ? ocg : mcg;
      mg = vmax8(mg, __shfl_xor_sync(kFullMask, mg, o));
    }
    if (lane_id() == 0) { s2_gmax_cpu = mc; s2_gmax_cpug = mcg; s2_gmax_g = mg; }
  }
  __syncthreads();
}

// (cost, node) rank sort of the whole partition (initial order; re-key of more
// than kRK nodes at once)
__device__ __noinline__ void order_sort2() {
  const Smem2 sm = SM2();
  const uint32_t mp = s2_cx.mp;
  const uint32_t bit = s2_cx.ncp > 1 ? 1u << s2_curp : 0u;  // several partitions: only this one's members are ordered
  for (uint32_t q = threadIdx.x; q < mp; q += kT2) {
    if (bit && !(sm.memb[q] & bit)) { sm.posn[q] = 0xffffu; continue; }
    const double c = sm.cost[q];
    uint32_t rank = 0;
    for (uint32_t o = 0; o < mp; ++o) {
      if (bit && !(sm.memb[o] & bit)) continue;
      const double co = sm.cost[o];
      rank += (co < c || (co == c && o < q)) ? 1u : 0u;
    }
    sm.ord[rank] = (uint16_t)q;
    sm.posn[q] = (uint16_t)rank;
  }
  __syncthreads();
  bounds_recompute2(0, sm.nblk);
}

// Re-key the `cnt` (<= kRK) distinct nodes s2_rk_node[] to the costs
// s2_rk_nc[] (all threads; NodeSelector::UpdateCost, JobScheduler.h:520-532, for
// every placed node at once). A surviving entry at old position p moves to
// p - #removed before p + #new keys at or before p, a shift that is constant
// between the 2*cnt places where a node leaves or arrives: the events are
// sorted and the affected range [first event, last event] is copied segment by
// segment — outside it nothing moves, as many nodes are removed as inserted.
// A re-keyed node lands at (survivors before its lower bound) + (its rank
// among the new keys).
__device__ __noinline__ void order_rekey2(uint32_t cnt, uint32_t nthr) {
  const Smem2 sm = SM2();
  const uint32_t mp = s2_cx.npos, tid = threadIdx.x, lane = lane_id(), wid = warp_id();  // positions of the current order
  if (cnt == 0) return;
  const uint32_t ngr = nthr / kGL;  // the first nthr threads of the CTA take part (named barrier 1)
  if (tid == 0) { s2_pmin = mp; s2_pmax = 0; s2_nlong = 0; }
  named_bar_sync(1, nthr);
  const uint32_t gl = g_lane();
  // lower bound of every new key among the old keys: one group per node, nine-way search
  for (uint32_t w0 = 0; w0 < cnt; w0 += ngr) {
    const uint32_t w = w0 + g_index();
    const bool act = w < cnt;
    const uint32_t u = act ? s2_rk_node[w] : 0u;
    const double nc = act ? s2_rk_nc[w] : 0.0;
    uint32_t lo = 0, hi = act ? mp : 0u;
    while (__any_sync(kFullMask, lo < hi)) {
      const uint32_t width = hi - lo;
      const bool narrow = width <= (uint32_t)kGL;
      const uint32_t p = narrow ? lo + gl : lo + ((gl + 1u) * width) / (uint32_t)(kGL + 1);
      bool lt = false;
      if (lo < hi && p < hi) {
        const uint32_t o = sm.ord[p];
        lt = key_lt(sm.cost[o], o, nc, u);
      }
      const uint32_t c = (uint32_t)__popc(g_ballot(lt));  // keys are sorted: a prefix of the lanes
      if (lo < hi) {
        if (narrow) { lo += c; hi = lo; }
        else {
          const uint32_t nlo = c ? lo + (c * width) / (uint32_t)(kGL + 1) + 1u : lo;
          const uint32_t nhi = c < (uint32_t)kGL ? lo + ((c + 1u) * width) / (uint32_t)(kGL + 1) : hi;
          lo = nlo;
          hi = nhi;
        }
      }
    }
    if (act && gl == 0) {
      const uint32_t rp = sm.posn[u];
      s2_ip[w] = lo;
      s2_rp[w] = rp;
      atomicMin(&s2_pmin, lo < rp ? lo : rp);
      atomicMax(&s2_pmax, lo > rp + 1 ? lo : rp + 1);
    }
  }
  named_bar_sync(1, nthr);
  for (uint32_t w0 = 0; w0 < cnt; w0 += ngr) {
    const uint32_t w = w0 + g_index();
    const bool act = w < cnt;
    uint32_t rank = 0, rem = 0;
    if (act) {
      const uint32_t u = s2_rk_node[w], ip = s2_ip[w];
      const double nc = s2_rk_nc[w];
      for (uint32_t x = gl; x < cnt; x += kGL) {
        rank += key_lt(s2_rk_nc[x], s2_rk_node[x], nc, u) ? 1u : 0u;
        rem += s2_rp[x] < ip ? 1u : 0u;
      }
    }
#pragma unroll
    for (int o = 1; o < kGL; o <<= 1) {
      rank += __shfl_xor_sync(kFullMask, rank, o);
      rem += __shfl_xor_sync(kFullMask, rem, o);
    }
    if (act && gl == 0) s2_np[w] = s2_ip[w] - rem + rank;
  }
  // The survivors of [pmin, pmax) shift by (insertions at or before) - (removals before), which is
  // constant between the 2*cnt places where it changes: sort those events (removals first at equal
  // positions, so the vacated position ends the segment before it), then copy segment by segment.
  const uint32_t pmin = s2_pmin, pmax = s2_pmax;
  const uint32_t nev = 2u * cnt;
  if (tid < nev) {
    const bool is_ins = tid >= cnt;
    const uint32_t x = is_ins ? tid - cnt : tid;
    const uint32_t key = is_ins ? 2u * s2_ip[x] + 1u : 2u * (s2_rp[x] + 1u);
    uint32_t rank = 0;
    int d = is_ins ? 1 : -1;  // shift behind this event: every event up to and including it
    for (uint32_t y = 0; y < cnt; ++y) {
      const uint32_t kr = 2u * (s2_rp[y] + 1u), ki = 2u * s2_ip[y] + 1u;
      const bool rb = kr < key || (kr == key && y < tid);
      const bool ib = ki < key || (ki == key && y + cnt < tid);
      rank += (rb ? 1u : 0u) + (ib ? 1u : 0u);
      d += (ib ? 1 : 0) - (rb ? 1 : 0);
    }
    s2_ev_a[rank] = (key >> 1) | (is_ins ? 0u : 0x80000000u);
    s2_ev_d[rank] = d;
  }
  named_bar_sync(1, nthr);
  // segment k = [event k, event k+1): a short one is copied by its own thread, the long ones
  // (usually the one stretch between where the nodes left and where they arrive) by everybody
  if (tid + 1 < nev) {
    const uint32_t a = s2_ev_a[tid] & 0x7fffffffu, nx = s2_ev_a[tid + 1];
    const uint32_t b = (nx & 0x7fffffffu) - (nx >> 31);  // a removal event at e: position e - 1 is the vacated one
    const int d = s2_ev_d[tid];
    if (b > a + (uint32_t)kShortSeg) {
      s2_long[atomicAdd(&s2_nlong, 1u)] = (uint16_t)tid;
    } else {
      for (uint32_t p = a; p < b; ++p) {
        const uint32_t q = sm.ord[p];
        const uint32_t np = (uint32_t)((int)p + d);
        sm.tmp[np] = (uint16_t)q;
        sm.posn[q] = (uint16_t)np;
      }
    }
  }
  named_bar_sync(1, nthr);
  const uint32_t nlong = s2_nlong;
  for (uint32_t i = 0; i < nlong; ++i) {
    const uint32_t k = s2_long[i];
    const uint32_t a = s2_ev_a[k] & 0x7fffffffu, nx = s2_ev_a[k + 1];
    const uint32_t b = (nx & 0x7fffffffu) - (nx >> 31);
    const int d = s2_ev_d[k];
    for (uint32_t p0 = a + tid; p0 < b; p0 += 2u * nthr) {  // two loads in flight
      const uint32_t p1 = p0 + nthr;
      const bool h1 = p1 < b;
      const uint32_t q0 = sm.ord[p0], q1 = h1 ? sm.ord[p1] : 0u;
      const uint32_t n0 = (uint32_t)((int)p0 + d), n1 = (uint32_t)((int)p1 + d);
      sm.tmp[n0] = (uint16_t)q0;
      sm.posn[q0] = (uint16_t)n0;
      if (h1) { sm.tmp[n1] = (uint16_t)q1; sm.posn[q1] = (uint16_t)n1; }
    }
  }
  if (tid < cnt) {  // (tmp slots no survivor takes; s2_np is complete since the barrier above)
    const uint32_t u = s2_rk_node[tid];
    sm.tmp[s2_np[tid]] = (uint16_t)u;
    sm.posn[u] = (uint16_t)s2_np[tid];
    sm.cost[u] = s2_rk_nc[tid];
  }
  named_bar_sync(1, nthr);
  for (uint32_t p0 = pmin + tid; p0 < pmax; p0 += 2u * nthr) {
    const uint32_t p1 = p0 + nthr;
    const bool h1 = p1 < pmax;
    const uint16_t v0 = sm.tmp[p0], v1 = h1 ? sm.tmp[p1] : (uint16_t)0;
    sm.ord[p0] = v0;
    if (h1) sm.ord[p1] = v1;
  }
  named_bar_sync(1, nthr);
}
// bounds of the blocks a re-key touched (all threads, after order_rekey2)
__device__ __forceinline__ void rekey_bounds2(uint32_t cnt) {
  if (cnt) bounds_recompute2(s2_pmin / kBlk, (s2_pmax < s2_cx.npos ? s2_pmax : s2_cx.npos - 1) / kBlk);
}


// pending-reason label of a job that starts later (JobScheduler.cpp:5829-5865): bit 1 = a node
// of a partition whose first reservation starts inside the job's window ("Resource Reserved"),
// bit 0 = the allocation does not fit the node's res_avail now ("Resource"); none: "Priority"
__device__ __forceinline__ uint32_t later_label2(uint32_t q, bool short_now, int64_t limit) {
  uint32_t l = short_now ? 1u : 0u;
  if (s2_cx.part < s2_cx.cl.n_comp && s2_cx.tl.first_resv[s2_cx.base + q] < s2_cx.now + limit) l |= 2u;
  return l;
}
__device__ __forceinline__ uint8_t later_reason2(uint32_t label) {
  return (label & 2u) ? CRANE_REASON_RESERVED : ((label & 1u) ? CRANE_REASON_RESOURCE : CRANE_REASON_PRIORITY);
}

// n-th (1-based) set bit of m, 32 if there is none
__device__ __forceinline__ uint32_t nth_set_bit(uint32_t m, uint32_t n) {
  if ((uint32_t)__popc(m) < n || n == 0) return 32u;
  uint32_t pos = 0;
#pragma unroll
  for (uint32_t w = 16; w >= 1; w >>= 1) {
    const uint32_t c = (uint32_t)__popc((m >> pos) & ((1u << w) - 1u));
    if (c < n) { n -= c; pos += w; }
  }
  return pos;
}

// outputs of one placed (job, node) pair and the node's new summary, by lane 0 of its group
__device__ __forceinline__ void write_node2(const JobQ& jq, uint32_t q, uint32_t rank, const Row& alloc, uint32_t nn, const Row& seg0) {
  const Smem2 sm = SM2S();
  sm.nseg[q] = (uint16_t)nn;
  if (nn >= s2_cx.max_jobs) sm.skip[q] = 1;
  sm.cpu0[q] = seg0.cpu_raw;
  if (sm.gcnt) sm.gcnt[q] = (seg0.g[0] | seg0.g[1]) ? pack_gres_counts(seg0) : 0ull;
  const uint32_t dst = jq.alloc_off + rank;
  s2_cx.out.alloc_node[dst] = s2_cx.cl.slot_node[s2_cx.base + q];
  s2_cx.out.alloc_ntasks[dst] = jq.ntasks_per_node;
  s2_cx.out.alloc_res[dst] = alloc;
  s2_cx.tl.n[s2_cx.base + q] = nn;
}
// output slot of a job's node q: its rank among the job's K nodes node(0..K) by node index
// (deviation D3), by one group
template <class NodeAt>
__device__ __forceinline__ uint32_t g_out_rank(uint32_t K, uint32_t q, bool act, NodeAt node) {
  uint32_t rank = 0;
  if (act && K > 1)
    for (uint32_t m = g_lane(); m < K; m += kGL) rank += node(m) < q ? 1u : 0u;
#pragma unroll
  for (int o = 1; o < kGL; o <<= 1) rank += __shfl_xor_sync(kFullMask, rank, o);
  return rank;
}
// job-level outputs of a placed job; `label` as later_label2 built it (starts after now only)
__device__ __forceinline__ void write_job2(const JobQ& jq, int64_t start, uint32_t label) {
  s2_cx.out.start_time[jq.job] = start;
  s2_cx.out.end_time[jq.job] = start + jq.time_limit;
  s2_cx.out.n_alloc[jq.job] = jq.node_num;
  s2_cx.out.reason[jq.job] = start == s2_cx.now ? CRANE_REASON_NONE : later_reason2(label);
}

// The exact test of node q for an immediate start of the job, in the current state
// (JobScheduler.cpp:5285-5334): every segment of [now, now + time_limit) holds the
// request (exclusive: res_total), res_avail itself holds it (:5310) and
// GetFeasibleResourceInNode passes on res_avail Ckmin'ed with the window. kAlloc:
// *alloc receives the allocation (exclusive: res_total) of a passing node. By one
// group; every lane of the warp calls it, a group without work with act = false.
template <bool kAlloc>
__device__ __forceinline__ bool g_exact(const JobQ& jq, uint32_t q, bool act, Row* alloc = nullptr) {
  const TimelineDev& tl = s2_cx.tl;
  const bool exclusive = jq_exclusive(jq);
  const uint32_t g = s2_cx.base + (act ? q : 0u);
  const uint32_t ns = act ? SM2S().nseg[q] : 0u;
  Row tot, a0;
  row_zero(tot);
  row_zero(a0);
  if (act) {
    if (exclusive) tot = node_total2(q);
    else a0 = tl.avail0[g];
  }
  Win2 w;
  g_window(tl.ent + (size_t)g * tl.cap, ns, s2_cx.now + jq.time_limit, jq.req.cpu_raw, jq.req.mem, exclusive, jq_has_gres(jq), tot,
           act, w);
  bool ok = act && w.ok;
  if (exclusive) {
    if (kAlloc && act) *alloc = tot;
  } else if (ok) {
    ok = a0.cpu_raw >= jq.req.cpu_raw && a0.mem >= jq.req.mem;  // res_avail itself (JobScheduler.cpp:5310)
    if (ok) {
      Row wr;
      win_row(w, a0, jq.req, wr);
      ok = feasible<kAlloc>(jq.req, wr, C_DICT2, alloc);
    }
  }
  return ok;
}

// Scheduler of several overlapping partitions: membership bytes, one cost array and
// one order per partition over the shared node states; every NodeSelector starts from
// the same NodeRater costs (JobScheduler.h:492-505). All threads; s2_cx is set.
__device__ __noinline__ void init_orders2(const uint8_t* slot_memb) {
  const uint32_t tid = threadIdx.x, mp = s2_cx.mp, ncp = s2_cx.ncp;
  const Smem2 s0 = smem2_layout(mp, s2_cx.words, s2_cx.ring, s2_cx.gres != 0, ncp, 0);
  for (uint32_t q = tid; q < mp; q += kT2) s0.memb[q] = slot_memb[s2_cx.base + q];
  for (uint32_t p = 1; p < ncp; ++p) {
    const Smem2 sp = smem2_layout(mp, s2_cx.words, s2_cx.ring, s2_cx.gres != 0, ncp, p);
    for (uint32_t q = tid; q < mp; q += kT2) sp.cost[q] = s0.cost[q];
  }
  __syncthreads();
  if (tid < ncp) {
    uint32_t c = 0;
    for (uint32_t q = 0; q < mp; ++q) c += (s0.memb[q] >> tid) & 1u;
    s2_mcount[tid] = c;
  }
  __syncthreads();
  for (uint32_t p = 0; p < ncp; ++p) {
    if (tid == 0) { s2_curp = p; s2_cx.npos = s2_mcount[p]; }
    __syncthreads();
    order_sort2();
    __syncthreads();
  }
}

// Scheduler with several (overlapping) partitions: the job in hand decides whose order is walked
__device__ __forceinline__ void enter_partition2(const JobQ& jq) {
  if (s2_cx.ncp > 1) {
    __syncthreads();
    if (threadIdx.x == 0) {
      s2_curp = jq_part(jq);
      s2_cx.npos = s2_mcount[s2_curp];
    }
    __syncthreads();
  }
}

// ---- validation of the candidate lists (all threads) ---------------------------------
// In an over-subscribed partition most nodes that pass the pre-filter (first timeline
// segment) fail the window test — backfill reservations sit on every node — so the
// speculative pick fails, the batch is cut and the job walks the order alone. For a
// few batches after such a failure every immediate-start job lists kSpare candidates
// more than it needs and every listed candidate gets the exact test of the batch-start
// state at once (one group per (job, entry) pair). The list keeps the passing ones, so
// a failing candidate is replaced inside the batch; a job with fewer than node_num
// passing ones in a COMPLETE list (select2 walked to the end of the order) is a backfill
// job (JobScheduler.cpp:5269-5278) right away. Exact: a node that fails now fails in
// every later state of the tick; a listed node that passes and is not touched by an
// earlier job of the batch still is in its batch-start state when the job picks it; and
// everything in front of a pick is either listed (tested) or fails the pre-filter.
__shared__ uint32_t s2_vok[kMaxJ], s2_voff[kMaxJ + 1];
__device__ __noinline__ void validate2(uint32_t nj) {
  const uint32_t tid = threadIdx.x, lane = lane_id(), gl = g_lane(), gi = g_index();
  if (tid < 32) {  // pairs per job, exclusive prefix
    uint32_t c = 0;
    if (lane < nj) {
      const BJob2 b = s2_bj[lane];
      if (b.state == 0 && b.mode == 0) c = b.n0;
      s2_vok[lane] = 0;
    }
    uint32_t inc = c;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
      const uint32_t up = __shfl_up_sync(kFullMask, inc, o);
      if ((int)lane >= o) inc += up;
    }
    if (lane < nj) s2_voff[lane] = inc - c;
    if (lane == 31) s2_voff[kMaxJ] = inc;
  }
  __syncthreads();
  const uint32_t npairs = s2_voff[kMaxJ];
  if (npairs == 0) return;
  for (uint32_t x0 = 0; x0 < npairs; x0 += kNG) {
    const uint32_t x = x0 + gi;
    const bool act = x < npairs;
    // the job of pair x: the last job whose offset is <= x (jobs without pairs share the next one's offset)
    uint32_t t = 0;
    {
      uint32_t best = 0;
      for (uint32_t j = gl; j < nj; j += kGL)
        if (s2_voff[j] <= x) best = j + 1u;
#pragma unroll
      for (int o = 1; o < kGL; o <<= 1) {
        const uint32_t ob = __shfl_xor_sync(kFullMask, best, o);
        best = ob > best ? ob : best;
      }
      t = best ? best - 1u : 0u;
    }
    const uint32_t e = act ? x - s2_voff[t] : 0u;
    const bool ok = g_exact<false>(s2_jobs[s2_bj[t].slot], act ? s2_cl[0][t][e] : 0u, act);
    if (ok && gl == 0) atomicOr(&s2_vok[t], 1u << e);
  }
  __syncthreads();
  // group t compacts the list of job t (every lane of the warp takes part in the ballots)
  {
    BJob2 b;
    b.slot = 0; b.K = 0; b.need = 0; b.tfirst = 0; b.n0 = 0; b.n1 = 0; b.mode = 0; b.state = 0;
    if (gi < nj) b = s2_bj[gi];
    const bool qual = gi < nj && b.state == 0 && b.mode == 0;
    const uint32_t want = b.need + (uint32_t)kSpare < (uint32_t)kMaxT ? b.need + (uint32_t)kSpare : (uint32_t)kMaxT;  // what select2 was asked for
    const bool complete = b.n0 < want;  // the walk reached the end of the order: nothing passes the pre-filter beyond the list
    const uint32_t n0 = qual ? b.n0 : 0u;
    const uint32_t mask = qual ? s2_vok[gi] : 0u;
    uint32_t kept = 0;
    for (uint32_t e0 = 0; e0 < (uint32_t)kMaxT; e0 += kGL) {
      const uint32_t e = e0 + gl;
      const bool keep = e < n0 && ((mask >> e) & 1u);
      const uint16_t v = e < n0 ? s2_cl[0][gi][e] : (uint16_t)0;
      const uint32_t gb = g_ballot(keep);
      __syncwarp();
      if (keep) s2_cl[0][gi][kept + (uint32_t)__popc(gb & ((1u << gl) - 1u))] = v;
      kept += (uint32_t)__popc(gb);
      __syncwarp();
    }
    if (qual && gl == 0) {
      // fewer than K passing ones in a complete list: a backfill job; in a truncated list: the
      // resolve will stop the batch at this job (its walk has to go on past the list)
      const uint32_t mode = (complete && kept < b.K) ? 1u : 0u;
      const uint32_t state = (mode && b.n1 < b.K) ? 2u : 0u;
      s2_bj[gi].n0 = kept; s2_bj[gi].mode = mode; s2_bj[gi].state = state;
      const uint32_t nl = state ? 0u : (mode ? b.n1 : kept);
      s2_jw[gi] = b.K | b.tfirst << 8 | mode << 16 | state << 17 | nl << 24;
      s2_jst[gi] = (state == 0 && mode == 1u && b.K > 1u) ? 0u : 3u;
    }
  }
  __syncthreads();
}

// ---- general task distribution (ntasks_per_node_max > min or an uneven ntasks) --------
// JobScheduler.cpp:5193-5222, 5258-5361: every capable node can take between
// ntasks_per_node_min and _max tasks; the K nodes with the most tasks are kept in a
// std::priority_queue (top = fewest tasks) until K nodes hold >= ntasks tasks; tasks
// are then handed out in pop order. The queue is restated with libstdc++'s own heap
// algorithm (std::push_heap / std::pop_heap: __push_heap, __adjust_heap), so equal
// task counts leave the heap in the reference's order.
struct Heap2 {
  uint16_t nt[kHeapMax];   // tasks the node can take
  uint16_t q[kHeapMax];    // node
  uint32_t size, sum;
};
__shared__ Heap2 s2_heap[2];                 // [0] by res_total (backfill), [1] by the window minimum (immediate start)
__shared__ uint16_t s2_g_nt[2][kNG];         // per window candidate: tasks by res_total / by the window minimum
__shared__ uint16_t s2_g_node[kHeapMax], s2_g_n[kHeapMax];  // hand-out: node, tasks, in pop order
__shared__ uint32_t s2_g_done;

// comp(a, b) of std::priority_queue<Info>: Info::operator< is "has more tasks"
__device__ __forceinline__ bool heap_less2(uint32_t a_nt, uint32_t b_nt) { return a_nt > b_nt; }
__device__ inline void heap_push2(Heap2& h, uint32_t nt, uint32_t q) {  // push_back + std::push_heap
  uint32_t hole = h.size++;
  while (hole > 0) {
    const uint32_t parent = (hole - 1) / 2;
    if (!heap_less2(h.nt[parent], nt)) break;
    h.nt[hole] = h.nt[parent]; h.q[hole] = h.q[parent];
    hole = parent;
  }
  h.nt[hole] = (uint16_t)nt; h.q[hole] = (uint16_t)q;
}
__device__ inline void heap_pop2(Heap2& h) {  // std::pop_heap + pop_back
  const uint32_t len = h.size - 1;
  if (len == 0) { h.size = 0; return; }
  const uint32_t vnt = h.nt[len], vq = h.q[len];   // value = *(last-1); *(last-1) = *first
  uint32_t hole = 0, second = 0;
  while ((int32_t)second < ((int32_t)len - 1) / 2) {  // __adjust_heap
    second = 2 * (second + 1);
    if (heap_less2(h.nt[second], h.nt[second - 1])) --second;
    h.nt[hole] = h.nt[second]; h.q[hole] = h.q[second];
    hole = second;
  }
  if ((len & 1u) == 0 && (int32_t)second == ((int32_t)len - 2) / 2) {
    second = 2 * (second + 1);
    h.nt[hole] = h.nt[second - 1]; h.q[hole] = h.q[second - 1];
    hole = second - 1;
  }
  while (hole > 0) {  // __push_heap(first, hole, 0, value)
    const uint32_t parent = (hole - 1) / 2;
    if (!heap_less2(h.nt[parent], vnt)) break;
    h.nt[hole] = h.nt[parent]; h.q[hole] = h.q[parent];
    hole = parent;
  }
  h.nt[hole] = (uint16_t)vnt; h.q[hole] = (uint16_t)vq;
  h.size = len;
}

// get_max_tasks (JobScheduler.cpp:5207-5222): tasks the row can take, 0 if not even the minimum
__device__ __noinline__ uint32_t max_tasks2(const View& min_view, const View& req_task, uint32_t tmin, uint32_t tmax, const Row& res) {
  Row got;
  if (!feasible<true>(min_view, res, C_DICT2, &got)) return 0;
  Row rest = res;
  row_sub(rest, got);
  uint32_t n = tmin;
  while (n < tmax && feasible<true>(req_task, rest, C_DICT2, &got)) {
    ++n;
    row_sub(rest, got);
  }
  return n;
}

// ---- the one-job path: one job, start to finish (any node_num), JobScheduler.cpp:5224-5404 ----
// The walk over the order in windows of 256 positions; up to 32 candidates of a
// window are tested at once, one group each. Uniform tasks (kGeneral = false): the
// candidates are the pre-filter ones, each gets the exact test, the first K passing
// ones are the pick and with fewer than K the job backfills on the first K capable
// nodes. General task distribution: every capable node counts the tasks it can take
// by res_total and by the window minimum into the two heaps above, which decide.
// Both then share the earliest common start, the placement and the job tail.
template <bool kGeneral>
__device__ __noinline__ void single2(uint32_t ji) {
  enter_partition2(s2_jobs[ji % s2_cx.ring]);
  const Smem2 sm = SM2();
  const uint32_t tid = threadIdx.x, gl = g_lane(), gi = g_index();
  const uint32_t mp = s2_cx.npos, base = s2_cx.base, ring = s2_cx.ring;
  const int64_t now = s2_cx.now;
  const TimelineDev& tl = s2_cx.tl;
  const uint32_t slot = ji % ring;
  mbar_wait(&s2_bar[slot], (ji / ring) & 1u);
  const JobQ& jq = s2_jobs[slot];
  JSel2 js;
  jsel_load(jq, sm.bits_ring + (size_t)slot * s2_cx.words, js);
  const uint32_t K = jq.node_num;
  const bool exclusive = js.exclusive;
  const int64_t limit = jq.time_limit;
  const View req = jq.req;  // general task distribution: what a node needs at least (min_res_view)
  const int64_t w_end = now + limit;
  // general task distribution: a node with n tasks needs req_node + n * req_task
  const View req_node = kGeneral ? s2_cx.req_node[jq.job] : req, req_task = kGeneral ? s2_cx.req_task[jq.job] : req;
  const uint32_t tmin = jq.ntasks_per_node, tmax = jq.ntpn_max, ntasks = jq.ntasks;
  if (K > mp || K == 0 || (kGeneral && K >= (uint32_t)kHeapMax)) {
    if (tid == 0) s2_cx.out.reason[jq.job] = CRANE_REASON_RESOURCE;
    return;
  }
  uint16_t* const list2 = reinterpret_cast<uint16_t*>(sm.scratch);  // uniform tasks: the first K capable nodes
  uint32_t nsel = 0, ntot = 0, pos = 0;
  if (tid == 0) {
    s2_label = 0;
    if (kGeneral) { s2_heap[0].size = 0; s2_heap[0].sum = 0; s2_heap[1].size = 0; s2_heap[1].sum = 0; s2_g_done = 0; }
  }
  if (kGeneral) __syncthreads();
#ifdef CRANE_PROFILE
  if (!kGeneral && tid == 0) s2_prof_singles += 1;
#endif
  while (pos < mp && (kGeneral ? !s2_g_done : nsel < K)) {
    // skip a window none of whose blocks can hold a candidate (once the first K
    // capable nodes are known)
    if (!kGeneral && ntot >= K) {
      bool any = false;
      for (uint32_t b = pos / kBlk; b < sm.nblk && b < (pos + kT2) / kBlk; ++b) any = any || block_promising2(sm, js, b);
      if (!any) { pos += kT2; continue; }
    }
    const uint32_t p = pos + tid;
    uint32_t q = 0;
    bool cap = false, cand = false;
    if (p < mp) {
      q = sm.ord[p];
      cap = capable2(sm, js, q);
      cand = cap && (kGeneral || prefilter2(sm, js, q));
    }
    if (tid == 0) s2_cutpos = pos + kT2;
    uint32_t totc;
    const uint32_t rank_c = block_excl_scan(cand ? 1u : 0u, totc);
    const uint32_t ncand = totc < (uint32_t)kNG ? totc : (uint32_t)kNG;
#ifdef CRANE_PROFILE
    if (!kGeneral && tid == 0) { s2_prof_windows += 1; s2_prof_tests += ncand; }
#endif
    if (cand && rank_c < (uint32_t)kNG) s2_chunk[rank_c] = (uint16_t)q;
    if (cand && rank_c == (uint32_t)kNG - 1u && totc > (uint32_t)kNG) s2_cutpos = p + 1;  // the rest of the window comes back
    __syncthreads();
    const uint32_t cutpos = s2_cutpos;
    if constexpr (kGeneral) {
      // tasks every candidate can take by res_total and by the window minimum
      // (JobScheduler.cpp:5258-5334), one group each
      const bool act = gi < ncand;
      uint32_t qg = 0, g = 0, ns = 0;
      Row tot, a0;
      row_zero(tot);
      row_zero(a0);
      bool fits = false;  // res_avail holds the minimum (JobScheduler.cpp:5310)
      if (act) {
        qg = s2_chunk[gi];
        g = base + qg;
        ns = sm.nseg[qg];
        tot = node_total2(qg);
        a0 = tl.avail0[g];
        fits = !exclusive && feasible<false>(req, a0, C_DICT2, nullptr);
      }
      Win2 w;
      g_window<true>(tl.ent + (size_t)g * tl.cap, ns, w_end, req.cpu_raw, req.mem, exclusive, true, tot, act && (exclusive || fits), w);
      if (act && gl == 0) {
        const uint32_t n_total = max_tasks2(req, req_task, tmin, tmax, tot);  // > 0: the node is capable
        uint32_t n_avail = 0;
        if (exclusive) {
          n_avail = w.ok ? n_total : 0u;  // JobScheduler.cpp:5285-5307
        } else if (fits) {
          Row wr;
          win_row_min(w, a0, req, wr);
          n_avail = max_tasks2(req, req_task, tmin, tmax, wr);
        }
        s2_g_nt[0][gi] = (uint16_t)n_total;
        s2_g_nt[1][gi] = (uint16_t)n_avail;
      }
      __syncthreads();
      // heaps, in node order (one thread: the reference's loop body, JobScheduler.cpp:5269-5334)
      if (tid == 0) {
        Heap2& ht = s2_heap[0];
        Heap2& ha = s2_heap[1];
        for (uint32_t c = 0; c < ncand; ++c) {
          const uint32_t n_total = s2_g_nt[0][c], n_avail = s2_g_nt[1][c], qn = s2_chunk[c];
          if (n_total == 0) continue;
          if (ht.size < K || ht.sum < ntasks) {
            ht.sum += n_total;
            heap_push2(ht, n_total, qn);
            if (ht.size > K) { ht.sum -= ht.nt[0]; heap_pop2(ht); }
          }
          if (n_avail) {
            ha.sum += n_avail;
            heap_push2(ha, n_avail, qn);
            if (ha.size > K) { ha.sum -= ha.nt[0]; heap_pop2(ha); }
            if (ha.size == K && ha.sum >= ntasks) { s2_g_done = 1; break; }
          }
        }
      }
      __syncthreads();
    } else {
      // the first K capable nodes in order: where a backfill goes (JobScheduler.cpp:5269-5278)
      const bool capc = cap && p < cutpos && ntot < K;
      uint32_t tott;
      const uint32_t rank_t = block_excl_scan(capc ? 1u : 0u, tott);
      if (capc && ntot + rank_t < K) list2[ntot + rank_t] = (uint16_t)q;
      ntot = ntot + tott < K ? ntot + tott : K;
      // the exact test of the window's candidates, one group each
      const bool act = gi < ncand;
      const bool ok = g_exact<false>(jq, act ? s2_chunk[gi] : 0u, act);
      if (gl == 0) s2_ok[gi] = ok ? 1u : 0u;
      __syncthreads();
      if (warp_id() == 0) {  // the passing ones, in order
        const uint32_t lane = lane_id();
        const bool okl = lane < ncand && s2_ok[lane];
        const unsigned m = __ballot_sync(kFullMask, okl);
        const uint32_t r = nsel + (uint32_t)__popc(m & ((1u << lane) - 1u));
        if (okl && r < K) sm.list[r] = s2_chunk[lane];
        if (lane == 0) s2_nsel = nsel + (uint32_t)__popc(m) < K ? nsel + (uint32_t)__popc(m) : K;
      }
      __syncthreads();
      nsel = s2_nsel;
    }
    pos = cutpos;
  }

  // ---- the decision (JobScheduler.cpp:5338-5404): start now on `nodes`, or backfill on them
  bool start_now, can_bf;
  const uint16_t* nodes;
  if constexpr (kGeneral) {
    start_now = s2_heap[1].size == K && s2_heap[1].sum >= ntasks;
    can_bf = s2_heap[0].size == K && s2_heap[0].sum >= ntasks;
    __syncthreads();
    if (tid == 0 && (start_now || can_bf)) {  // hand-out: tasks in pop order
      Heap2& h = s2_heap[start_now ? 1 : 0];
      int32_t rest = (int32_t)ntasks - (int32_t)K;
      uint32_t k = 0;
      while (h.size) {
        const int32_t cap_n = (int32_t)h.nt[0] - 1;
        const int32_t n = (rest < cap_n ? rest : cap_n) + 1;
        s2_g_node[k] = h.q[0];
        s2_g_n[k] = (uint16_t)n;
        rest -= n - 1;
        ++k;
        heap_pop2(h);
      }
    }
    __syncthreads();
    nodes = s2_g_node;
  } else {
    start_now = nsel == K;
    can_bf = ntot >= K;
    nodes = start_now ? sm.list : list2;
  }
  // the allocation of node k out of `src`
  auto alloc_from = [&](uint32_t k, const Row& src, Row& alloc) {
    if constexpr (kGeneral) {
      View full;
      view_node_plus_tasks(full, req_node, req_task, s2_g_n[k]);
      feasible_alloc(full, src, alloc, s2_cx.dslot);
    } else {
      feasible_alloc(req, src, alloc, s2_cx.dslot);
    }
  };
  int64_t T0 = now;
  bool placed = start_now;
  if (!start_now && can_bf) {
    // earliest common start of the K nodes, allocation against res_total (JobScheduler.cpp:5371-5404,
    // JobScheduler.h:806-849): T <- max over the nodes of their earliest fit >= T, to the fixed point
    bool found = false, failed = false;
    for (uint32_t it = 0; !found && !failed; ++it) {
      long long emax = INT64_MIN, emin = kInf;
      for (uint32_t k0 = 0; k0 < K; k0 += kNG) {
        const uint32_t k = k0 + gi;
        const bool act = k < K;
        uint32_t q = 0, g = 0, ns = 0;
        Row alloc;
        row_zero(alloc);
        if (act) {
          q = nodes[k];
          g = base + q;
          ns = sm.nseg[q];
          const Row tot = node_total2(q);
          if (exclusive) alloc = tot; else alloc_from(k, tot, alloc);
        }
        const int64_t e = g_earliest(tl.ent + (size_t)g * tl.cap, ns, alloc, T0, limit, act);
        if (act) { emax = e > emax ? e : emax; emin = e < emin ? e : emin; }
      }
      if (gl == 0) { s2_e[it & 1u][gi] = emax; s2_e2[it & 1u][gi] = emin; }
      __syncthreads();
      long long hi = INT64_MIN, lo = kInf;
      const uint32_t ng = K < (uint32_t)kNG ? K : (uint32_t)kNG;
      for (uint32_t i = 0; i < ng; ++i) {
        const long long x = s2_e[it & 1u][i], y = s2_e2[it & 1u][i];
        hi = x > hi ? x : hi;
        lo = y < lo ? y : lo;
      }
      if (hi == kInf) failed = true;
      else if (lo == hi) { found = true; T0 = hi; }  // every node fits from exactly this time on
      else T0 = hi;
    }
    placed = found && T0 - now <= s2_cx.max_window;  // JobScheduler.h:809
  }
  if (placed) {
    // ---- the K nodes from T0 on: allocation, timeline update, outputs
    for (uint32_t k0 = 0; k0 < K; k0 += kNG) {
      const uint32_t k = k0 + gi;
      const bool act = k < K;
      const uint32_t q = act ? nodes[k] : 0u, g = base + q, ns = act ? sm.nseg[q] : 0u;
      TlEntry* E = tl.ent + (size_t)g * tl.cap;
      Row alloc;
      row_zero(alloc);
      if (!kGeneral && start_now) {
        g_exact<true>(jq, q, act, &alloc);  // out of the window (the node passed this test in the walk)
      } else {
        Row tot;
        row_zero(tot);
        if (act) tot = node_total2(q);
        Row src = tot;
        if (kGeneral && start_now) {  // out of the window minimum
          Win2 w;
          g_window<true>(E, ns, w_end, req.cpu_raw, req.mem, false, true, tot, act && !exclusive, w);
          if (act && !exclusive) win_row_min(w, tl.avail0[g], req, src);
        }
        if (act) { if (exclusive) alloc = tot; else alloc_from(k, src, alloc); }
      }
      Row seg0;
      row_zero(seg0);
      const uint32_t nn = g_update(E, ns, T0, T0 + limit, alloc, act, seg0);
      const uint32_t rank = g_out_rank(K, q, act, [&](uint32_t m) { return (uint32_t)nodes[m]; });
      if (act && gl == 0) {
        write_node2(jq, q, rank, alloc, nn, seg0);
        if (kGeneral) s2_cx.out.alloc_ntasks[jq.alloc_off + rank] = s2_g_n[k];
        // pending-reason label for future starts (JobScheduler.cpp:5842-5848)
        if (T0 != now) atomicOr(&s2_label, later_label2(q, !row_le(alloc, tl.avail0[g]), limit));
      }
    }
  }
  __syncthreads();
  const bool full_rekey = K > (uint32_t)kRK;
  if (placed) {
    if (tid == 0) write_job2(jq, T0, s2_label);
    // the node's cost grows by its allocation's cpu share (JobScheduler.h:46-52)
    for (uint32_t k = tid; k < K; k += kT2) {
      const uint32_t q = nodes[k];
      const int64_t tot_cpu = node_total_cpu2(q);
      const int64_t cpu = exclusive ? tot_cpu : kGeneral ? req_node.cpu_raw + req_task.cpu_raw * (int64_t)s2_g_n[k] : req.cpu_raw;
      const double nc = __dadd_rn(sm.cost[q], cost_step(s2_cx.cost_policy, limit, cpu, tot_cpu));
      if (full_rekey) sm.cost[q] = nc; else { s2_rk_node[k] = q; s2_rk_nc[k] = nc; }
    }
  } else if (tid == 0) {
    s2_cx.out.reason[jq.job] = CRANE_REASON_RESOURCE;  // JobScheduler.cpp:5802
  }
  if (!kGeneral) {  // list2 lives in the scratch words: back to zero
    __syncthreads();
    for (uint32_t i = tid; i < (K + 1) / 2 + 1 && i < s2_cx.mp + 4; i += kT2) sm.scratch[i] = 0;
  }
  __syncthreads();
  if (placed) {
    if (full_rekey) order_sort2();
    else {
      order_rekey2(K, kT2);
      __syncthreads();
      rekey_bounds2(K);
    }
  }
}

__global__ void __launch_bounds__(kT2, 1) k_commit2(Commit2Args a) {
  const uint32_t part = a.part_list ? a.part_list[blockIdx.x] : blockIdx.x;
  const uint32_t base = a.cl.part_base[part];
  const uint32_t mp = a.cl.part_base[part + 1] - base;
  const uint32_t words = a.words_per_row;
  const uint32_t ring = a.ring;
  const uint32_t tid = threadIdx.x, lane = lane_id(), wid = warp_id();
  const uint32_t gl = g_lane(), gi = g_index();

  const Smem2 sm = smem2_layout(mp, words, ring, a.gres != 0);

  // ---- load node state -------------------------------------------------------
  for (uint32_t q = tid; q < mp; q += kT2) {
    const uint32_t g = base + q;
    sm.cost[q] = a.tl.cost0[g];
    const Row s0 = a.tl.ent[(size_t)g * a.tl.cap].seg;
    sm.cpu0[q] = s0.cpu_raw;
    if (sm.gcnt) sm.gcnt[q] = pack_gres_counts(s0);
    sm.skip[q] = a.tl.skip[g];
    sm.nseg[q] = (uint16_t)a.tl.n[g];
    sm.cls[q] = a.cl.slot_class[g];
  }
  const uint32_t ncp = a.sched_nparts ? a.sched_nparts[part] : 1u;
  for (uint32_t p = tid; p < mp + 4; p += kT2) sm.scratch[p] = 0;
  if (tid < kMaxClasses) s2_classrow[tid] = a.cl.class_rows[(size_t)part * kMaxClasses + tid];
  if (tid == 0) {
    s2_cx.cl = a.cl; s2_cx.tl = a.tl; s2_cx.out = a.out;
    s2_cx.now = a.now; s2_cx.max_window = a.max_window; s2_cx.base = base; s2_cx.mp = mp; s2_cx.words = words;
    s2_cx.ncp = ncp; s2_cx.npos = mp; s2_curp = 0;
    s2_cx.max_jobs = a.max_jobs; s2_cx.ring = ring; s2_cx.gres = a.gres; s2_cx.dslot = a.dslot; s2_cx.cost_policy = a.cost_policy; s2_cx.part = part; s2_cx.req_node = a.req_node; s2_cx.req_task = a.req_task;
    s2_prof_windows = 0; s2_prof_tests = 0; s2_prof_singles = 0;
    for (uint32_t s = 0; s < ring; ++s) mbar_init(&s2_bar[s], 1);
    fence_mbar_init();
  }
  __syncthreads();
  if (ncp > 1) init_orders2(a.slot_memb); else order_sort2();

  const uint32_t r_begin = a.part_job_off[part], r_end = a.part_job_off[part + 1];
  const uint32_t njobs = r_end - r_begin;
  const uint32_t row_bytes = words * 4;
  const int64_t now = a.now;
  uint32_t issued = 0;
  PROF_DECL;

  // job records and capability-bitmap rows arrive through a shared-memory ring
  // filled by TMA bulk copies (cp.async.bulk + mbarrier); the slot of job i is
  // free once job i - ring is finished. Called by all threads after a CTA barrier.
  auto ensure_issued = [&](uint32_t finished) {
    const uint32_t hi = njobs < finished + ring ? njobs : finished + ring;
    if (wid == 0) {
      for (uint32_t i = issued + lane; i < hi; i += 32) {
        const uint32_t slot = i % ring;
        mbar_expect_tx(&s2_bar[slot], (uint32_t)sizeof(JobQ) + row_bytes);
        tma_load_1d(&s2_jobs[slot], &a.jobq[r_begin + i], (uint32_t)sizeof(JobQ), &s2_bar[slot]);
        tma_load_1d(sm.bits_ring + (size_t)slot * words, a.bitmap + (size_t)(r_begin + i) * words, row_bytes, &s2_bar[slot]);
      }
    }
    if (issued < hi) issued = hi;
  };

  // =============================== dispatcher =====================================
  uint32_t ji = 0;
  uint32_t jcap = kMaxJ;     // jobs offered to the next batch: twice what the last one placed (a batch that is cut
                             // early wastes the selection of the jobs behind the cut)
  uint32_t vcredit = 0;      // batches for which complete candidate lists are validated before the resolve (validate2)
  bool want_single = s2_cx.ncp > 1;  // the job at ji goes down the one-job path (overlapping partitions: every job,
                                     // each in its own partition's order)
  while (ji < njobs) {
    ensure_issued(ji);
    PROF(0);
    if (want_single) {
      if (wid == 0 && lane == 0) mbar_wait(&s2_bar[ji % ring], (ji / ring) & 1u);
      __syncthreads();
      if (jq_general(s2_jobs[ji % ring])) single2<true>(ji); else single2<false>(ji);
      PROF(7);
      ++ji;
      want_single = s2_cx.ncp > 1;
      __syncthreads();
      continue;
    }
    // ---- form the batch: warp 0, lane = job -------------------------------------
    if (wid == 0) {
      uint32_t myK = 0, myslot = 0;
      bool okj = false;
      const uint32_t j = ji + lane;
      if (lane < jcap && j < njobs) {
        myslot = j % ring;
        mbar_wait(&s2_bar[myslot], (j / ring) & 1u);
        myK = s2_jobs[myslot].node_num;
        okj = myK >= 1 && myK <= mp && myK <= (uint32_t)kMaxT && !jq_general(s2_jobs[myslot]);
      }
      uint32_t cum = okj ? myK : (uint32_t)kMaxT + 1u;
      for (int o = 1; o < 32; o <<= 1) {
        const uint32_t up = __shfl_up_sync(kFullMask, cum, o);
        if ((int)lane >= o) cum = cum + up > 0xffffu ? 0xffffu : cum + up;
      }
      const unsigned good = __ballot_sync(kFullMask, okj && cum <= (uint32_t)kMaxT);
      const uint32_t nj = good == kFullMask ? 32u : (uint32_t)__ffs((int)~good) - 1u;
      if (lane < nj) {
        BJob2 b;
        b.slot = myslot; b.K = myK; b.need = cum; b.tfirst = cum - myK; b.n0 = 0; b.n1 = 0; b.mode = 0; b.state = 0;
        s2_bj[lane] = b;
      }
      if (lane == 0) { s2_nj = nj; s2_njr = nj; s2_nbf = 0; }
    }
    __syncthreads();
    const uint32_t nj = s2_nj;
    if (nj == 0) { want_single = true; continue; }
    PROF(1);

    // ---- select: group t lists the candidates of job t -------------------------
    const bool jact = gi < nj;
    BJob2 bj;
    bj.slot = 0; bj.K = 0; bj.need = 0; bj.tfirst = 0; bj.n0 = 0; bj.n1 = 0; bj.mode = 0; bj.state = 0;
    {
      JSel2 js;
      js.bits = nullptr; js.req_cpu = 0; js.spec8 = 0; js.name_need = nullptr; js.gnames = 0; js.exclusive = false; js.has_gres = false;
      if (jact) {
        bj = s2_bj[gi];
        jsel_load(s2_jobs[bj.slot], sm.bits_ring + (size_t)bj.slot * words, js);
      }
      uint32_t n0, n1;
      // (while lists are validated, a job lists spare candidates: the ones that fail are replaced inside the batch)
      const uint32_t want = vcredit ? (bj.need + (uint32_t)kSpare < (uint32_t)kMaxT ? bj.need + (uint32_t)kSpare : (uint32_t)kMaxT) : bj.need;
      select2(sm, mp, js, jact ? want : 0u, jact, s2_cl[0][gi], s2_cl[1][gi], n0, n1);
      bj.n0 = n0; bj.n1 = n1;
      // fewer than K pre-filter candidates: only a backfill is possible (taken
      // nodes lose resources, they never gain candidates); fewer than K capable
      // nodes: "Resource" whatever the jobs before it do
      bj.mode = n0 < bj.K ? 1u : 0u;
      bj.state = (bj.mode && n1 < bj.K) ? 2u : 0u;
      if (jact) {
        // cost a node of class c gets when this job is placed on it (JobScheduler.h:46-52)
        const JobQ& jq = s2_jobs[bj.slot];
        for (uint32_t c = gl; c < (uint32_t)kDeltaClasses; c += kGL) {
          const int64_t tot_cpu = s2_classrow[c].cpu_raw;
          s2_jdelta[gi][c] = tot_cpu > 0 ? cost_step(a.cost_policy, jq.time_limit, js.exclusive ? tot_cpu : jq.req.cpu_raw, tot_cpu) : 0.0;
        }
        for (uint32_t w = bj.tfirst + gl; w < bj.need; w += kGL) s2_tjob[w] = gi;
        if (gl == 0) {
          s2_bj[gi].n0 = bj.n0; s2_bj[gi].n1 = bj.n1; s2_bj[gi].mode = bj.mode; s2_bj[gi].state = bj.state;
          const uint32_t nl = bj.state ? 0u : (bj.mode ? bj.n1 : bj.n0);
          s2_jw[gi] = bj.K | bj.tfirst << 8 | bj.mode << 16 | bj.state << 17 | nl << 24;
          s2_joblabel[gi] = 0;
          s2_T0[gi] = now;
          s2_jst[gi] = (bj.state == 0 && bj.mode == 1u && bj.K > 1u) ? 0u : 3u;
        }
      }
    }
    __syncthreads();
    if (vcredit) {  // a pick failed the exact test a few batches ago: complete lists are validated up front
      validate2(nj);
      --vcredit;
    }
    PROF(2);

    // ---- resolve (warp 0)  ||  speculative evaluation (warps 1-7) ---------------------
    // Task slot w is worked by group 31 - w in every phase. While warp 0 resolves,
    // the other warps already run the exact test of each slot's first guess: the
    // entry the job takes if the jobs before it take the entries before (no state
    // is touched). After the resolve the slots whose guess was wrong — and those of
    // warp 0's groups — are tested again.
    const uint32_t myslot = (uint32_t)kNG - 1u - gi;
    const uint32_t nslots = s2_bj[nj - 1].need;
    uint32_t ev_q = 0xffffu;      // node the results below belong to
    bool tok = false;
    Row talloc;                   // the allocation: out of the window minimum (immediate start, JobScheduler.cpp:5340-5361)
    row_zero(talloc);             // or against res_total (backfill, :5381-5403)
    bool tshort = false;          // backfill label: the allocation does not fit res_avail now (JobScheduler.cpp:5842-5848)
    int64_t te0 = kInf;           // backfill: earliest fit >= now
    // the job my slot belongs to (fixed when the batch was formed)
    uint32_t tjob = 0, tmode = 0, tK = 1, tfirst = 0, tstate = 2;
    const JobQ* tjq = &s2_jobs[0];
    if (myslot < nslots) {
      tjob = s2_tjob[myslot];
      // (s2_bj[].state is rewritten by the resolve below: everything here comes from
      // words nobody writes during this phase)
      const uint32_t jw = s2_jw[tjob];
      tjq = &s2_jobs[s2_bj[tjob].slot];
      tK = jw & 0xffu; tfirst = (jw >> 8) & 0xffu; tmode = (jw >> 16) & 1u; tstate = (jw >> 17) & 3u;
    }
    const bool texcl = jq_exclusive(*tjq);
    const int64_t tlimit = tjq->time_limit;
    uint32_t njr = nj, NT = 0;
    bool tact = false;
    uint32_t tq = 0xffffu;
    for (uint32_t pass = 0; pass < 2; ++pass) {
      bool do_eval = false;
      uint32_t q = 0xffffu;
      if (pass == 0) {
        if (wid == 0) {
          // in job order every job takes its first K free candidates. Lane = list
          // entry while a job picks, lane = task slot for the tasks made so far
          // (node, new cost). A taken node is marked in its scratch word. The batch
          // ends before a job whose candidates were taken by the jobs before it, or
          // for which a taken node, at its NEW key, sorts before the job's last pick
          // while it still is a candidate: that node would be among the first K of
          // the updated order, so the job has to see the node's update first. "Still a
          // candidate" is judged on the node's first segment after the earlier job: the
          // timeline starts at `now`, so a job that starts now takes its cpu out of that
          // segment, and a node it filled is no clash.
          uint32_t tv = 0xffffu, tslot = 0xffffffffu;  // my task slot: node (0xffff = void), job
          int64_t tcpu = 0;                            // cpu of my node's first segment after my slot's job
          double tnc = 0.0;
          uint32_t njr_l = nj;
          uint32_t nw = s2_jw[0];
          uint32_t nq = lane < (nw >> 24) ? (uint32_t)s2_cl[(nw >> 16) & 1u][0][lane] : 0xffffu;
          double ncq = nq != 0xffffu ? sm.cost[nq] : 0.0;
          for (uint32_t t = 0; t < nj; ++t) {
            const uint32_t jw = nw, lq = nq;
            const double cq = ncq;
            if (t + 1 < nj) {  // the next job's list is on its way while this one is decided
              nw = s2_jw[t + 1];
              nq = lane < (nw >> 24) ? (uint32_t)s2_cl[(nw >> 16) & 1u][t + 1][lane] : 0xffffu;
              ncq = nq != 0xffffu ? sm.cost[nq] : 0.0;
            }
            const uint32_t K = jw & 0xffu, tf = (jw >> 8) & 0xffu, mode = (jw >> 16) & 1u, state = (jw >> 17) & 3u;
            const bool mine = lane >= tf && lane < tf + K;  // my slot belongs to this job
            if (mine) tslot = t;
            if (state != 0) continue;                       // fewer than K capable nodes: no tasks, "Resource"
            const bool fr = lq != 0xffffu && sm.scratch[lq] == 0;
            const unsigned m = __ballot_sync(kFullMask, fr);
            const uint32_t kth = K == 1 ? (m ? (uint32_t)__ffs((int)m) - 1u : 32u) : nth_set_bit(m, K);
            if (kth >= 32u) {
              if (lane == 0) s2_bj[t].state = 1;
              njr_l = t;
              break;
            }
            const uint32_t cm = m & (kth >= 31u ? 0xffffffffu : ((2u << kth) - 1u));
            const uint32_t q_last = __shfl_sync(kFullMask, lq, (int)kth);
            const double c_last = __shfl_sync(kFullMask, cq, (int)kth);
            unsigned cl = __ballot_sync(kFullMask, tv != 0xffffu && key_lt(tnc, tv, c_last, q_last));
            if (cl) {  // rare: is that node still a candidate of this job?
              JSel2 jt;
              const uint32_t slot = s2_bj[t].slot;
              jsel_load(s2_jobs[slot], sm.bits_ring + (size_t)slot * words, jt);
              const bool rel = ((cl >> lane) & 1u) && capable2(sm, jt, tv) && (mode || prefilter_cpu2(sm, jt, tv, tcpu));
              cl = __ballot_sync(kFullMask, rel);
            }
            if (cl) {
              if (lane == 0) s2_bj[t].state = 3;
              njr_l = t;
              break;
            }
            double nc = 0.0;
            if ((cm >> lane) & 1u) {
              sm.scratch[lq] = 1;
              const uint8_t c = sm.cls[lq];
              nc = c < kDeltaClasses ? __dadd_rn(cq, s2_jdelta[t][c]) : new_cost2(s2_jobs[s2_bj[t].slot], lq, sm.cost);
            }
            // pick number i of the job goes to task slot tf + i
            const uint32_t src = mine ? (K == 1 ? kth : nth_set_bit(cm, lane - tf + 1u)) : 0u;
            const uint32_t pq = __shfl_sync(kFullMask, lq, (int)(src & 31u));
            const double pnc = __shfl_sync(kFullMask, nc, (int)(src & 31u));
            if (mine) {
              tv = pq; tnc = pnc;
              tcpu = sm.cpu0[pq];
              if (!mode) {  // starts now (exclusive: takes res_total)
                const JobQ& jq = s2_jobs[s2_bj[t].slot];
                tcpu -= jq_exclusive(jq) ? node_total_cpu2(pq) : jq.req.cpu_raw;
              }
            }
            __syncwarp();
          }
          const uint32_t NTl = njr_l ? ((s2_jw[njr_l - 1] >> 8) & 0xffu) + (s2_jw[njr_l - 1] & 0xffu) : 0u;
          if (lane < NTl) {
            BTask2 t;
            t.q = tv; t.job = tv != 0xffffu ? tslot : 0xffffffffu; t.nc = tnc;
            s2_task[lane] = t;
          }
          __syncwarp();
          if (tv != 0xffffu) sm.scratch[tv] = 0;  // the marks go back to zero
          if (lane == 0) { s2_njr = njr_l; s2_cut = NTl; }
        } else if (myslot < nslots && tstate == 0) {
          // first guess of my slot: entry `myslot` of the job's list if the list is
          // long enough for all the jobs before it to be served, else its own i-th entry
          const uint32_t jw = s2_jw[tjob];
          const uint32_t nl = jw >> 24;
          const uint32_t gidx = nl >= tfirst + tK ? myslot : myslot - tfirst;
          if (gidx < nl) { q = s2_cl[tmode][tjob][gidx]; do_eval = true; }
        }
      } else {
        njr = s2_njr;
        NT = njr ? s2_bj[njr - 1].need : 0u;
        tact = myslot < NT && s2_task[myslot].job < njr;
        if (tact) tq = s2_task[myslot].q;
        do_eval = tact && ev_q != tq;
        q = tq;
      }
      // ---- the exact test of node q for my slot's job, no state touched -------------
      {
        const uint32_t g = base + (do_eval ? q : 0u);
        const uint32_t ns = do_eval ? sm.nseg[q] : 0u;
        const TlEntry* E = a.tl.ent + (size_t)g * a.tl.cap;
        Row ea0, etot;
        row_zero(ea0);
        row_zero(etot);
        if (do_eval) {
          ev_q = q;
          ea0 = a.tl.avail0[g];
          if (texcl || tmode) etot = node_total2(q);
        }
        Win2 w;
        g_window(E, ns, now + tlimit, tjq->req.cpu_raw, tjq->req.mem, texcl, jq_has_gres(*tjq), etot, do_eval && !tmode, w);
        if (do_eval && !tmode) {
          tok = w.ok;
          if (texcl) talloc = etot;
          else if (tok) {
            tok = ea0.cpu_raw >= tjq->req.cpu_raw && ea0.mem >= tjq->req.mem;  // res_avail itself (JobScheduler.cpp:5310)
            if (tok) {
              Row wr;
              win_row(w, ea0, tjq->req, wr);
              tok = feasible<true>(tjq->req, wr, C_DICT2, &talloc);
            }
          }
        } else if (do_eval) {
          if (texcl) talloc = etot; else feasible<true>(tjq->req, etot, C_DICT2, &talloc);
          tshort = !row_le(talloc, ea0);
        }
        const int64_t e = g_earliest(E, ns, talloc, now, tlimit, do_eval && tmode);
        if (do_eval && tmode) te0 = e;
      }
      __syncthreads();
      if (pass == 0) PROF(3);
    }
    if (njr < nj) PROF_CNT(s2_bj[njr].state == 1u ? 9 : 10, 1);
    if (njr == 0) { want_single = true; continue; }  // (nothing is taken before the first job: cannot happen)

    // earliest start of the backfill jobs (JobScheduler.h:806-849): a one-node job
    // is decided by its node's earliest fit; the nodes of a wider job iterate
    // T <- max over nodes of the earliest fit >= T to the fixed point
    TlEntry* const tE = a.tl.ent + (size_t)(base + (tact ? tq : 0u)) * a.tl.cap;
    const uint32_t tns = tact ? sm.nseg[tq] : 0u;
    if (tact && tmode) {
      if (tK == 1) {
        tok = te0 != kInf && te0 - now <= a.max_window;  // JobScheduler.h:809
        if (gl == 0) s2_T0[tjob] = te0;
      } else if (gl == 0) {
        s2_e[0][myslot] = te0;
        atomicAdd(&s2_nbf, 1u);
      }
    }
    __syncthreads();
    if (s2_nbf) {
      for (uint32_t it = 0;; ++it) {
        bool still = false;
        if (tid < njr && s2_jst[tid] == 0u) {
          const BJob2 b = s2_bj[tid];
          long long tmax = INT64_MIN, tmin = kInf;
          for (uint32_t w = b.tfirst; w < b.need; ++w) {
            const long long x = s2_e[it & 1u][w];
            tmax = x > tmax ? x : tmax;
            tmin = x < tmin ? x : tmin;
          }
          if (tmax == kInf) s2_jst[tid] = 2u;
          else if (tmin == tmax) { s2_T0[tid] = tmax; s2_jst[tid] = (tmax - now <= a.max_window) ? 1u : 2u; }
          else { s2_T0[tid] = tmax; still = true; }
        }
        if (!__syncthreads_or(still ? 1 : 0)) break;
        const bool bact = tact && tmode && tK > 1 && s2_jst[tjob] == 0u;
        const int64_t e = g_earliest(tE, tns, talloc, bact ? (int64_t)s2_T0[tjob] : now, tlimit, bact);
        if (bact && gl == 0) s2_e[(it + 1) & 1u][myslot] = e;
        __syncthreads();
      }
      if (tact && tmode && tK > 1) tok = s2_jst[tjob] == 1u;
    }
    if (tact && gl == 0 && !tok) atomicMin(&s2_cut, tfirst);  // a job is placed only if all its nodes pass
    __syncthreads();
    const uint32_t cut = s2_cut;
    PROF(4);

    // ---- commit the jobs before the cut (warps 4-7)  ||  re-key their nodes (warps 0-3) ----
    // With at most 16 tasks the committing groups (31 - w) all sit in warps 4-7,
    // and the order can be re-keyed by the other half of the CTA at the same time:
    // the new costs are known since the resolve, and the re-key only reads what
    // the commit does not write.
    const bool overlap = NT <= (uint32_t)kNG / 2;
    uint32_t cnt = 0;
    {
      // placed nodes and their new costs (every thread computes the same list position)
      const unsigned pm = __ballot_sync(kFullMask, lane < cut && s2_task[lane].job < njr);
      cnt = (uint32_t)__popc(pm);
      if (wid == 0 && ((pm >> lane) & 1u)) {
        const uint32_t i = (uint32_t)__popc(pm & ((1u << lane) - 1u));
        s2_rk_node[i] = s2_task[lane].q;
        s2_rk_nc[i] = s2_task[lane].nc;
      }
    }
    if (!overlap) __syncthreads();
    if (!overlap || wid >= 4) {
      const bool cact = tact && myslot < cut;
      int64_t start = now;
      if (cact && tmode) start = s2_T0[tjob];
      Row seg0;
      row_zero(seg0);
      const uint32_t nn = g_update(tE, tns, start, start + tlimit, talloc, cact, seg0);
      const uint32_t rank = g_out_rank(tK, tq, cact, [&](uint32_t m) { return s2_task[tfirst + m].q; });
      if (cact && gl == 0) {
        write_node2(*tjq, tq, rank, talloc, nn, seg0);
        if (start != now) atomicOr(&s2_joblabel[tjob], later_label2(tq, tshort, tlimit));
      }
    }
    if (overlap) {
      if (wid < 4) order_rekey2(cnt, kT2 / 2);
    } else {
      __syncthreads();
      order_rekey2(cnt, kT2);
    }
    __syncthreads();
    PROF(5);
    // job-level outputs. The job at the cut: a failed backfill is final — the
    // reference takes exactly these nodes (the first K capable ones) and gives up
    // when they have no common start inside the window (JobScheduler.cpp:5371-5404,
    // 5802) — a failed immediate start continues its walk on the one-job path.
    const uint32_t fjob = cut < NT ? s2_tjob[cut] : 0xffffffffu;
    uint32_t done = cut < NT ? fjob : njr;
    if (tid < done) {
      const BJob2 b = s2_bj[tid];
      const JobQ& jq = s2_jobs[b.slot];
      if (b.state == 2u) a.out.reason[jq.job] = CRANE_REASON_RESOURCE;
      else write_job2(jq, b.mode ? (int64_t)s2_T0[tid] : now, s2_joblabel[tid]);
    }
    if (fjob != 0xffffffffu) {
      const BJob2 b = s2_bj[fjob];
      if (b.mode == 1u) {
        if (tid == 0) a.out.reason[s2_jobs[b.slot].job] = CRANE_REASON_RESOURCE;
        ++done;
        PROF_CNT(12, 1);
      } else {
        want_single = true;
        vcredit = kValidateFor;
        PROF_CNT(11, 1);
      }
    }
    rekey_bounds2(cnt);
    __syncthreads();
    PROF(6);
    PROF_CNT(13, done);
    PROF_CNT(14, 1);
    ji += done;
    jcap = 2u * done + 4u < (uint32_t)kMaxJ ? 2u * done + 4u : (uint32_t)kMaxJ;
  }
  PROF_CNT(8, s2_prof_windows);
  PROF_CNT(15, s2_prof_tests);
  PROF_CNT(9, 0);
#ifdef CRANE_PROFILE
  if (threadIdx.x == 0) prof_acc[12] = prof_acc[12] | (s2_prof_singles << 32);
#endif
  PROF_FLUSH(a.prof);
}

}  // namespace crane
