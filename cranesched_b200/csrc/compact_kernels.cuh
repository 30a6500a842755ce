// compact_kernels.cuh — sm_90a kernels of crane_sched_compact.
//
// The resident pending and running tables keep a row's index until the table is
// replaced, so erased rows stay behind as tombstones and resolved dependency entries
// stay behind retired. Compaction rewrites the tables with only their live rows and
// open entries, on the device, where the gate state lives:
//   live rows   k_rt_live_keys + the stable LSD radix sort (the regroup's): the live rows
//               first, in row order; k_cp_map scatters their ranks into the old -> new map
//   columns     one gather per table (k_cp_cols, the regroup's too): new row c = c-th live row
//   CSR tables  lengths of the live rows, their exclusive scan (k_sort_scan) and one warp
//               per row copying its entries (k_cp_csr)
//   entries     k_cp_ent_keys flags the open entries of live rows, the same sort lists them
//               in entry order, k_cp_entries copies them with dependent and dependee mapped
// Live rows and kept entries keep their order, so every order-sensitive step of a run
// (the stable priority sort, FIFO, the regroup's sorts and fp64 sums, account grouping)
// sees the same sequence as on the uncompacted tables.
// crane_sched_steps_compact rewrites the resident step tables with the same gathers (the
// host lists their live rows, since it holds every flag that decides liveness) and
// k_cp_spans for the allocation pool.
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

// One fixed-width column of a gather: new row c takes old row live ? live[c] : c, for the
// new rows c < rows
struct ColCopy {
  const void* src;
  void* dst;
  uint32_t bytes;  // of an element
  uint32_t rows;
};

// The columns of one table (the pending table's 18 with the gate's 5 at most)
constexpr int kMaxCols = 24;
struct ColSet {
  uint32_t n;
  ColCopy col[kMaxCols];
};

template <class W>
__device__ __forceinline__ void cp_elem(const ColCopy& d, uint32_t r, uint32_t c) {
  const uint32_t w = d.bytes / sizeof(W);
  const W* s = static_cast<const W*>(d.src) + (size_t)r * w;
  W* t = static_cast<W*>(d.dst) + (size_t)c * w;
  for (uint32_t k = 0; k < w; ++k) t[k] = s[k];
}

// Thread per new row, every column of the set in turn; elements go in 8-byte words when
// their size allows (Row and View are 8-byte aligned)
__global__ void k_cp_cols(ColSet s, const uint32_t* live, uint32_t n_live) {
  const uint32_t c = blockIdx.x * blockDim.x + threadIdx.x;
  if (c >= n_live) return;
  const uint32_t r = live ? live[c] : c;
  for (uint32_t k = 0; k < s.n; ++k) {
    const ColCopy& d = s.col[k];
    if (c >= d.rows) continue;
    if (d.bytes % 8 == 0) cp_elem<uint64_t>(d, r, c);
    else if (d.bytes % 4 == 0) cp_elem<uint32_t>(d, r, c);
    else cp_elem<uint8_t>(d, r, c);
  }
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

// crane_sched_steps_compact: one warp per kept scheduled step (old row rows[c], new row
// new_rows[c]); its node_num node rows of the allocation pool move from alloc_at[old] to
// new_at[c], and lane 0 points the new alloc_at there. A step's span is not a CSR row (the
// spans lie in the order the passes scheduled them, not in row order), hence not k_cp_csr.
__global__ void k_cp_spans(const uint32_t* alloc_at, const uint32_t* node_num, const uint32_t* sa_node,
                           const Row* sa_res, const uint32_t* rows, const uint32_t* new_rows, const uint32_t* new_at,
                           uint32_t n, uint32_t* new_alloc_at, uint32_t* new_sa_node, Row* new_sa_res) {
  const int lane = lane_id();
  const uint32_t warps = blockDim.x >> 5;
  for (uint32_t c = blockIdx.x * warps + warp_id(); c < n; c += gridDim.x * warps) {
    const uint32_t r = rows[c], s0 = alloc_at[r], cnt = node_num[r], d0 = new_at[c];
    for (uint32_t k = lane; k < cnt; k += 32) {
      new_sa_node[d0 + k] = sa_node[s0 + k];
      new_sa_res[d0 + k] = sa_res[s0 + k];
    }
    if (lane == 0) new_alloc_at[new_rows[c]] = d0;
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
// event row matches); a null map is the identity.
__global__ void k_cp_entries(GateDev s, GateDev d, const uint32_t* keep, uint32_t n_keep,
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
  d.delay[c] = s.delay[e];
}

}  // namespace crane
