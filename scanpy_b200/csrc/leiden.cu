// leiden.cu — Leiden community detection on a symmetric weighted CSR graph (sm_90a).
//
// Replaces leidenalg.find_partition(RBConfigurationVertexPartition) / igraph community_leiden as
// called by the reference at src/scanpy/tools/_leiden.py:184-187,195-196 (and eliminates the Python
// tuple-list graph build of src/scanpy/_utils/__init__.py:278-306: the CSR is consumed directly).
// Objective (SURVEY.md Appendix A3):  Q = 1/(2m) sum_c [ sum_{i,j in c} A_ij - gamma K_c^2 / (2m) ].
//
// One Leiden pass = repeat { local moving -> refinement -> aggregation } until nothing merges:
//   decide_kernel<false>  warp per vertex: weights towards neighbouring communities are summed in
//                         registers (degree <= 32: one neighbour per lane, 32-step shuffle reduce
//                         by community id) or in the vertex's own slice of a global hash scratch
//                         (hubs, aggregated levels); best gain  w(v,c) - gamma k_v K_c / 2m.
//   lm_apply_kernel       applies the decided moves, updates K_c with integer atomics, re-activates
//                         the neighbours of moved vertices.
//   decide_kernel<true>   refinement: singleton vertices merge into refined communities inside their
//                         parent community; singleton->singleton merges only towards a smaller id
//                         whose owner stays put, so refined communities stay connected.
//   agg_* kernels         refined communities become super-vertices: per-super-vertex open-addressing
//                         hash slices (capacity = sum of member degrees) accumulate the edge weights.
// Determinism: moves are decided against a snapshot and applied in a separate kernel; every
// accumulated quantity (edge weights, strengths K_c) is a fixed-point int64, so atomic order
// cannot change any sum; ties break towards the smaller community id.  Same seed => same labels.
// Fixed point: one unit is 2^-e of the input weight, e = 32 - ceil(log2(max arc weight)) (lower by one bit per doubling
// beyond 2^30 arcs), so the largest arc is <= 2^32 units and the total < 2^62.  The objective is invariant under a
// uniform weight scale and the scale is a power of two, so w and w * 2^k give bit-identical runs; UMAP connectivities
// (max weight 1) get e = 32.  NaN, infinite or negative weights are rejected (SB2_E_BADARG).
// HBM-bound integer/gather work; per local-move sweep ~ 12*E (idx + weight) + 4*E (community gather) B.
#include <math.h>
#include <string.h>

#include <algorithm>
#include <vector>

#include "common.cuh"

namespace {

typedef unsigned long long u64;

struct Level {
  int32_t n;
  const int64_t* indptr;
  const int32_t* indices;
  const int64_t* w;  // fixed-point arc weights
  int64_t* k;        // fixed-point strengths (incl. self loops)
};

__host__ __device__ __forceinline__ uint32_t mix32(uint32_t x) {
  x ^= x >> 16; x *= 0x7feb352dU; x ^= x >> 15; x *= 0x846ca68bU; x ^= x >> 16;
  return x;
}

// One read of the arc weights: scan[0] = bit pattern of the largest weight (non-negative floats order like their bits as
// int32), scan[1] = 1 if some weight is NaN, infinite or negative (-0.0 counts as 0).
__global__ void weight_scan_kernel(const float* __restrict__ w, int64_t n, int32_t* __restrict__ scan) {
  int32_t mx = 0, bad = 0;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) {
    const float x = w[i];
    if (!(x >= 0.0f) || isinf(x)) bad = 1;
    else mx = max(mx, __float_as_int(x));
  }
  mx = __reduce_max_sync(0xffffffffu, mx);
  bad = __reduce_or_sync(0xffffffffu, bad);
  if ((threadIdx.x & 31) == 0) {
    if (mx) atomicMax(&scan[0], mx);
    if (bad) atomicOr(&scan[1], 1);
  }
}
// ceil(log2(x)) of a positive finite float given by its bits (normal or subnormal)
__device__ __forceinline__ int ceil_log2_f32(int32_t bits) {
  const int32_t be = bits >> 23, man = bits & 0x7FFFFF;
  if (be == 0) return -149 + (32 - __clz(man - 1));   // subnormal: man * 2^-149
  return be - 127 + (man != 0);
}
// Fixed point with a per-graph power-of-two scale 2^e, e = 32 - ceil(log2(max w)) - extra_shift: the largest arc becomes
// at most 2^32 units, so a total of up to 2^30 arcs stays below 2^62 (extra_shift lowers e for more arcs).  A power of two
// keeps the conversion exact under power-of-two rescaling of the input: w * 2^k gives the same int64 weights.
__global__ void to_fixed_kernel(const float* __restrict__ w, int64_t n, const int32_t* __restrict__ scan, int extra_shift,
                                int64_t* __restrict__ out) {
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const int32_t mx = scan[0];
  const int e = (mx > 0 ? 32 - ceil_log2_f32(mx) : 32) - extra_shift;
  out[i] = llrint(scalbn((double)w[i], e));   // (a flagged graph is rejected before these values are used)
}
__global__ void strength_kernel(int32_t n, const int64_t* __restrict__ indptr, const int64_t* __restrict__ w,
                                int64_t* __restrict__ k, u64* __restrict__ total) {
  const int32_t v = blockIdx.x * blockDim.x + threadIdx.x;
  int64_t s = 0;
  if (v < n) {
    for (int64_t e = indptr[v]; e < indptr[v + 1]; ++e) s += w[e];
    k[v] = s;
  }
  // block reduce -> one atomic
  __shared__ int64_t red[8];
  const int64_t t = block_sum(s, red);
  if (threadIdx.x == 0) atomicAdd(total, (u64)t);
}
__global__ void comm_stats_kernel(int32_t n, const int32_t* __restrict__ comm, const int64_t* __restrict__ k,
                                  u64* __restrict__ K, int32_t* __restrict__ csize) {
  const int32_t v = blockIdx.x * blockDim.x + threadIdx.x;
  if (v >= n) return;
  atomicAdd(&K[comm[v]], (u64)k[v]);
  atomicAdd(&csize[comm[v]], 1);
}
__global__ void iota_kernel(int32_t* __restrict__ a, int64_t n) {
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) a[i] = (int32_t)i;
}

// ---------------------------------------------------------------------------------------------
// REFINE=false: local moving.  key(u) = comm[u];  stay gain uses K[a]-k_v.
// REFINE=true : refinement.    only singleton v (rsize[ref[v]]==1); neighbours restricted to the same
//               parent community; key(u) = ref[u]; stay gain = 0.
// target[v]: >=0 move to that community, -1 stay (and deactivate), -2 skipped this sweep (stay active)
template <bool REFINE>
__global__ void __launch_bounds__(256)
decide_kernel(Level L, const int32_t* __restrict__ wl, int32_t w_begin, int32_t w_end, const int32_t* __restrict__ comm,
              const int32_t* __restrict__ ref, const int64_t* __restrict__ K, const int32_t* __restrict__ csize,
              double gamma, double total, uint32_t seed, int sweep, int noskip, int32_t* __restrict__ hkeys,
              int64_t* __restrict__ hvals, int32_t* __restrict__ target, uint8_t* __restrict__ tsingle, int by_position, int cshift) {
  // wl[w_begin .. w_end): the vertices this launch decides (local moving: the active vertices; refinement: the vertices
  // that are still singletons of the refined partition), sorted by vertex id.  Decisions are taken against a snapshot.
  // by_position = 0: results go to target[v] / tsingle[v]; 1: to target[wi] / tsingle[wi] (the rank's slice of a
  // work-list sharded over ranks: the slices are all-gathered, then scattered by vertex id - see share_decisions)
  const int lane = threadIdx.x & 31;
  const int32_t wi = w_begin + blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  if (wi >= w_end) return;
  const int32_t v = wl[wi];
  const int32_t oi = by_position ? wi : v;   // where this vertex's decision is written
  if (!REFINE) {
    if (noskip == 0) {
      // the vertices are dealt into 2^cshift pseudo-random classes (re-dealt every 2^cshift sweeps); a sweep lets ONE class
      // decide, so a vertex always sees the moves of the other classes: 2 classes normally, 8 for small input graphs
      // (closer to the sequential algorithm's one-vertex-at-a-time semantics, where sweeps cost microseconds)
      const uint32_t cls = (mix32((uint32_t)v * 0x9E3779B9U + seed * 0x85EBCA6BU + (uint32_t)(sweep >> cshift)) + (uint32_t)sweep) & ((1u << cshift) - 1u);
      if (cls) { if (lane == 0) target[oi] = -2; return; }
    }
  } else {
    if (csize[ref[v]] != 1) { if (lane == 0) { target[oi] = -1; tsingle[oi] = 0; } return; }
  }
  const int64_t e0 = L.indptr[v], e1 = L.indptr[v + 1];
  const int deg = (int)(e1 - e0);
  const int32_t a = REFINE ? ref[v] : comm[v];
  const int32_t pv = comm[v];
  const double kv = (double)L.k[v];
  const double scale = gamma * kv / total;
  double best_gain = -1e300;
  int32_t best = -1;
  double wa = 0.0;  // weight towards own community (local moving only)
  // swap guard, applied while candidates are collected (so the next-best admissible community is still found):
  // a singleton may join another SINGLETON only towards the smaller id (local moving: community id, refinement:
  // vertex id == label of a singleton); everything else is admissible
  const bool v_single = REFINE ? true : csize[a] == 1;
  auto allowed = [&](int32_t c) -> bool { return !(v_single && csize[c] == 1 && c > (REFINE ? v : a)); };

  if (deg <= 32) {
    int32_t c = -1 - lane;  // unique negative = "no neighbour"
    int64_t w = 0;
    if (lane < deg) {
      const int32_t u = L.indices[e0 + lane];
      if (u != v && (!REFINE || comm[u] == pv)) {
        c = REFINE ? ref[u] : comm[u];
        w = L.w[e0 + lane];
      }
    }
    // lanes that look at the same community form a group (MATCH.ANY); the group's arc weights - non-negative
    // fixed point, <= 2^32 each - are summed exactly with three 24-bit-limb warp reductions (REDUX) instead
    // of 32 rounds of shuffles
    const unsigned grp = __match_any_sync(0xffffffffu, c);
    const bool leader = (__ffs(grp) - 1) == lane;
    const u64 uw = (u64)w;
    const unsigned s0 = __reduce_add_sync(grp, (unsigned)(uw & 0xFFFFFFull));
    const unsigned s1 = __reduce_add_sync(grp, (unsigned)((uw >> 24) & 0xFFFFFFull));
    const unsigned s2 = __reduce_add_sync(grp, (unsigned)(uw >> 48));
    const int64_t tot = (int64_t)((u64)s0 + ((u64)s1 << 24) + ((u64)s2 << 48));
    if (c >= 0 && leader) {
      if (!REFINE && c == a) wa = (double)tot;
      else if (allowed(c)) { best_gain = (double)tot - scale * (double)K[c]; best = c; }
    }
  } else {
    // hash slice [2 e0, 2 e1): capacity = 2 deg, at least twice the number of distinct neighbouring communities.  An
    // aggregated row lists every neighbour once, so refinement's keys (refined labels, singletons at first) are nearly
    // all distinct: at capacity deg the linear probing would run at load ~1 with probe chains that grow with the row.
    // At load <= 1/2 they stay short (the slot order changes no sum and no arg-max, so the decisions are the same)
    const int64_t h0 = 2 * e0, h1 = 2 * e1;
    const uint32_t cap = (uint32_t)(h1 - h0);
    for (int64_t s = h0 + lane; s < h1; s += 32) { hkeys[s] = -1; hvals[s] = 0; }
    __syncwarp();
    for (int64_t e = e0 + lane; e < e1; e += 32) {
      const int32_t u = L.indices[e];
      if (u == v || (REFINE && comm[u] != pv)) continue;
      const int32_t c = REFINE ? ref[u] : comm[u];
      uint32_t slot = mix32((uint32_t)c) % cap;
      for (;;) {
        const int32_t prev = atomicCAS(&hkeys[h0 + slot], -1, c);
        if (prev == -1 || prev == c) { atomicAdd((u64*)&hvals[h0 + slot], (u64)L.w[e]); break; }
        slot = slot + 1 == cap ? 0 : slot + 1;
      }
    }
    __syncwarp();
    for (int64_t s = h0 + lane; s < h1; s += 32) {
      const int32_t c = hkeys[s];
      if (c < 0) continue;
      const double tot = (double)hvals[s];
      if (!REFINE && c == a) { wa = tot; continue; }
      if (!allowed(c)) continue;
      const double gain = tot - scale * (double)K[c];
      if (gain > best_gain || (gain == best_gain && c < best)) { best_gain = gain; best = c; }
    }
  }
  // warp arg-max (gain desc, id asc); own-community weight summed (only one lane holds it)
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    const double og = __shfl_xor_sync(0xffffffffu, best_gain, o);
    const int32_t ob = __shfl_xor_sync(0xffffffffu, best, o);
    const double owa = __shfl_xor_sync(0xffffffffu, wa, o);
    wa += owa;
    if (ob >= 0 && (best < 0 || og > best_gain || (og == best_gain && ob < best))) { best_gain = og; best = ob; }
  }
  if (lane == 0) {
    int32_t t = -1;
    uint8_t ts = 0;
    const double stay = REFINE ? 0.0 : wa - scale * ((double)K[a] - kv);
    if (best >= 0 && best_gain > stay + 0.5) {
      t = best;
      ts = (REFINE && csize[best] == 1) ? 1 : 0;
    }
    // Empty-community move (leidenalg's consider_empty_community / igraph's "empty cluster" candidate): a vertex whose
    // best option is still worse than being alone (gain 0) leaves for an empty community.  The empty label it takes is
    // ITS OWN vertex id - free iff csize[v] == 0, and no other vertex can claim it in the same sweep, so simultaneous
    // decisions never collide.  (If somebody else currently uses label v the vertex waits for a later sweep.)
    if (!REFINE && csize[a] > 1 && csize[v] == 0) {
      const double cur = t >= 0 ? best_gain : stay;
      if (0.0 > cur + 0.5) t = v;
    }
    target[oi] = t;
    if (REFINE) tsingle[oi] = ts;
  }
}
// by-position decisions (gathered from all ranks) -> by-vertex arrays
__global__ void scatter_decisions_kernel(const int32_t* __restrict__ wl, int32_t n_wl, const int32_t* __restrict__ t_pos,
                                         const uint8_t* __restrict__ ts_pos, int32_t* __restrict__ target, uint8_t* __restrict__ tsingle) {
  const int32_t wi = blockIdx.x * blockDim.x + threadIdx.x;
  if (wi >= n_wl) return;
  target[wl[wi]] = t_pos[wi];
  if (ts_pos) tsingle[wl[wi]] = ts_pos[wi];
}
__global__ void compact_flags_kernel(int32_t n, const int32_t* __restrict__ flag, const int64_t* __restrict__ pos,
                                     const int32_t* __restrict__ src, int32_t* __restrict__ out) {
  const int32_t i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n && flag[i]) out[pos[i]] = src ? src[i] : i;
}

__global__ void lm_apply_kernel(Level L, const int32_t* __restrict__ wl, int32_t n_wl, int32_t* __restrict__ comm,
                                const int32_t* __restrict__ target, u64* __restrict__ K, int32_t* __restrict__ csize,
                                int32_t* __restrict__ in_next, u64* __restrict__ counters, uint32_t salt, int independent) {
  // counters[0]: accepted moves of this sweep.  in_next[u] = 1 marks the next sweep's active vertices (those skipped by
  // this half-sweep, those deferred + the neighbours of every moved vertex); the list itself is built by a prefix sum
  // over the flags, so it is sorted by vertex id - identical on every rank and from run to run.
  // Independent-set rule (small input graphs only, `independent`): of two ADJACENT vertices that both decided to move, only the one with the higher (salted
  // hash) priority moves in this sweep; the other stays active and decides again against the new state.  A move's gain
  // was computed from its neighbours' communities - which therefore did not change under it - so simultaneous moves can
  // no longer undo each other (the classic failure of synchronous Louvain / Leiden sweeps).
  const int32_t wi = blockIdx.x * blockDim.x + threadIdx.x;
  if (wi >= n_wl) return;
  const int32_t v = wl[wi];
  const int32_t t = target[v];
  if (t == -2) { in_next[v] = 1; return; }
  if (t < 0) return;
  const int64_t e0 = L.indptr[v], e1 = L.indptr[v + 1];
  const uint32_t pv = mix32((uint32_t)v * 0x9E3779B9U + salt);
  for (int64_t e = e0; independent && e < e1; ++e) {
    const int32_t u = L.indices[e];
    if (u == v || target[u] < 0) continue;
    const uint32_t pu = mix32((uint32_t)u * 0x9E3779B9U + salt);
    if (pu > pv || (pu == pv && u > v)) { in_next[v] = 1; return; }   // a moving neighbour outranks v: defer
  }
  const int32_t a = comm[v];
  const u64 kv = (u64)L.k[v];
  comm[v] = t;
  atomicAdd(&K[a], (u64)0 - kv);
  atomicAdd(&K[t], kv);
  atomicAdd(&csize[a], -1);
  atomicAdd(&csize[t], 1);
  for (int64_t e = e0; e < e1; ++e) in_next[L.indices[e]] = 1;
  atomicAdd(&counters[0], 1ull);
}
// decisions are only valid for the sweep that took them: clear the listed vertices' entries (the independent-set rule
// reads target[] of arbitrary neighbours)
__global__ void reset_targets_kernel(const int32_t* __restrict__ wl, int32_t n_wl, int32_t* __restrict__ target) {
  const int32_t wi = blockIdx.x * blockDim.x + threadIdx.x;
  if (wi < n_wl) target[wl[wi]] = -1;
}

__global__ void rf_init_kernel(int32_t n, const int64_t* __restrict__ k, int32_t* __restrict__ ref,
                               int64_t* __restrict__ Kref, int32_t* __restrict__ rsize) {
  const int32_t v = blockIdx.x * blockDim.x + threadIdx.x;
  if (v >= n) return;
  ref[v] = v;
  Kref[v] = k[v];
  rsize[v] = 1;
}
// Louvain (no refinement phase): the aggregate's super-vertices are the communities themselves
// (community labels at an aggregated level are labels of an older level and may exceed L.n, so each community is named by
// its smallest member, like a refined community is named by a vertex id)
__global__ void lv_rep_kernel(int32_t n, const int32_t* __restrict__ comm, int32_t* __restrict__ rep) {
  const int32_t v = blockIdx.x * blockDim.x + threadIdx.x;
  if (v < n) atomicMin(&rep[comm[v]], v);
}
__global__ void lv_ref_kernel(int32_t n, const int32_t* __restrict__ comm, const int32_t* __restrict__ rep,
                              int32_t* __restrict__ ref, int32_t* __restrict__ rsize) {
  const int32_t v = blockIdx.x * blockDim.x + threadIdx.x;
  if (v >= n) return;
  const int32_t r = rep[comm[v]];
  ref[v] = r;
  atomicAdd(&rsize[r], 1);
}
__global__ void rf_apply_kernel(const int32_t* __restrict__ wl, int32_t n_wl, const int64_t* __restrict__ k,
                                const int32_t* __restrict__ target, const uint8_t* __restrict__ tsingle, int32_t* __restrict__ ref,
                                u64* __restrict__ Kref, int32_t* __restrict__ rsize, u64* __restrict__ counters) {
  const int32_t wi = blockIdx.x * blockDim.x + threadIdx.x;
  if (wi >= n_wl) return;
  const int32_t v = wl[wi];
  const int32_t t = target[v];
  if (t < 0) return;
  // a singleton target (label == vertex id) must itself stay put, otherwise v would join an abandoned label
  // (a singleton target is itself on the work-list, so its target[] entry is this round's)
  if (tsingle[v] && target[t] >= 0) return;
  ref[v] = t;
  atomicAdd(&Kref[t], (u64)k[v]);
  Kref[v] = 0;
  atomicAdd(&rsize[t], 1);
  rsize[v] = 0;
  atomicAdd(&counters[0], 1ull);
}
// next round's work-list: the vertices of this round's list that are still singletons (singletons never re-form);
// flag by list position, compacted in order by a prefix sum
__global__ void rf_flag_kernel(const int32_t* __restrict__ wl, int32_t n_wl, const int32_t* __restrict__ ref,
                               const int32_t* __restrict__ rsize, int32_t* __restrict__ flag) {
  const int32_t wi = blockIdx.x * blockDim.x + threadIdx.x;
  if (wi >= n_wl) return;
  flag[wi] = rsize[ref[wl[wi]]] == 1 ? 1 : 0;
}

// ---------------------------------------------------------------------------------------------
// aggregation
__global__ void flag_nonempty_kernel(int32_t n, const int32_t* __restrict__ rsize, int32_t* __restrict__ flag) {
  const int32_t v = blockIdx.x * blockDim.x + threadIdx.x;
  if (v < n) flag[v] = rsize[v] > 0 ? 1 : 0;
}
__global__ void agg_map_kernel(int32_t n, const int32_t* __restrict__ ref, const int64_t* __restrict__ newid_scan,
                               const int32_t* __restrict__ comm, const int64_t* __restrict__ indptr,
                               int32_t* __restrict__ rnew, int32_t* __restrict__ comm_new, int32_t* __restrict__ degsum) {
  const int32_t v = blockIdx.x * blockDim.x + threadIdx.x;
  if (v >= n) return;
  const int32_t r = (int32_t)newid_scan[ref[v]];
  rnew[v] = r;
  comm_new[r] = comm[v];  // all members share the parent community
  atomicAdd(&degsum[r], (int32_t)(indptr[v + 1] - indptr[v]));
}
__global__ void agg_clear_kernel(int64_t n, int32_t* __restrict__ hkeys, int64_t* __restrict__ hvals) {
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) { hkeys[i] = -1; hvals[i] = 0; }
}
__global__ void __launch_bounds__(256)
agg_insert_kernel(Level L, const int32_t* __restrict__ rnew, const int64_t* __restrict__ slice,
                  int32_t* __restrict__ hkeys, int64_t* __restrict__ hvals) {
  const int lane = threadIdx.x & 31;
  const int32_t v = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  if (v >= L.n) return;
  const int32_t r = rnew[v];
  const int64_t s0 = slice[r];
  const uint32_t cap = (uint32_t)(slice[r + 1] - s0);
  for (int64_t e = L.indptr[v] + lane; e < L.indptr[v + 1]; e += 32) {
    const int32_t c = rnew[L.indices[e]];
    uint32_t slot = mix32((uint32_t)c) % cap;
    for (;;) {
      const int32_t prev = atomicCAS(&hkeys[s0 + slot], -1, c);
      if (prev == -1 || prev == c) { atomicAdd((u64*)&hvals[s0 + slot], (u64)L.w[e]); break; }
      slot = slot + 1 == cap ? 0 : slot + 1;
    }
  }
}
__global__ void __launch_bounds__(256)
agg_count_kernel(int32_t nc, const int64_t* __restrict__ slice, const int32_t* __restrict__ hkeys,
                 int32_t* __restrict__ cnt) {
  const int lane = threadIdx.x & 31;
  const int32_t r = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  if (r >= nc) return;
  int c = 0;
  for (int64_t s = slice[r] + lane; s < slice[r + 1]; s += 32) c += hkeys[s] >= 0;
  c = warp_sum(c);
  if (lane == 0) cnt[r] = c;
}
__global__ void __launch_bounds__(256)
agg_fill_kernel(int32_t nc, const int64_t* __restrict__ slice, const int32_t* __restrict__ hkeys,
                const int64_t* __restrict__ hvals, const int64_t* __restrict__ indptr_new,
                int32_t* __restrict__ indices_new, int64_t* __restrict__ w_new) {
  const int lane = threadIdx.x & 31;
  const int32_t r = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  if (r >= nc) return;
  int64_t out = indptr_new[r];
  for (int64_t s0 = slice[r]; s0 < slice[r + 1]; s0 += 32) {
    const int64_t s = s0 + lane;
    const bool has = s < slice[r + 1] && hkeys[s] >= 0;
    const unsigned m = __ballot_sync(0xffffffffu, has);
    if (has) {
      const int64_t p = out + __popc(m & ((1u << lane) - 1u));
      indices_new[p] = hkeys[s];
      w_new[p] = hvals[s];
    }
    out += __popc(m);
  }
}
// block-per-super-vertex variants for coarse levels (few super-vertices with very long hash slices)
__global__ void __launch_bounds__(256)
agg_count_block_kernel(int32_t nc, const int64_t* __restrict__ slice, const int32_t* __restrict__ hkeys,
                       int32_t* __restrict__ cnt) {
  __shared__ int total;
  const int32_t r = blockIdx.x;
  if (threadIdx.x == 0) total = 0;
  __syncthreads();
  int c = 0;
  for (int64_t s = slice[r] + threadIdx.x; s < slice[r + 1]; s += blockDim.x) c += hkeys[s] >= 0;
  c = warp_sum(c);
  if ((threadIdx.x & 31) == 0 && c) atomicAdd(&total, c);
  __syncthreads();
  if (threadIdx.x == 0) cnt[r] = total;
}
__global__ void __launch_bounds__(256)
agg_fill_block_kernel(int32_t nc, const int64_t* __restrict__ slice, const int32_t* __restrict__ hkeys,
                      const int64_t* __restrict__ hvals, const int64_t* __restrict__ indptr_new,
                      int32_t* __restrict__ indices_new, int64_t* __restrict__ w_new) {
  __shared__ int cursor;  // entry order inside a row is irrelevant (all reductions are exact integers)
  const int32_t r = blockIdx.x;
  if (threadIdx.x == 0) cursor = 0;
  __syncthreads();
  const int64_t out = indptr_new[r];
  for (int64_t s = slice[r] + threadIdx.x; s < slice[r + 1]; s += blockDim.x) {
    if (hkeys[s] >= 0) {
      const int p = atomicAdd(&cursor, 1);
      indices_new[out + p] = hkeys[s];
      w_new[out + p] = hvals[s];
    }
  }
}
__global__ void compose_kernel(int64_t n0, int32_t* __restrict__ node_of, const int32_t* __restrict__ rnew) {
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n0) node_of[i] = rnew[node_of[i]];
}
__global__ void gather_kernel(int64_t n0, const int32_t* __restrict__ node_of, const int32_t* __restrict__ comm,
                              int32_t* __restrict__ out) {
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n0) out[i] = comm[node_of[i]];
}

// ---------------------------------------------------------------------------------------------
// modularity pieces and final renumbering
__global__ void internal_weight_kernel(int32_t n, const int64_t* __restrict__ indptr, const int32_t* __restrict__ indices,
                                       const int64_t* __restrict__ w, const int32_t* __restrict__ comm,
                                       u64* __restrict__ internal) {
  const int32_t v = blockIdx.x * blockDim.x + threadIdx.x;
  long long s = 0;
  if (v < n) {
    const int32_t c = comm[v];
    for (int64_t e = indptr[v]; e < indptr[v + 1]; ++e)
      if (comm[indices[e]] == c) s += w[e];
  }
  s = warp_sum(s);
  if ((threadIdx.x & 31) == 0 && s != 0) atomicAdd(internal, (u64)s);
}
__global__ void relabel_kernel(int64_t n, int32_t* __restrict__ comm, const int32_t* __restrict__ newid) {
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) comm[i] = newid[comm[i]];
}

struct Work {
  sb2_ctx* ctx;
  cudaStream_t st;
  int32_t n0;
  u64* K;          // [n0]
  int32_t* csize;  // [n0]
  int32_t* hkeys;  // [2 E0]
  int64_t* hvals;  // [2 E0]
  int32_t* target; // [n0]
  uint8_t* tsingle;
  int32_t* wl[2];     // work-lists (vertices to decide this sweep / next sweep)
  int32_t* in_next;   // membership flags of the next work-list
  int64_t* pos;       // [n0 + 1] prefix sums of the flags
  int32_t* t_pos;     // [n0 + pad] decisions by list position (sharded decide)
  uint8_t* ts_pos;
  u64* counter;    // device counters [4]
  double gamma;
  double total;    // 2m in fixed units
  uint32_t seed;
  int64_t moves_total;
  int last_sweeps;
  bool first_pass;
  bool careful;     // small INPUT graphs (n0 < CAREFUL_N): 8 vertex classes per round of sweeps + independent-set rule - closer
                    // to the sequential algorithm, at a cost in sweeps that only a graph this small can afford
  bool exact;       // SB2_LEIDEN_EXACT=1: no first-pass / refinement cut-offs (every phase runs to its fixed point)
  bool timing;      // SB2_TIMING set: per-level sweep / round counts on stderr
  bool verbose;     // SB2_TIMING and SB2_VERBOSE set: one line per sweep
  int64_t syncs;    // host synchronisations of the sweep loops and the aggregation (SB2_TIMING summary)
};

inline unsigned gridw(int64_t n) { return (unsigned)ceil_div64(n, 8); }    // warp per item, 8 warps/CTA
inline unsigned gridt(int64_t n) { return (unsigned)ceil_div64(n, 256); }  // thread per item

// Decide the work-list wl[0, n_wl).  With a communicator attached (one process per GPU, every rank holding the same
// graph and the same state) a long list is SHARDED: each rank decides a contiguous slice, the slices are all-gathered
// (NCCL, 4 B per listed vertex) and scattered by vertex id; every rank then applies all moves, so the replicas stay
// bit-identical to each other and to a single-GPU run - decisions only read the snapshot.
constexpr int32_t SHARD_MIN = 32768;
// the two performance cut-offs (first-pass local moving below 0.5 % movers, refinement below 0.1 % merges) only apply to
// levels this large: below, every phase runs to its fixed point (the sweeps cost microseconds there)
constexpr int32_t CUTOFF_MIN_N = 100000;
template <bool REFINE>
int32_t decide(Work& w, const Level& L, const int32_t* wl, int32_t n_wl, const int32_t* comm, const int32_t* ref, const int64_t* K,
               const int32_t* csize, int sweep, int noskip) {
  sb2_ctx* ctx = w.ctx;
  const int cshift = w.careful ? 3 : 1;   // 2^cshift vertex classes per round of sweeps (decide_kernel)
  const int P = ctx->nccl_comm ? ctx->n_ranks : 1;
  if (P == 1 || n_wl < SHARD_MIN) {
    decide_kernel<REFINE><<<gridw(n_wl), 256, 0, w.st>>>(L, wl, 0, n_wl, comm, ref, K, csize, w.gamma, w.total, w.seed, sweep, noskip,
                                                         w.hkeys, w.hvals, w.target, w.tsingle, 0, cshift);
    SB2_LAUNCH_CHECK(ctx);
    return SB2_OK;
  }
  const int32_t chunk = (int32_t)ceil_div64(n_wl, P);
  const int32_t b = std::min<int64_t>((int64_t)ctx->rank * chunk, n_wl), e = std::min<int64_t>((int64_t)(ctx->rank + 1) * chunk, n_wl);
  if (e > b) {
    decide_kernel<REFINE><<<gridw(e - b), 256, 0, w.st>>>(L, wl, b, e, comm, ref, K, csize, w.gamma, w.total, w.seed, sweep, noskip,
                                                          w.hkeys, w.hvals, w.t_pos, w.ts_pos, 1, cshift);
    SB2_LAUNCH_CHECK(ctx);
  }
  SB2_TRY(sb2_comm_allgather(ctx, w.t_pos + (size_t)ctx->rank * chunk, w.t_pos, (int64_t)chunk * 4));
  if (REFINE) SB2_TRY(sb2_comm_allgather(ctx, w.ts_pos + (size_t)ctx->rank * chunk, w.ts_pos, (int64_t)chunk));
  scatter_decisions_kernel<<<gridt(n_wl), 256, 0, w.st>>>(wl, n_wl, w.t_pos, REFINE ? w.ts_pos : nullptr, w.target, w.tsingle);
  SB2_LAUNCH_CHECK(ctx);
  return SB2_OK;
}

// flags[0, n) -> out = the flagged positions (or src[position]) in order; *n_out = their number (host, synchronises);
// *counter0 (optional) = w.counter[0] read in the same synchronisation
int32_t compact(Work& w, int32_t n, const int32_t* src, int32_t* out, int32_t* n_out, u64* counter0) {
  sb2_ctx* ctx = w.ctx;
  SB2_TRY(sb2_scan_i32_to_i64(ctx, w.in_next, n, w.pos));
  compact_flags_kernel<<<gridt(n), 256, 0, w.st>>>(n, w.in_next, w.pos, src, out);
  SB2_LAUNCH_CHECK(ctx);
  int64_t cnt = 0;
  SB2_CUDA(cudaMemcpyAsync(&cnt, w.pos + n, sizeof(int64_t), cudaMemcpyDeviceToHost, w.st));
  if (counter0) SB2_CUDA(cudaMemcpyAsync(counter0, w.counter, sizeof(u64), cudaMemcpyDeviceToHost, w.st));
  SB2_CUDA(cudaStreamSynchronize(w.st));
  ++w.syncs;
  *n_out = (int32_t)cnt;
  return SB2_OK;
}

int32_t local_move(Work& w, const Level& L, int32_t* comm, int64_t* moves_out) {
  sb2_ctx* ctx = w.ctx;
  SB2_CUDA(cudaMemsetAsync(w.K, 0, sizeof(u64) * w.n0, w.st));
  SB2_CUDA(cudaMemsetAsync(w.csize, 0, sizeof(int32_t) * w.n0, w.st));
  comm_stats_kernel<<<gridt(L.n), 256, 0, w.st>>>(L.n, comm, L.k, w.K, w.csize);
  SB2_LAUNCH_CHECK(ctx);
  iota_kernel<<<gridt(L.n), 256, 0, w.st>>>(w.wl[0], L.n);   // first sweep: every vertex
  SB2_LAUNCH_CHECK(ctx);
  SB2_CUDA(cudaMemsetAsync(w.target, 0xFF, sizeof(int32_t) * (size_t)L.n, w.st));   // no decision pending anywhere
  int cur = 0, noskip = 0;
  int32_t n_wl = L.n;
  u64 prev_c = ~0ull;
  int64_t moves = 0;
  const int max_sweeps = 200;
  for (int sweep = 0; sweep < max_sweeps && n_wl > 0; ++sweep) {
    w.last_sweeps = sweep + 1;
    SB2_CUDA(cudaMemsetAsync(w.in_next, 0, sizeof(int32_t) * (size_t)L.n, w.st));
    SB2_CUDA(cudaMemsetAsync(w.counter, 0, 2 * sizeof(u64), w.st));
    SB2_TRY(decide<false>(w, L, w.wl[cur], n_wl, comm, nullptr, (const int64_t*)w.K, w.csize, sweep, noskip));
    lm_apply_kernel<<<gridt(n_wl), 256, 0, w.st>>>(L, w.wl[cur], n_wl, comm, w.target, w.K, w.csize, w.in_next, w.counter,
                                                   w.seed * 0x85EBCA6BU + (uint32_t)sweep, w.careful ? 1 : 0);
    SB2_LAUNCH_CHECK(ctx);
    reset_targets_kernel<<<gridt(n_wl), 256, 0, w.st>>>(w.wl[cur], n_wl, w.target);
    SB2_LAUNCH_CHECK(ctx);
    u64 c = 0;
    SB2_TRY(compact(w, L.n, nullptr, w.wl[cur ^ 1], &n_wl, &c));
    moves += (int64_t)c;
    cur ^= 1;
    if (w.verbose) fprintf(stderr, "[sb2 leiden]     sweep %d noskip=%d moves=%llu next=%d\n", sweep, noskip, c, n_wl);
    if (c == 0) {
      if (noskip) break;
      noskip = 1;  // confirm with a sweep in which every active vertex decides
    } else if (w.first_pass && !w.exact && L.n >= CUTOFF_MIN_N && (int64_t)c * 200 < (int64_t)L.n) {
      // First pass only: once fewer than 0.5 % of the vertices still move, what remains is communities
      // merging one vertex at a time in slow waves - the aggregated level does that in a single move, and the
      // following passes (which run local moving to exact convergence) pick up any leftover single-vertex gain.
      break;
    } else if ((int64_t)c * 512 < (int64_t)L.n && (!noskip || c < prev_c)) {
      // tail: few vertices still move, simultaneous conflicting moves are unlikely -> let every active vertex
      // decide each sweep (halves the number of tail sweeps); falls back to half-sweeps if it stops shrinking
      noskip = 1;
    } else {
      noskip = 0;
    }
    prev_c = c;
  }
  *moves_out = moves;
  if (w.timing) fprintf(stderr, "[sb2 leiden]   local_move n=%d sweeps=%d moves=%lld\n", L.n, w.last_sweeps, (long long)moves);
  return SB2_OK;
}

int32_t refine(Work& w, const Level& L, const int32_t* comm, int32_t* ref, int64_t* Kref, int32_t* rsize) {
  sb2_ctx* ctx = w.ctx;
  rf_init_kernel<<<gridt(L.n), 256, 0, w.st>>>(L.n, L.k, ref, Kref, rsize);
  SB2_LAUNCH_CHECK(ctx);
  iota_kernel<<<gridt(L.n), 256, 0, w.st>>>(w.wl[0], L.n);   // every vertex starts as a singleton
  SB2_LAUNCH_CHECK(ctx);
  int cur = 0;
  int32_t n_wl = L.n;
  for (int round = 0; round < 64 && n_wl > 0; ++round) {
    SB2_CUDA(cudaMemsetAsync(w.counter, 0, 2 * sizeof(u64), w.st));
    SB2_TRY(decide<true>(w, L, w.wl[cur], n_wl, comm, ref, Kref, rsize, round, 1));
    rf_apply_kernel<<<gridt(n_wl), 256, 0, w.st>>>(w.wl[cur], n_wl, L.k, w.target, w.tsingle, ref, (u64*)Kref, rsize, w.counter);
    SB2_LAUNCH_CHECK(ctx);
    rf_flag_kernel<<<gridt(n_wl), 256, 0, w.st>>>(w.wl[cur], n_wl, ref, rsize, w.in_next);
    SB2_LAUNCH_CHECK(ctx);
    u64 c = 0;
    int32_t n_next = 0;
    SB2_TRY(compact(w, n_wl, w.wl[cur], w.wl[cur ^ 1], &n_next, &c));
    if (w.timing) fprintf(stderr, "[sb2 leiden]   refine n=%d round=%d singletons=%d merges=%llu\n", L.n, round, n_wl, c);
    cur ^= 1;
    n_wl = n_next;
    // the first rounds do nearly all the merging; stragglers (< 0.1 % of the vertices per round) simply stay
    // singletons of the refined partition, which only makes the aggregate marginally larger
    if (c == 0 || (!w.exact && L.n >= CUTOFF_MIN_N && round >= 2 && c * 1000 < (u64)L.n)) break;
  }
  return SB2_OK;
}

}  // namespace

// quality of `comm` (labels < n) on the level-0 fixed-point graph; K/csize scratch sized n
static int32_t quality_device(sb2_ctx* ctx, ScratchScope& scr, int32_t n, const int64_t* indptr, const int32_t* indices,
                              const int64_t* wfx, const int64_t* kfx, double total, double gamma, const int32_t* comm,
                              double* q_out, int32_t n_labels = -1) {
  cudaStream_t st = ctx->stream;
  u64* K;
  int32_t* csize;
  u64* internal;
  SB2_TRY(scr.alloc(&K, (size_t)n));
  SB2_TRY(scr.alloc(&csize, (size_t)n));
  SB2_TRY(scr.alloc(&internal, 2));
  SB2_CUDA(cudaMemsetAsync(K, 0, sizeof(u64) * n, st));
  SB2_CUDA(cudaMemsetAsync(csize, 0, sizeof(int32_t) * n, st));
  SB2_CUDA(cudaMemsetAsync(internal, 0, 16, st));
  comm_stats_kernel<<<gridt(n), 256, 0, st>>>(n, comm, kfx, K, csize);
  SB2_LAUNCH_CHECK(ctx);
  internal_weight_kernel<<<gridt(n), 256, 0, st>>>(n, indptr, indices, wfx, comm, internal);
  SB2_LAUNCH_CHECK(ctx);
  const int32_t nl = (n_labels > 0 && n_labels < n) ? n_labels : n;  // labels are < nl (compact after renumbering)
  std::vector<u64> hK((size_t)nl);
  u64 hin = 0;
  SB2_CUDA(cudaMemcpyAsync(hK.data(), K, sizeof(u64) * nl, cudaMemcpyDeviceToHost, st));
  SB2_CUDA(cudaMemcpyAsync(&hin, internal, sizeof(u64), cudaMemcpyDeviceToHost, st));
  SB2_CUDA(cudaStreamSynchronize(st));
  if (total <= 0.0) { *q_out = 0.0; return SB2_OK; }
  double pen = 0.0;
  for (int32_t c = 0; c < nl; ++c) {
    const double kc = (double)(long long)hK[c];
    pen += kc * kc;
  }
  *q_out = ((double)(long long)hin - gamma * pen / total) / total;
  return SB2_OK;
}

// renumber labels (< n) by decreasing size, ties -> smaller first member; returns #communities.
// Sizes / first members are gathered with integer atomics, only the (few) non-empty labels travel to the host
// for the sort.
namespace {
__global__ void label_stats_kernel(int64_t n, const int32_t* __restrict__ comm, int32_t* __restrict__ csize,
                                   int32_t* __restrict__ minmem) {
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  atomicAdd(&csize[comm[i]], 1);
  atomicMin(&minmem[comm[i]], (int32_t)i);
}
__global__ void label_compact_kernel(int64_t n, const int32_t* __restrict__ csize, const int32_t* __restrict__ minmem,
                                     const int64_t* __restrict__ pos, int32_t* __restrict__ lab, int32_t* __restrict__ sz,
                                     int32_t* __restrict__ mm) {
  const int64_t c = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (c >= n || csize[c] <= 0) return;
  const int64_t p = pos[c];
  lab[p] = (int32_t)c; sz[p] = csize[c]; mm[p] = minmem[c];
}
__global__ void label_scatter_kernel(int32_t nc, const int32_t* __restrict__ lab, const int32_t* __restrict__ rank,
                                     int32_t* __restrict__ newid) {
  const int32_t p = blockIdx.x * blockDim.x + threadIdx.x;
  if (p < nc) newid[lab[p]] = rank[p];
}
}  // namespace
static int32_t renumber_device(sb2_ctx* ctx, ScratchScope& scr, int64_t n, int32_t* comm, int32_t* n_comms) {
  cudaStream_t st = ctx->stream;
  int32_t *csize, *minmem, *newid, *flag, *lab, *sz, *mm, *rank;
  int64_t* pos;
  SB2_TRY(scr.alloc(&csize, (size_t)n));
  SB2_TRY(scr.alloc(&minmem, (size_t)n));
  SB2_TRY(scr.alloc(&newid, (size_t)n));
  SB2_TRY(scr.alloc(&flag, (size_t)n));
  SB2_TRY(scr.alloc(&pos, (size_t)n + 1));
  SB2_CUDA(cudaMemsetAsync(csize, 0, sizeof(int32_t) * n, st));
  SB2_CUDA(cudaMemsetAsync(minmem, 0x7f, sizeof(int32_t) * n, st));
  label_stats_kernel<<<gridt(n), 256, 0, st>>>(n, comm, csize, minmem);
  SB2_LAUNCH_CHECK(ctx);
  flag_nonempty_kernel<<<gridt(n), 256, 0, st>>>((int32_t)n, csize, flag);
  SB2_LAUNCH_CHECK(ctx);
  SB2_TRY(sb2_scan_i32_to_i64(ctx, flag, n, pos));
  int64_t nc64 = 0;
  SB2_CUDA(cudaMemcpyAsync(&nc64, pos + n, sizeof(int64_t), cudaMemcpyDeviceToHost, st));
  SB2_CUDA(cudaStreamSynchronize(st));
  const int32_t nc = (int32_t)nc64;
  SB2_TRY(scr.alloc(&lab, (size_t)nc * 4));
  sz = lab + nc; mm = sz + nc; rank = mm + nc;
  label_compact_kernel<<<gridt(n), 256, 0, st>>>(n, csize, minmem, pos, lab, sz, mm);
  SB2_LAUNCH_CHECK(ctx);
  std::vector<int32_t> h((size_t)nc * 3);
  SB2_CUDA(cudaMemcpyAsync(h.data(), lab, sizeof(int32_t) * (size_t)nc * 3, cudaMemcpyDeviceToHost, st));
  SB2_CUDA(cudaStreamSynchronize(st));
  const int32_t* hsz = h.data() + nc;
  const int32_t* hmm = h.data() + 2 * (size_t)nc;
  std::vector<int32_t> ord((size_t)nc), hrank((size_t)nc);
  for (int32_t p = 0; p < nc; ++p) ord[p] = p;
  std::sort(ord.begin(), ord.end(), [&](int32_t a, int32_t b) {
    if (hsz[a] != hsz[b]) return hsz[a] > hsz[b];
    return hmm[a] < hmm[b];
  });
  for (int32_t r = 0; r < nc; ++r) hrank[ord[r]] = r;
  SB2_CUDA(cudaMemcpyAsync(rank, hrank.data(), sizeof(int32_t) * (size_t)nc, cudaMemcpyHostToDevice, st));
  label_scatter_kernel<<<gridt(nc), 256, 0, st>>>(nc, lab, rank, newid);
  SB2_LAUNCH_CHECK(ctx);
  relabel_kernel<<<gridt(n), 256, 0, st>>>(n, comm, newid);
  SB2_LAUNCH_CHECK(ctx);
  SB2_CUDA(cudaStreamSynchronize(st));
  *n_comms = nc;
  return SB2_OK;
}

static int32_t prepare_level0(sb2_ctx* ctx, ScratchScope& scr, int64_t n, const int64_t* d_indptr, const float* d_weights,
                              int64_t* nnz_out, int64_t** wfx, int64_t** kfx, double* total) {
  cudaStream_t st = ctx->stream;
  int64_t nnz = 0;
  SB2_CUDA(cudaMemcpyAsync(&nnz, d_indptr + n, sizeof(int64_t), cudaMemcpyDeviceToHost, st));
  SB2_CUDA(cudaStreamSynchronize(st));
  *nnz_out = nnz;
  SB2_TRY(scr.alloc(wfx, (size_t)nnz));
  SB2_TRY(scr.alloc(kfx, (size_t)n));
  u64* tot;   // [0] total, [1] the weight scan (two int32)
  SB2_TRY(scr.alloc(&tot, 2));
  int32_t* scan = (int32_t*)(tot + 1);
  SB2_CUDA(cudaMemsetAsync(tot, 0, 16, st));
  // every fixed-point arc is <= 2^32 units; beyond 2^30 arcs the scale drops by the missing bits so that the total
  // stays below 2^62
  int extra_shift = 0;
  while ((nnz >> extra_shift) > ((int64_t)1 << 30)) ++extra_shift;
  if (nnz > 0) {
    weight_scan_kernel<<<(unsigned)std::min<int64_t>(gridt(nnz), 1024), 256, 0, st>>>(d_weights, nnz, scan);
    SB2_LAUNCH_CHECK(ctx);
    to_fixed_kernel<<<gridt(nnz), 256, 0, st>>>(d_weights, nnz, scan, extra_shift, *wfx);
    SB2_LAUNCH_CHECK(ctx);
  }
  strength_kernel<<<gridt(n), 256, 0, st>>>((int32_t)n, d_indptr, *wfx, *kfx, tot);
  SB2_LAUNCH_CHECK(ctx);
  u64 ht[2] = {0, 0};
  SB2_CUDA(cudaMemcpyAsync(ht, tot, sizeof(ht), cudaMemcpyDeviceToHost, st));
  SB2_CUDA(cudaStreamSynchronize(st));
  int32_t hscan[2];
  memcpy(hscan, &ht[1], sizeof(hscan));
  if (hscan[1]) {
    sb2_set_error("bad argument: edge weights must be finite and non-negative (found NaN, inf or a negative weight)");
    return SB2_E_BADARG;
  }
  *total = (double)(long long)ht[0];
  return SB2_OK;
}

extern "C" int32_t sb2_modularity_csr_f32(sb2_ctx* ctx, int64_t n, const int64_t* d_indptr, const int32_t* d_indices,
                                          const float* d_weights, double resolution, const int32_t* d_membership,
                                          double* h_modularity) {
  SB2_CHECK_ARG(ctx && d_indptr && d_indices && d_weights && d_membership && h_modularity, "null pointer");
  SB2_CHECK_ARG(n >= 1 && n < INT32_MAX, "n");
  SB2_CUDA(cudaSetDevice(ctx->device));
  ScratchScope scr(ctx);
  int64_t nnz, *wfx, *kfx;
  double total;
  SB2_TRY(prepare_level0(ctx, scr, n, d_indptr, d_weights, &nnz, &wfx, &kfx, &total));
  // labels may be arbitrary non-negative ints < n
  return quality_device(ctx, scr, (int32_t)n, d_indptr, d_indices, wfx, kfx, total, resolution, d_membership, h_modularity);
}

static int32_t leiden_core(sb2_ctx* ctx, int64_t n, const int64_t* d_indptr, const int32_t* d_indices,
                           const float* d_weights, double resolution, int32_t n_iterations, uint64_t seed,
                           int32_t* d_membership, double* h_modularity, int32_t* h_n_comms,
                           sb2_leiden_info* info, bool louvain = false) {
  SB2_CHECK_ARG(ctx && d_indptr && d_indices && d_weights && d_membership && h_modularity && h_n_comms, "null pointer");
  SB2_CHECK_ARG(n >= 1 && n < INT32_MAX, "n");
  SB2_CHECK_ARG(resolution >= 0.0, "resolution");
  SB2_CUDA(cudaSetDevice(ctx->device));
  cudaStream_t st = ctx->stream;
  ScratchScope scr(ctx);
  const int32_t n0 = (int32_t)n;
  int64_t nnz0, *wfx0, *kfx0;
  double total;
  SB2_TRY(prepare_level0(ctx, scr, n, d_indptr, d_weights, &nnz0, &wfx0, &kfx0, &total));

  Work w{};
  w.ctx = ctx; w.st = st; w.n0 = n0; w.gamma = resolution; w.total = total;
  w.seed = (uint32_t)(seed ^ (seed >> 32));
  { const char* ex = getenv("SB2_LEIDEN_EXACT"); w.exact = ex && atoi(ex) > 0; }
  w.careful = n0 < 65536;
  w.timing = getenv("SB2_TIMING") != nullptr;
  w.verbose = w.timing && getenv("SB2_VERBOSE") != nullptr;
  SB2_TRY(scr.alloc(&w.K, (size_t)n0));
  SB2_TRY(scr.alloc(&w.csize, (size_t)n0));
  SB2_TRY(scr.alloc(&w.hkeys, (size_t)std::max<int64_t>(2 * nnz0, 1)));   // decide: 2 slots per arc; aggregation: 1
  SB2_TRY(scr.alloc(&w.hvals, (size_t)std::max<int64_t>(2 * nnz0, 1)));
  SB2_TRY(scr.alloc(&w.target, (size_t)n0));
  SB2_TRY(scr.alloc(&w.tsingle, (size_t)n0));
  SB2_TRY(scr.alloc(&w.wl[0], (size_t)n0));
  SB2_TRY(scr.alloc(&w.wl[1], (size_t)n0));
  SB2_TRY(scr.alloc(&w.in_next, (size_t)n0));
  SB2_TRY(scr.alloc(&w.pos, (size_t)n0 + 1));
  SB2_TRY(scr.alloc(&w.t_pos, (size_t)n0 + 64));    // + padding: the all-gather moves n_ranks equal chunks
  SB2_TRY(scr.alloc(&w.ts_pos, (size_t)n0 + 64));
  SB2_TRY(scr.alloc(&w.counter, 4));
  int32_t *node_of, *comm, *comm_next, *ref, *rsize, *rnew, *flag, *degsum, *cnt;
  int64_t *Kref, *scan_tmp;
  SB2_TRY(scr.alloc(&node_of, (size_t)n0));
  SB2_TRY(scr.alloc(&comm, (size_t)n0));
  SB2_TRY(scr.alloc(&comm_next, (size_t)n0));
  SB2_TRY(scr.alloc(&ref, (size_t)n0));
  SB2_TRY(scr.alloc(&rsize, (size_t)n0));
  SB2_TRY(scr.alloc(&rnew, (size_t)n0));
  SB2_TRY(scr.alloc(&flag, (size_t)n0));
  SB2_TRY(scr.alloc(&degsum, (size_t)n0));
  SB2_TRY(scr.alloc(&cnt, (size_t)n0));
  SB2_TRY(scr.alloc(&Kref, (size_t)n0));
  SB2_TRY(scr.alloc(&scan_tmp, (size_t)n0 + 1));
  int64_t* slice;
  SB2_TRY(scr.alloc(&slice, (size_t)n0 + 1));

  iota_kernel<<<gridt(n0), 256, 0, st>>>(d_membership, n0);
  SB2_LAUNCH_CHECK(ctx);

  int passes = 0, levels = 0;
  int64_t prev_higher_moves = -1;
  PhaseTimer pt(st);
  double t_lm = 0, t_rf = 0, t_agg = 0, t_fin = 0;
  int n_lm = 0;
  if (total > 0.0) {
    for (;;) {
      // ---- one Leiden pass starting from d_membership on the level-0 graph ----
      Level L{n0, d_indptr, d_indices, wfx0, kfx0};
      SB2_CUDA(cudaMemcpyAsync(comm, d_membership, sizeof(int32_t) * n0, cudaMemcpyDeviceToDevice, st));
      iota_kernel<<<gridt(n0), 256, 0, st>>>(node_of, n0);
      SB2_LAUNCH_CHECK(ctx);
      w.first_pass = passes == 0 && n_iterations != 1;
      int64_t pass_moves = 0, higher_moves = 0;
      int lev = 0;
      bool idle_pass = false;
      ScratchScope lvl(ctx);  // aggregated graphs of this pass
      for (;;) {
        int64_t mv = 0;
        pt.reset();
        SB2_TRY(local_move(w, L, comm, &mv));
        const double lm0 = t_lm;
        pt.lap(&t_lm);
        if (w.timing) fprintf(stderr, "[sb2 leiden]   level n=%d local_move %.3f ms\n", L.n, t_lm - lm0);
        ++n_lm;
        pass_moves += mv;
        if (lev > 0) higher_moves += mv;
        // A pass whose level-0 sweep moves nothing, started from a partition on which the previous pass already
        // found no move at any aggregated level, would replay that pass exactly (refinement and aggregation are
        // deterministic functions of the partition; "no improving move exists" does not depend on the seed).
        if (lev == 0 && mv == 0 && passes > 0 && prev_higher_moves == 0 && n_iterations < 0) { idle_pass = true; break; }
        ++lev;
        levels = lev;
        if (louvain) {
          SB2_CUDA(cudaMemsetAsync(rsize, 0, sizeof(int32_t) * L.n, st));
          SB2_CUDA(cudaMemsetAsync(cnt, 0x7f, sizeof(int32_t) * n0, st));  // cnt doubles as the representative table here
          lv_rep_kernel<<<gridt(L.n), 256, 0, st>>>(L.n, comm, cnt);
          SB2_LAUNCH_CHECK(ctx);
          lv_ref_kernel<<<gridt(L.n), 256, 0, st>>>(L.n, comm, cnt, ref, rsize);
          SB2_LAUNCH_CHECK(ctx);
        } else {
          SB2_TRY(refine(w, L, comm, ref, Kref, rsize));
        }
        const double rf0 = t_rf;
        pt.lap(&t_rf);
        if (w.timing) fprintf(stderr, "[sb2 leiden]   level n=%d refine %.3f ms\n", L.n, t_rf - rf0);
        // compact refined labels
        flag_nonempty_kernel<<<gridt(L.n), 256, 0, st>>>(L.n, rsize, flag);
        SB2_LAUNCH_CHECK(ctx);
        SB2_TRY(sb2_scan_i32_to_i64(ctx, flag, L.n, scan_tmp));
        int64_t nc64 = 0;
        SB2_CUDA(cudaMemcpyAsync(&nc64, scan_tmp + L.n, sizeof(int64_t), cudaMemcpyDeviceToHost, st));
        SB2_CUDA(cudaStreamSynchronize(st));
        ++w.syncs;
        const int32_t nc = (int32_t)nc64;
        if (nc >= L.n) break;  // nothing merged: the aggregate would not shrink
        // ---- aggregate ----
        SB2_CUDA(cudaMemsetAsync(degsum, 0, sizeof(int32_t) * nc, st));
        agg_map_kernel<<<gridt(L.n), 256, 0, st>>>(L.n, ref, scan_tmp, comm, L.indptr, rnew, comm_next, degsum);
        SB2_LAUNCH_CHECK(ctx);
        SB2_TRY(sb2_scan_i32_to_i64(ctx, degsum, nc, slice));
        int64_t eL = 0;
        SB2_CUDA(cudaMemcpyAsync(&eL, slice + nc, sizeof(int64_t), cudaMemcpyDeviceToHost, st));
        SB2_CUDA(cudaStreamSynchronize(st));
        ++w.syncs;
        if (eL > 0) {
          agg_clear_kernel<<<gridt(eL), 256, 0, st>>>(eL, w.hkeys, w.hvals);
          SB2_LAUNCH_CHECK(ctx);
          agg_insert_kernel<<<gridw(L.n), 256, 0, st>>>(L, rnew, slice, w.hkeys, w.hvals);
          SB2_LAUNCH_CHECK(ctx);
        }
        // mapping by mean slice length: warp per super-vertex while slices are short, CTA per super-vertex at
        // the coarse levels where a few thousand super-vertices own millions of slots
        const bool coarse = eL > (int64_t)nc * 256;
        if (coarse) agg_count_block_kernel<<<(unsigned)nc, 256, 0, st>>>(nc, slice, w.hkeys, cnt);
        else agg_count_kernel<<<gridw(nc), 256, 0, st>>>(nc, slice, w.hkeys, cnt);
        SB2_LAUNCH_CHECK(ctx);
        int64_t* indptr_new;
        SB2_TRY(lvl.alloc(&indptr_new, (size_t)nc + 1));
        SB2_TRY(sb2_scan_i32_to_i64(ctx, cnt, nc, indptr_new));
        int64_t nnz_new = 0;
        SB2_CUDA(cudaMemcpyAsync(&nnz_new, indptr_new + nc, sizeof(int64_t), cudaMemcpyDeviceToHost, st));
        SB2_CUDA(cudaStreamSynchronize(st));
        ++w.syncs;
        int32_t* indices_new;
        int64_t *w_new, *k_new;
        SB2_TRY(lvl.alloc(&indices_new, (size_t)std::max<int64_t>(nnz_new, 1)));
        SB2_TRY(lvl.alloc(&w_new, (size_t)std::max<int64_t>(nnz_new, 1)));
        SB2_TRY(lvl.alloc(&k_new, (size_t)nc));
        if (coarse) agg_fill_block_kernel<<<(unsigned)nc, 256, 0, st>>>(nc, slice, w.hkeys, w.hvals, indptr_new, indices_new, w_new);
        else agg_fill_kernel<<<gridw(nc), 256, 0, st>>>(nc, slice, w.hkeys, w.hvals, indptr_new, indices_new, w_new);
        SB2_LAUNCH_CHECK(ctx);
        SB2_CUDA(cudaMemsetAsync(w.counter + 2, 0, sizeof(u64), st));
        strength_kernel<<<gridt(nc), 256, 0, st>>>(nc, indptr_new, w_new, k_new, w.counter + 2);
        SB2_LAUNCH_CHECK(ctx);
        compose_kernel<<<gridt(n0), 256, 0, st>>>(n0, node_of, rnew);
        SB2_LAUNCH_CHECK(ctx);
        std::swap(comm, comm_next);
        L = Level{nc, indptr_new, indices_new, w_new, k_new};
        pt.lap(&t_agg);
      }
      if (idle_pass) { ++passes; break; }
      prev_higher_moves = higher_moves;
      gather_kernel<<<gridt(n0), 256, 0, st>>>(n0, node_of, comm, d_membership);
      SB2_LAUNCH_CHECK(ctx);
      SB2_CUDA(cudaStreamSynchronize(st));
      ++passes;
      w.moves_total += pass_moves;
      w.seed = mix32(w.seed + 0x9E3779B9U);
      if (n_iterations >= 0 ? passes >= n_iterations : pass_moves == 0) break;
      if (passes >= 64) break;
    }
  }
  pt.reset();
  SB2_TRY(renumber_device(ctx, scr, n, d_membership, h_n_comms));
  SB2_TRY(quality_device(ctx, scr, n0, d_indptr, d_indices, wfx0, kfx0, total, resolution, d_membership, h_modularity, *h_n_comms));
  pt.lap(&t_fin);
  if (pt.on)
    fprintf(stderr, "[sb2 leiden] n=%d passes=%d local_move %.1f ms (%d calls) refine %.1f ms aggregate %.1f ms finalize %.1f ms syncs=%lld\n",
            n0, passes, t_lm, n_lm, t_rf, t_agg, t_fin, (long long)w.syncs);
  if (info) {
    info->passes = passes;
    info->levels = levels;
    info->moves = w.moves_total;
  }
  return SB2_OK;
}

// Small graphs: the synchronous sweeps have a higher run-to-run variance than the sequential algorithm (on the reference's
// pbmc68k_reduced graph about one seed in four ends 0.5 % below the optimum every sequential run finds), and a run costs
// milliseconds - so the optimiser is started from 4 seeds derived from `seed` and the best partition is returned.  The
// result is still a deterministic function of (graph, resolution, n_iterations, seed).  SB2_LEIDEN_RESTARTS overrides
// the number of starts; graphs of SMALL_N vertices or more always use one.
extern "C" int32_t sb2_leiden_csr_f32(sb2_ctx* ctx, int64_t n, const int64_t* d_indptr, const int32_t* d_indices,
                                      const float* d_weights, double resolution, int32_t n_iterations, uint64_t seed,
                                      int32_t* d_membership, double* h_modularity, int32_t* h_n_comms,
                                      sb2_leiden_info* info) {
  SB2_CHECK_ARG(ctx && d_membership && h_modularity && h_n_comms, "null pointer");
  constexpr int64_t SMALL_N = 65536;
  int starts = n < SMALL_N ? 4 : 1;
  if (const char* e = getenv("SB2_LEIDEN_RESTARTS")) starts = n < SMALL_N ? std::max(1, atoi(e)) : 1;
  if (starts == 1)
    return leiden_core(ctx, n, d_indptr, d_indices, d_weights, resolution, n_iterations, seed, d_membership, h_modularity, h_n_comms, info);
  SB2_CUDA(cudaSetDevice(ctx->device));
  ScratchScope scr(ctx);
  int32_t* best;
  SB2_TRY(scr.alloc(&best, (size_t)n));
  double best_q = -1e300;
  int32_t best_nc = 0;
  sb2_leiden_info best_info{};
  for (int r = 0; r < starts; ++r) {
    double q = 0.0;
    int32_t nc = 0;
    sb2_leiden_info inf{};
    const uint64_t sr = r == 0 ? seed : seed * 0x9E3779B97F4A7C15ULL + 0xD1B54A32D192ED03ULL * (uint64_t)r;
    SB2_TRY(leiden_core(ctx, n, d_indptr, d_indices, d_weights, resolution, n_iterations, sr, d_membership, &q, &nc, &inf));
    if (q > best_q) {
      best_q = q; best_nc = nc; best_info = inf;
      SB2_CUDA(cudaMemcpyAsync(best, d_membership, sizeof(int32_t) * (size_t)n, cudaMemcpyDeviceToDevice, ctx->stream));
    }
  }
  SB2_CUDA(cudaMemcpyAsync(d_membership, best, sizeof(int32_t) * (size_t)n, cudaMemcpyDeviceToDevice, ctx->stream));
  SB2_CUDA(cudaStreamSynchronize(ctx->stream));
  *h_modularity = best_q;
  *h_n_comms = best_nc;
  if (info) *info = best_info;
  return SB2_OK;
}

// Louvain (Blondel et al. 2008) = the same local moving and aggregation without the refinement phase, one pass to its
// fixed point: what `louvain.find_partition(g, RBConfigurationVertexPartition, resolution_parameter, weights, seed)` and
// igraph's `community_multilevel` optimise (src/scanpy/tools/_louvain.py:150-176).  Same outputs as sb2_leiden_csr_f32.
extern "C" int32_t sb2_louvain_csr_f32(sb2_ctx* ctx, int64_t n, const int64_t* d_indptr, const int32_t* d_indices,
                                       const float* d_weights, double resolution, uint64_t seed, int32_t* d_membership,
                                       double* h_modularity, int32_t* h_n_comms, sb2_leiden_info* info) {
  SB2_CHECK_ARG(ctx && d_membership && h_modularity && h_n_comms, "null pointer");
  return leiden_core(ctx, n, d_indptr, d_indices, d_weights, resolution, 1, seed, d_membership, h_modularity, h_n_comms, info, true);
}
