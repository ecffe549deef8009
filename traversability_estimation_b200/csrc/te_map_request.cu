// te_map_request.cu — the te_map side of the footprint: the circular paths of a request answered on the map's persistent
// traversability_footprint cache (launch_map_request_device: work list, dedup, evaluation of every distinct circle, replay of the
// service loop, polygons), the merge of a fresh sweep into the cache (launch_map_merge) and the moves of selected maps between
// their slots and packed scratch (launch_map_slots).  Compiled with --fmad=false: the replay folds the reference's double sums.
#include "te_fp_device.cuh"

#include <cub/device/device_radix_sort.cuh>
#include <cub/device/device_scan.cuh>

#include <algorithm>
#include <cmath>
#include <type_traits>

namespace te {
namespace {

// ---------------------------------------------------------------------------------------------------------------------------
// The circular paths of a request on a te_map (launch_map_request_device).  The traversability_footprint cache there persists
// across the paths of a request and across requests, so which isTraversable calls run, and what they read, depends on what
// earlier calls stored.  Every circle the paths could check is a MapKey (one per distinct map, centre, cell, radius and polygon
// flag); k_map_eval_circles_dev evaluates every key on the cache as the request found it, one warp per key, and k_req_replay
// then runs the service loop in order over these records.  A te_map may hold a batch of maps of one geometry (map m's layers,
// cache and memo start m * rows * cols cells into theirs); a key belongs to one of them.
struct MapKey {
  double cx, cy, rmin;  // isTraversable(center, rmin + offset, cup, ..., rmin)
  int ci, cj;           // getIndex(center)
  int cup;              // computeUntraversablePolygon
  int map;              // the map of the batch (0 on a single map)
};
struct MapRecord {
  double t;       // the walk's traversability output (double), or the cached value
  float cache;    // what the walk stores at (ci, cj), or the cached value
  int state;      // 0: walked, traversable; 1: walked, untraversable; 2: the cell was cached when the request began
};

// Key k of the request, by the whole warp w of a block of four: its record (k_map_eval_circles_dev).
// AT: the maps sit at their own positions (FpArgs::pos), and the walk takes the key's map's tables and position.  Maps with
// parameters of their own (FpArgs::mp): the walk takes the key's map's.
template <bool AT, bool EACH>
__device__ __forceinline__ void map_eval_circle_d(const FpArgs& A0, const Layers& L, const PathArgs& P, const MapKey* __restrict__ keys,
                                                  int k, const float* __restrict__ cache, MapRecord* __restrict__ recs) {
  __shared__ Layers s_L[4];
  __shared__ PathArgs s_P[4];
  const int w = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const MapKey K = keys[k];
  FpArgs Am;
  if constexpr (AT || EACH) Am = map_view_d<AT, EACH>(A0, K.map);
  const FpArgs& A = AT || EACH ? Am : A0;
  MapRecord& R = recs[k];
  // The key's map: its layers, memo and cache start mo cells in.  The walk takes the shifted layer and path arguments from a
  // per-warp copy in shared memory (by reference, as it takes the kernel's own), so no register holds them across the call.
  const long long mo = (long long)K.map * A.rows * A.cols_total;
  const float c0 = __ldg(cache + mo + (size_t)K.cj * A.rows + K.ci);
  if (finitef(c0)) {  // :673-675
    if (lane == 0) { R.t = (double)c0; R.cache = c0; R.state = 2; }
    return;
  }
  if (lane == 0) {
    s_L[w] = shift_layers_d(L, mo);
    s_P[w] = P;
    s_P[w].memo += mo;
  }
  __syncwarp();
  const double rmax = K.rmin + map_walk_offset_d<EACH>(A0, P.offset, K.map);
  const int nr = (int)ceil(rmax / A.res);
  const FreshCircle f = fresh_circle_d(A, s_L[w], s_P[w], K.cx, K.cy, K.ci, K.cj, K.rmin, rmax, nr, K.cup != 0);
  if (lane == 0) { R.t = f.t; R.cache = f.cache; R.state = f.ok ? 0 : 1; }
}

// The key count is on the device (*nkeys), so the warps stride over the keys.  The polygons of the failed paths come after the
// replay (k_req_polygons).
template <bool AT, bool EACH>
__global__ void __launch_bounds__(128, 4) k_map_eval_circles_dev(FpArgs A, Layers L, PathArgs P, const MapKey* __restrict__ keys,
                                                              const unsigned long long* __restrict__ nkeys, const float* __restrict__ cache,
                                                              MapRecord* __restrict__ recs) {
  const long long n = (long long)*nkeys;
  for (long long k = (blockIdx.x * blockDim.x + threadIdx.x) >> 5; k < n; k += (gridDim.x * blockDim.x) >> 5)  // whole warps
    map_eval_circle_d<AT, EACH>(A, L, P, keys, (int)k, cache, recs);
}

// traversabilityFootprint(radius, offset) on a cache: a cached cell takes the memoised branch and keeps its value, every other cell
// gets the sweep's.  `out` (may be null or `cache` itself) receives the cache afterwards.  Block row y merges n cells: `fresh` and
// `out` from y * n on, the cache from slot[y] * n on (slot null: y * n).
__global__ void __launch_bounds__(256) k_map_merge(float* cache, const float* __restrict__ fresh, float* out, size_t n,
                                                   const int* __restrict__ slot) {
  const size_t y = blockIdx.y;
  cache += (slot ? (size_t)slot[y] : y) * n;
  fresh += y * n;
  if (out) out += y * n;
  for (size_t c = (size_t)blockIdx.x * blockDim.x + threadIdx.x; c < n; c += (size_t)gridDim.x * blockDim.x) {
    const float v = finitef(cache[c]) ? cache[c] : fresh[c];
    cache[c] = v;
    if (out) out[c] = v;
  }
}

// Selected maps between their slots of a te_map and packed scratch (launch_map_slots).  PUT: layer l of packed map j goes to
// dst[l] + slot[j] * cells, the cache / memo slots of the map are emptied (NaN bits 0xffffffff, memo 0: not evaluated) and its
// slots of the fill layers take fill_bits.  Not PUT: src[l] + slot[j] * cells goes to packed map j of dst[l].  V cells per thread
// and access (V = 4: 16-byte accesses).
template <bool PUT, int V>
__global__ void __launch_bounds__(256) k_map_slots(MapSlots a) {
  using Vec = typename std::conditional<V == 4, float4, float>::type;
  using Bytes = typename std::conditional<V == 4, unsigned, unsigned char>::type;
  const size_t step = (size_t)gridDim.x * blockDim.x * V;
  for (int j = blockIdx.y; j < a.nsel; j += gridDim.y) {
    const size_t packed = (size_t)j * a.cells, resident = (size_t)(a.slot ? a.slot[j] : j) * a.cells;
    const size_t s0 = PUT ? packed : resident, d0 = PUT ? resident : packed;
    for (size_t c = ((size_t)blockIdx.x * blockDim.x + threadIdx.x) * V; c < a.cells; c += step) {
#pragma unroll
      for (int l = 0; l < kMapSlotLayers; ++l)
        if (a.dst[l]) *reinterpret_cast<Vec*>(a.dst[l] + d0 + c) = __ldg(reinterpret_cast<const Vec*>(a.src[l] + s0 + c));
      if (PUT) {
        const float nan = __int_as_float(-1), f = __uint_as_float(a.fill_bits);
        Vec e, v;
        if constexpr (V == 4) {
          e = make_float4(nan, nan, nan, nan);
          v = make_float4(f, f, f, f);
        } else {
          e = nan;
          v = f;
        }
        if (a.cache) *reinterpret_cast<Vec*>(a.cache + resident + c) = e;
        if (a.memo) *reinterpret_cast<Bytes*>(a.memo + resident + c) = 0;
#pragma unroll
        for (int l = 0; l < kMapSlotLayers; ++l)
          if (a.fill[l]) *reinterpret_cast<Vec*>(a.fill[l] + resident + c) = v;
      }
    }
  }
}

// ---------------------------------------------------------------------------------------------------------------------------
// The work list of the circular paths of a request on a te_map (launch_map_request_device), whichever memory the request came
// from.  It holds one entry per isTraversable call a circular path could make (a single pose; every fourth LineIterator cell of an
// in-map segment) and a "gate" wherever the service loop breaks without a check (a failed checkInclination, a segment with an end
// outside the map).  The list is laid out per map, each map's entries contiguous and in request order (k_req_count ..
// k_req_list); the key entries are deduplicated on their key's bits (k_req_dedup) and every distinct key is walked once on the
// cache as the request found it (k_map_eval_circles_dev); k_req_replay then runs the service loop, one warp per map, and
// k_req_polygons publishes the polygons of the failed paths.
enum : int { kEntKey = 1, kEntOutside = 2, kEntGate = 4, kEntSegEnd = 8, kEntPathEnd = 16 };
struct ReqEntry {
  double cx, cy;  // the centre: a segment cell's centre, a single pose's position
  int q;          // the path
  int flags;      // kEnt*: a key (an in-map centre), a single pose outside the map, or a gate; the last of its segment / path
  int ci, cj;     // getIndex(centre) (kEntKey)
  int seg;        // segment k (1 .. n-1) of the path; 0: a single pose
  int freps;      // a failing segment cell's polygon is hulled into the path's this often (:407-412)
  int map;        // the path's map
  int key;        // k_req_dedup: the canonical entry of a key entry (the first to claim the hash slot)
};
// The failing circle of a replayed path: 0 none, 1 fromCircle(fx, fy), 2 the blocked cells of key `key` (k_req_polygons).
struct ReqFail {
  double fx, fy;
  int fkind, key, freps, pad;
};
constexpr unsigned short kReqNoMap = 0xffff;  // sort key of a pose without entries (maps are 0 .. 65534)
// CUB sorts short arrays with one single-tile kernel and longer ones with several: the sort always runs over at least this many
// keys (the poses, then kReqNoMap), so that a request launches the same kernels whatever its pose count.
constexpr int kReqSortMin = 1 << 16;
struct DevReq {
  int npaths, nposes, nmaps;
  int nsort;                    // keys sorted: max(nposes, kReqSortMin)
  long long map_cells, max_checks;
  const int* path_begin;
  const double* poses;          // 7 doubles per pose
  const double* radius;
  const int* fp_begin;
  const int* path_map;          // nullptr: one map
  const unsigned char* cup;
  const float* rslope;          // robot_slope of map 0, nullptr: no checkInclination
  double offset;                // the call's; FpArgs::mp: each map's own
  unsigned char* is_safe;
  double* trav_out;
  double* area_out;
  UntravOut O;                  // O.count nullptr: no polygons
  // workspace (launch_map_request_device)
  unsigned char* status;        // per path: 0 polygonal, 1 replayed, 2 not checked, 3 empty circular path, 4 cut by max_checks
  long long* cnt;               // per pose (+1): entries
  long long* gofs;              // their exclusive scan in request order
  unsigned short* pkey;         // per pose: the sort key (the map, kReqNoMap)
  int* pidx;                    // per pose: its index
  unsigned short* skey;         // sorted
  int* order;                   // poses sorted stably by map
  int* lcnt;                    // entries of the sorted poses (+1)
  int* lofs;                    // their exclusive scan: the list offsets
  int* map_range;               // per map: [first, last) sorted pose index (0, 0: no entries)
  ReqEntry* entries;            // max_checks
  int* kid;                     // per entry: the key id of a canonical key entry
  int* table;                   // hash table of entry index + 1, tmask + 1 slots
  unsigned tmask;
  MapKey* keys;                 // max_checks
  MapRecord* recs;
  ReqFail* fails;               // per path
  unsigned long long* counters; // candidates, keys, stored
  // host memory: a non-finite x or y is checked as the service loop checks it (a single pose outside the map, a segment gate)
  // instead of leaving its path unchecked; only k_req_paths reads it (last, so the other kernels' parameters keep their offsets)
  bool nonfinite_ok;
};

// The path of pose p: the last q with path_begin[q] <= p (k_check_polygon_items' search).
__device__ __forceinline__ int req_path_of_d(const DevReq& D, int p) {
  int lo = 0, hi = D.npaths - 1;
  while (lo < hi) {
    const int mid = (lo + hi + 1) >> 1;
    if (D.path_begin[mid] <= p) lo = mid; else hi = mid - 1;
  }
  return lo;
}

__device__ __forceinline__ bool req_circular_d(const DevReq& D, int q) { return D.fp_begin[q + 1] == D.fp_begin[q]; }

// One thread per path: whether circular path q can be checked (radius, rings, pose range, finite positions unless
// D.nonfinite_ok, map) and every pose of it is found by req_path_of_d.
__global__ void __launch_bounds__(128) k_req_paths(FpArgs A, DevReq D) {
  const int q = blockIdx.x * blockDim.x + threadIdx.x;
  if (q >= D.npaths) return;
  if (!req_circular_d(D, q)) { D.status[q] = 0; return; }
  const int b = D.path_begin[q], n = D.path_begin[q + 1] - b;
  const double rmin = D.radius[q];
  const int m = D.path_map ? D.path_map[q] : 0;
  bool ok = m >= 0 && m < D.nmaps;
  const double offset = ok && A.mp ? A.mp[m].offset : D.offset;  // the map's own with FpArgs::mp
  ok = ok && rmin >= 0.0 && ceil((rmin + offset) / A.res) <= (double)kPathMaxRings && b >= 0 && n >= 0 && b <= D.nposes - n;
  for (int k = 0; k < n && ok; ++k)
    ok = (D.nonfinite_ok || (isfinite(D.poses[7 * (size_t)(b + k)]) && isfinite(D.poses[7 * (size_t)(b + k) + 1]))) &&
         req_path_of_d(D, b + k) == q;
  D.status[q] = !ok ? 2 : n == 0 ? 3 : 1;
}

// The entries pose p of a replayed path adds, written to E when E is not null (at most max_checks - off of them).  Returns their
// count.  Request order: a failed inclination's gate first, then the pose's circle (a single pose) or the segment's cells.
// AT: the maps sit at their own positions, and the path's map's tables and position apply.
template <bool AT>
__device__ long long req_pose_entries_d(const FpArgs& A0, const DevReq& D, int p, ReqEntry* E, long long room) {
  const int q = req_path_of_d(D, p);
  if (D.status[q] != 1) return 0;
  const int b = D.path_begin[q], n = D.path_begin[q + 1] - b, k = p - b;
  // poses before the first path or after the last belong to no path; the search gives them path 0 or npaths - 1
  if (!(k >= 0 && k < n) || (n > 1 && k == 0)) return 0;
  const int m = D.path_map ? D.path_map[q] : 0;
  FpArgs Am;
  if constexpr (AT) Am = map_args_d(A0, m);
  const FpArgs& A = AT ? Am : A0;
  const float* rslope = D.rslope ? D.rslope + m * D.map_cells : nullptr;
  const double ex = D.poses[7 * (size_t)p], ey = D.poses[7 * (size_t)p + 1];
  const double sx = n > 1 ? D.poses[7 * (size_t)(p - 1)] : ex, sy = n > 1 ? D.poses[7 * (size_t)(p - 1) + 1] : ey;
  const int last = (p == b + n - 1) ? kEntPathEnd : 0;
  long long c = 0;
  auto put = [&](double cx, double cy, int flags, int ci, int cj, int freps) {
    if (E && c < room) E[c] = ReqEntry{cx, cy, q, flags, ci, cj, n > 1 ? k : 0, freps, m, -1};
    ++c;
  };
  // the candidates count a check's circles whatever checkInclination says: the gate goes in front of them
  if (rslope && !inclination_ok_d(A, rslope, sx, sy, ex, ey)) put(ex, ey, kEntGate, 0, 0, 1);
  if (n == 1) {
    int i, j;
    if (get_index_d(A, ex, ey, i, j)) put(ex, ey, kEntKey | last, i, j, 1);
    else put(ex, ey, kEntOutside | last, 0, 0, 1);
    return c;
  }
  int si, sj, ei, ej;
  if (!get_index_d(A, sx, sy, si, sj) || !get_index_d(A, ex, ey, ei, ej)) {
    put(ex, ey, kEntGate | last, 0, 0, 1);
    return c;
  }
  LineD line(ei, ej, si, sj);
  const int nchk = (line.n + 3) / 4;
  if (!E) return c + nchk;
  for (int cc = 0; cc < line.n && c < room; ++cc, line.next()) {
    if (cc & 3) continue;
    const int flags = kEntKey | (cc / 4 == nchk - 1 ? kEntSegEnd | last : 0);
    put(A.X[line.li], A.Y[line.lj], flags, line.li, line.lj, (line.n - 1) / 4 - cc / 4 + 1);
  }
  return c;
}

// 1. Count: one thread per pose index (and one more for the scan's total).
template <bool AT>
__global__ void __launch_bounds__(128) k_req_count(FpArgs A, DevReq D) {
  const int p = blockIdx.x * blockDim.x + threadIdx.x;
  if (p > D.nposes) return;
  D.cnt[p] = p < D.nposes ? req_pose_entries_d<AT>(A, D, p, nullptr, 0) : 0;
}

// One thread per path after the scan: the capacity cut (a replayed or empty circular path whose entries end past max_checks, and
// so every later one), and the outputs of every circular path the replay does not answer.
__global__ void __launch_bounds__(128) k_req_cut(DevReq D) {
  const int q = blockIdx.x * blockDim.x + threadIdx.x;
  if (q >= D.npaths) return;
  int s = D.status[q];
  if ((s == 1 || s == 3) && D.gofs[D.path_begin[q + 1]] > D.max_checks) D.status[q] = s = 4;
  if (s == 0 || s == 1) return;
  const bool cup = D.cup != nullptr && D.cup[q] != 0;
  const bool checked = s == 3;  // an empty path: ok = n > 0 is false (:330-334)
  D.is_safe[q] = 0;
  D.trav_out[q] = checked ? 0.0 : nan("");
  D.area_out[q] = checked ? 0.0 : nan("");
  if (D.O.count) D.O.count[q] = (checked || !cup) ? 0 : -1;
}

// One thread per pose: the sort key (the pose's map, kReqNoMap without entries) and the pose index.
__global__ void __launch_bounds__(128) k_req_keys(DevReq D) {
  const int p = blockIdx.x * blockDim.x + threadIdx.x;
  if (p >= D.nsort) return;
  bool has = p < D.nposes && D.cnt[p] > 0;  // the padding sorts last
  int m = 0;
  if (has) {
    const int q = req_path_of_d(D, p);
    has = D.status[q] == 1;
    m = D.path_map ? D.path_map[q] : 0;
  }
  D.pkey[p] = has ? (unsigned short)m : kReqNoMap;
  D.pidx[p] = p;
}

// One thread per sorted pose index (and one more): its entry count, and the first / last sorted index of each map.
__global__ void __launch_bounds__(128) k_req_sorted(DevReq D) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i > D.nposes) return;
  const unsigned short m = i < D.nposes ? D.skey[i] : kReqNoMap;
  D.lcnt[i] = m != kReqNoMap ? (int)D.cnt[D.order[i]] : 0;
  if (m == kReqNoMap) return;
  if (i == 0 || D.skey[i - 1] != m) D.map_range[2 * m] = i;
  if (i == D.nposes - 1 || D.skey[i + 1] != m) D.map_range[2 * m + 1] = i + 1;
}

// 2. List: one thread per sorted pose index writes its entries at its offset.
template <bool AT>
__global__ void __launch_bounds__(128) k_req_list(FpArgs A, DevReq D) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= D.nposes || D.skey[i] == kReqNoMap) return;
  const int off = D.lofs[i];
  req_pose_entries_d<AT>(A, D, D.order[i], D.entries + off, D.max_checks - off);
}

__device__ __forceinline__ unsigned long long dbits_d(double d) { return (unsigned long long)__double_as_longlong(d); }

// The identity of a key entry's isTraversable call: map, centre, cell, radius and polygon flag, bit for bit.
__device__ __forceinline__ bool req_same_key_d(const DevReq& D, const ReqEntry& a, const ReqEntry& b) {
  const bool ca = D.cup && D.cup[a.q], cb = D.cup && D.cup[b.q];
  return a.map == b.map && dbits_d(a.cx) == dbits_d(b.cx) && dbits_d(a.cy) == dbits_d(b.cy) && a.ci == b.ci && a.cj == b.cj &&
         dbits_d(D.radius[a.q]) == dbits_d(D.radius[b.q]) && ca == cb;
}

// 3. Dedup: the threads stride over the entries.  A key entry claims its key's slot of an open-addressing table (linear probing); the entry that
// claims it is the key's canonical entry and allocates the key's id and MapKey, every other entry with that key records the
// canonical entry.  Which entry wins a slot varies from run to run; the key and its record do not.
__device__ __forceinline__ void req_dedup_entry_d(const DevReq& D, int e) {
  const ReqEntry E = D.entries[e];
  if (!(E.flags & kEntKey)) return;
  const bool cup = D.cup && D.cup[E.q];
  const double rmin = D.radius[E.q];
  unsigned long long h = dbits_d(E.cx) * 0x9E3779B97F4A7C15ULL;
  h = (h ^ (h >> 29)) + dbits_d(E.cy) * 0xBF58476D1CE4E5B9ULL;
  h = (h ^ (h >> 31)) + dbits_d(rmin) * 0x94D049BB133111EBULL;
  h ^= ((unsigned long long)(unsigned)E.ci << 33) ^ ((unsigned long long)(unsigned)E.cj << 1) ^ (unsigned long long)cup;
  h += (unsigned long long)(unsigned)E.map * 0xD6E8FEB86659FD93ULL;
  unsigned slot = (unsigned)(h ^ (h >> 32)) & D.tmask;
  int canon = -1;
  for (;;) {
    int s = D.table[slot];
    if (s == 0) {
      s = atomicCAS(D.table + slot, 0, e + 1);
      if (s == 0) { canon = e; break; }
    }
    if (req_same_key_d(D, D.entries[s - 1], E)) { canon = s - 1; break; }
    slot = (slot + 1) & D.tmask;
  }
  D.entries[e].key = canon;
  atomicAdd(D.counters + 0, 1ULL);  // candidates
  if (canon == e) {
    const int id = (int)atomicAdd(D.counters + 1, 1ULL);  // distinct keys
    D.kid[e] = id;
    D.keys[id] = MapKey{E.cx, E.cy, rmin, E.ci, E.cj, cup ? 1 : 0, E.map};
  }
}

__global__ void __launch_bounds__(256) k_req_dedup(DevReq D) {
  const int total = D.lofs[D.nposes];
  for (int e = blockIdx.x * blockDim.x + threadIdx.x; e < total; e += gridDim.x * blockDim.x) req_dedup_entry_d(D, e);
}

// 5. Replay: the service loop of one map, one warp per map, over the map's entries in request order, 32 at a time.  Why this is
// the sequential loop (one check after the other, as the reference runs it) exactly:
//   - Which value a check reads depends only on the checks before it in its map: in the sequential loop a cell holds the float of
//     the last executed earlier check of the request that walked it, or what it held when the request began.  The live cache
//     holds exactly those.  A check walks iff its cell is not finite (:673, isValid): empty, or holding a NaN or an infinity that
//     a walk stored (an invalid cell under a non-finite traversability_default, an infinite ring factor at offset 0).  Such a
//     cell was empty or non-finite when the request began, so every key at it has a walk as its record.
//   - Within a window every lane assumes that all lanes before it run.  At a cell whose live value is finite every lane reads it.
//     At any other cell a lane walks (its own record) iff every earlier lane of that cell walked and stored a non-finite float;
//     otherwise it reads the first finite float stored before it.  So under that assumption each lane's value and verdict are
//     the sequential loop's.
//   - The assumption holds up to and including the first failing lane f: no lane before it fails, and entries of one path are
//     consecutive, so the sequential loop runs lanes 0 .. f in this order.  They commit: a cell keeps the float of its last
//     committed walk, and one lane folds the values in visit order, so sums, add_segment_d and the verdicts are the sequential
//     loop's bit for bit.  Every committed walk counts as a store, so under a non-finite value `stored` can exceed the keys.
//   - The sequential loop then skips the rest of f's path (the `break`s); the next window starts at the first entry of a later
//     path.  Lanes after f that belong to later paths are evaluated again there: their assumption included dropped lanes, which
//     store nothing.
//   - Gates fail without a polygon, as the loop's `break`.  Maps share nothing, so their warps run independently.
// REC: walked_keys[kid] = 1 for every key whose walk commits (k_req_record).
template <bool REC>
__device__ __forceinline__ void req_replay_d(const FpArgs& A, const DevReq& D, float* cache, unsigned char* walked_keys) {
  __shared__ double s_t[4][32];
  __shared__ int s_v[4][32];
  const int w = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int m = (int)((blockIdx.x * blockDim.x + threadIdx.x) >> 5);
  if (m >= D.nmaps) return;  // whole warp
  const int lo = D.map_range[2 * m], hi = D.map_range[2 * m + 1];
  if (lo >= hi) return;  // a map without circular paths
  int e0 = D.lofs[lo];
  const int e1 = D.lofs[hi];
  float* const mc = cache + m * D.map_cells;
  const double tdefault = A.mp ? A.mp[m].tdefault : A.tdefault;  // the map's own with FpArgs::mp
  // lane 0: the path being folded
  int cur = -1, dead = -1, nLine = 0;
  bool ok = false;
  double result = 0.0, lengthPath = 0.0, sum = 0.0;
  ReqFail F{};
  unsigned long long stored = 0;
  while (e0 < e1) {
    const int e = e0 + lane;
    const bool have = e < e1;
    ReqEntry E{};
    if (have) E = D.entries[e];
    // the dropped rest of a failed path is a prefix of the window
    const unsigned dmask = __ballot_sync(0xffffffffu, have && E.q == dead);
    if (dmask & 1u) {
      e0 += (~dmask) ? __ffs((int)~dmask) - 1 : 32;
      continue;
    }
    const bool key = have && (E.flags & kEntKey);
    const unsigned long long cell = key ? (unsigned long long)E.cj * A.rows + E.ci : ~0ULL - lane;
    const unsigned peers = __match_any_sync(0xffffffffu, cell);
    float live = 0.0f, rcache = 0.0f;
    MapRecord R{};
    if (key) {
      live = mc[cell];
      R = D.recs[D.kid[E.key]];
      rcache = R.cache;
    }
    // the lanes before this one at its cell whose float is finite: the first of them is the first finite store before this lane
    const unsigned fin = peers & __ballot_sync(0xffffffffu, finitef(rcache)) & ((1u << lane) - 1u);
    const float first_cache = __shfl_sync(0xffffffffu, rcache, fin ? __ffs((int)fin) - 1 : lane);
    const bool walk = key && fin == 0 && !finitef(live);
    double t = 0.0;
    bool lok = true;
    int fk = 0;  // the lane's polygon kind if it fails
    if (key) {
      if (walk) { t = R.t; lok = R.state == 0; fk = 2; }  // :679-736
      else {                                              // :673-678
        const float v = finitef(live) ? live : first_cache;
        t = (double)v; lok = v != 0.0f; fk = 1;
      }
    } else if (have && (E.flags & kEntOutside)) {         // :662-667
      t = tdefault; lok = tdefault != 0.0; fk = 1;
    } else if (have) {                                    // a gate
      lok = false;
    }
    const unsigned fails = __ballot_sync(0xffffffffu, have && !lok);
    const int f = fails ? __ffs((int)fails) - 1 : 32;
    const int nhave = __popc(__ballot_sync(0xffffffffu, have));
    const int ncommit = min(f + 1, nhave);
    const bool commit_walk = walk && lane < ncommit;
    const unsigned walked = __ballot_sync(0xffffffffu, commit_walk);
    // the cell keeps the float of its last committed walk
    if (commit_walk && !(walked & peers & ~((2u << lane) - 1u))) mc[cell] = R.cache;
    if constexpr (REC)
      if (commit_walk) walked_keys[D.kid[E.key]] = 1;
    stored += __popc(walked);
    s_t[w][lane] = t;
    s_v[w][lane] = (lok ? 1 : 0) | (fk << 1);
    __syncwarp();
    if (lane == 0) {
      for (int l = 0; l < ncommit; ++l) {
        const ReqEntry G = D.entries[e0 + l];
        const double tl = s_t[w][l];
        const bool okl = s_v[w][l] & 1;
        if (G.q != cur) {  // a new path: :345-362
          cur = G.q; ok = true; result = 0.0; lengthPath = 0.0; sum = 0.0; nLine = 0;
          F = ReqFail{0.0, 0.0, 0, -1, 1, 0};
        }
        if (G.flags & kEntGate) {
          ok = false;  // :365-367, :389-396: break without a polygon
        } else if (G.seg == 0) {  // :365-387
          result = tl;
          ok = okl;
        } else {  // :398-452
          sum += tl;
          ++nLine;
          if (!okl) {
            ok = false;
            F.freps = G.freps;
          } else if (G.flags & kEntSegEnd) {
            const int b = D.path_begin[G.q];
            const double* pe = D.poses + 7 * (size_t)(b + G.seg);
            const double* ps = pe - 7;
            add_segment_d(sum / (double)nLine, pe[0] - ps[0], pe[1] - ps[1], G.seg, lengthPath, result);
            sum = 0.0;
            nLine = 0;
          }
        }
        if (!okl && !(G.flags & kEntGate)) {
          F.fkind = s_v[w][l] >> 1; F.fx = G.cx; F.fy = G.cy;
          F.key = F.fkind == 2 ? D.kid[G.key] : -1;
        }
        if (!ok || (G.flags & kEntPathEnd)) {  // the path's answer (:458-461)
          const int q = G.q;
          D.is_safe[q] = ok ? 1 : 0;
          D.trav_out[q] = ok ? result : 0.0;
          D.area_out[q] = 0.0;
          const bool cup = D.cup != nullptr && D.cup[q] != 0;
          if (!cup || ok || F.fkind == 0) F.fkind = 0;
          if (D.O.count && F.fkind == 0) D.O.count[q] = 0;
          D.fails[q] = F;
          if (!ok) dead = q;
          cur = -1;
        }
      }
    }
    dead = __shfl_sync(0xffffffffu, dead, 0);
    e0 += (f < nhave) ? f + 1 : nhave;
    __syncwarp();
  }
  if (lane == 0 && stored) atomicAdd(D.counters + 2, stored);
}

__global__ void __launch_bounds__(128) k_req_replay(FpArgs A, DevReq D, float* cache) { req_replay_d<false>(A, D, cache, nullptr); }

__global__ void __launch_bounds__(128) k_req_replay_rec(FpArgs A, DevReq D, float* cache, unsigned char* walked_keys) {
  req_replay_d<true>(A, D, cache, walked_keys);
}

// 7. Recording (a te_map's slope_footprint / step_footprint / roughness_footprint, `plane`): every key whose walk the replay
// committed walks its spiral again, one warp per key, and records the cells the reference's walk visits (record_circle_d).  A
// committed walk ran on an empty centre, so its visits are those of a walk on an empty cache.  Maps as k_map_eval_circles_dev.
template <bool AT, bool EACH>
__global__ void __launch_bounds__(128) k_req_record(FpArgs A0, Layers L, PathArgs P, const MapKey* __restrict__ keys,
                                                    const unsigned long long* __restrict__ nkeys,
                                                    const unsigned char* __restrict__ walked_keys, unsigned char* plane) {
  const long long n = (long long)*nkeys;
  for (long long k = (blockIdx.x * blockDim.x + threadIdx.x) >> 5; k < n; k += (gridDim.x * blockDim.x) >> 5) {  // whole warps
    if (!walked_keys[k]) continue;
    const MapKey K = keys[k];
    FpArgs Am;
    if constexpr (AT || EACH) Am = map_view_d<AT, EACH>(A0, K.map);
    const FpArgs& A = AT || EACH ? Am : A0;
    const long long mo = (long long)K.map * A.rows * A.cols_total;
    const double rmax = K.rmin + map_walk_offset_d<EACH>(A0, P.offset, K.map);
    record_circle_d(A, shift_layers_d(L, mo), P, plane + mo, P.memo + mo, K.cx, K.cy, K.ci, K.cj, K.rmin, rmax, (int)ceil(rmax / A.res), K.cup != 0);
  }
}

// 6. Polygons: one warp per path; a path the replay did not leave a failing circle to publish exits at once.  The pair
// k_check_paths_fresh_poly calls: fromCircle, or spiral_blockers_d on the failing key and write_cells_polygon_d with its freps.
template <bool AT, bool EACH>
__global__ void __launch_bounds__(128, 4) k_req_polygons(FpArgs A0, Layers L, PathArgs P, DevReq D, CircleTable C) {
  __shared__ int s_min[4][kFreshTableRows + 1], s_max[4][kFreshTableRows + 1];
  __shared__ int2 s_stack[4][2 * kFreshTableRows + 4];
  __shared__ int2 s_first[4][3];
  const int w = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int q = (int)((blockIdx.x * blockDim.x + threadIdx.x) >> 5);
  if (q >= D.npaths || D.status[q] != 1) return;  // whole warp
  const ReqFail F = D.fails[q];
  if (F.fkind == 0) return;
  const double rmax = D.radius[q] + map_walk_offset_d<EACH>(A0, D.offset, D.path_map ? D.path_map[q] : 0);
  const UntravScratch S{s_min[w], s_max[w], s_stack[w], s_first[w]};
  if (F.fkind == 1) {
    const int n = D.path_begin[q + 1] - D.path_begin[q];
    if (lane == 0) write_circle_polygon_d(C.cs, C.sn, F.fx, F.fy, rmax, n > 1, reinterpret_cast<double2*>(S.stack), D.O, q);
    return;
  }
  const MapKey K = D.keys[F.key];
  FpArgs Am;  // the key's map's tables and position (AT) and parameters (EACH)
  if constexpr (AT || EACH) Am = map_view_d<AT, EACH>(A0, K.map);
  const FpArgs& A = AT || EACH ? Am : A0;
  const long long mo = (long long)K.map * D.map_cells;
  L = shift_layers_d(L, mo);
  P.memo += mo;
  const int nr = (int)ceil(rmax / A.res);
  const int cnt = spiral_blockers_d(A, L, P, S, K.cx, K.cy, K.ci, K.cj, K.rmin, rmax, nr);
  if (lane == 0) write_cells_polygon_d(A, S, 2 * nr + 1, K.ci - nr, cnt, F.freps, D.O, q);
}

size_t align16(size_t b) { return (b + 15) / 16 * 16; }

// te_map_clear_footprint (resetTraversabilityFootprintLayers, TraversabilityMap.cpp:195-200): slope_footprint and step_footprint
// become NaN, roughness_footprint stays.
__global__ void __launch_bounds__(256) k_plane_clear(unsigned char* plane, size_t n) {
  for (size_t c = (size_t)blockIdx.x * blockDim.x + threadIdx.x; c < n; c += (size_t)gridDim.x * blockDim.x) plane[c] &= 0x30;
}

// Layer `field` (0 slope_footprint, 1 step_footprint, 2 roughness_footprint) of the recorded bytes as floats: the quiet NaN
// 0x7fc00000 the reference's layers hold where nothing wrote them (computeTraversability's add(), the bag's slope_footprint and
// step_footprint), 0.0f or 1.0f.
__global__ void __launch_bounds__(256) k_plane_decode(const unsigned char* __restrict__ plane, int field, float* __restrict__ out, size_t n) {
  for (size_t c = (size_t)blockIdx.x * blockDim.x + threadIdx.x; c < n; c += (size_t)gridDim.x * blockDim.x) {
    const unsigned f = (__ldg(plane + c) >> (2 * field)) & 3u;
    out[c] = f == 0u ? __int_as_float(0x7fc00000) : f == 1u ? 0.0f : 1.0f;
  }
}

unsigned plane_blocks(size_t n, int sms) { return (unsigned)std::max<size_t>(std::min<size_t>((n + 255) / 256, (size_t)sms * 8), 1); }

}  // namespace

void launch_plane_clear(unsigned char* plane, size_t n, int sms, cudaStream_t s) {
  k_plane_clear<<<plane_blocks(n, sms), 256, 0, s>>>(plane, n);
}

void launch_plane_decode(const unsigned char* plane, int field, float* out, size_t n, int sms, cudaStream_t s) {
  k_plane_decode<<<plane_blocks(n, sms), 256, 0, s>>>(plane, field, out, n);
}

int launch_map_request_device(FootprintState& st, const SlabView& v, const te_geometry* g, const te_footprint_params* p,
                              const PathChecks& r, float* cache, long long max_checks, bool nonfinite_ok, int sms, cudaStream_t s,
                              int* launches) {
  *launches = 0;
  const int npaths = r.npaths, nposes = r.nposes, nmaps = r.nmaps;
  if (nmaps < 1 || (!r.path_map && nmaps != 1)) { st.why = "a batch of maps needs a map per path"; return TE_ERR_BAD_ARG; }
  if (int rc = ensure_ring_table(st, s)) return rc;
  // the workspace: per path, per pose, per map, per entry (max_checks), the hash table and CUB's scratch
  const size_t np1 = (size_t)nposes + 1, nc = (size_t)std::max(max_checks, 1LL);
  const int nsort = std::max(nposes, kReqSortMin);
  unsigned tslots = 32;
  while (tslots < 2 * nc) tslots *= 2;
  size_t cub_scan1 = 0, cub_sort = 0, cub_scan2 = 0;
  if (cub::DeviceScan::ExclusiveSum(nullptr, cub_scan1, (const long long*)nullptr, (long long*)nullptr, (int)np1, s) != cudaSuccess ||
      cub::DeviceRadixSort::SortPairs(nullptr, cub_sort, (const unsigned short*)nullptr, (unsigned short*)nullptr, (const int*)nullptr,
                                      (int*)nullptr, nsort, 0, 16, s) != cudaSuccess ||
      cub::DeviceScan::ExclusiveSum(nullptr, cub_scan2, (const int*)nullptr, (int*)nullptr, (int)np1, s) != cudaSuccess) {
    st.why = "sizing the scan / sort scratch failed";
    return TE_ERR_CUDA;
  }
  const size_t cub_bytes = std::max(cub_scan1, std::max(cub_sort, cub_scan2));
  size_t off = 0;
  auto take = [&](size_t bytes) { const size_t o = off; off = align16(off + bytes); return o; };
  const size_t o_counters = take(4 * sizeof(unsigned long long)), o_range = take(2 * sizeof(int) * (size_t)nmaps);
  const size_t o_status = take((size_t)npaths), o_fails = take(sizeof(ReqFail) * (size_t)npaths);
  const size_t o_cnt = take(sizeof(long long) * np1), o_gofs = take(sizeof(long long) * np1);
  const size_t o_pkey = take(sizeof(unsigned short) * nsort), o_skey = take(sizeof(unsigned short) * nsort);
  const size_t o_pidx = take(sizeof(int) * nsort), o_order = take(sizeof(int) * nsort);
  const size_t o_lcnt = take(sizeof(int) * np1), o_lofs = take(sizeof(int) * np1);
  const size_t o_entries = take(sizeof(ReqEntry) * nc), o_kid = take(sizeof(int) * nc), o_keys = take(sizeof(MapKey) * nc);
  const size_t o_recs = take(sizeof(MapRecord) * nc), o_table = take(sizeof(int) * (size_t)tslots), o_cub = take(cub_bytes);
  const size_t o_walked = r.plane ? take(nc) : off;
  if (st.devreq.reserve(off) != cudaSuccess) { st.why = "allocating the device request workspace failed"; return TE_ERR_CUDA; }
  char* base = (char*)st.devreq.p;
  DevReq D{};
  D.npaths = npaths; D.nposes = nposes; D.nmaps = nmaps; D.nsort = nsort;
  D.map_cells = (long long)g->rows * g->cols; D.max_checks = max_checks;
  D.path_begin = r.path_begin; D.poses = r.poses; D.radius = r.radius; D.fp_begin = r.footprint_begin; D.path_map = r.path_map;
  D.cup = r.cup; D.rslope = r.robot_slope; D.offset = p->offset;
  D.is_safe = r.is_safe; D.trav_out = r.trav_out; D.area_out = r.area_out; D.O = UntravOut{r.max_vertices, r.ucount, r.uxy};
  D.status = (unsigned char*)(base + o_status); D.fails = (ReqFail*)(base + o_fails);
  D.cnt = (long long*)(base + o_cnt); D.gofs = (long long*)(base + o_gofs);
  D.pkey = (unsigned short*)(base + o_pkey); D.skey = (unsigned short*)(base + o_skey);
  D.pidx = (int*)(base + o_pidx); D.order = (int*)(base + o_order); D.lcnt = (int*)(base + o_lcnt); D.lofs = (int*)(base + o_lofs);
  D.map_range = (int*)(base + o_range); D.entries = (ReqEntry*)(base + o_entries); D.kid = (int*)(base + o_kid);
  D.table = (int*)(base + o_table); D.tmask = tslots - 1; D.keys = (MapKey*)(base + o_keys); D.recs = (MapRecord*)(base + o_recs);
  D.counters = (unsigned long long*)(base + o_counters);
  D.nonfinite_ok = nonfinite_ok;
  st.req_counters = D.counters;
  void* tmp = base + o_cub;
  if (cudaMemsetAsync(base + o_counters, 0, o_status - o_counters, s) != cudaSuccess ||  // counters and map ranges
      cudaMemsetAsync(D.table, 0, sizeof(int) * (size_t)tslots, s) != cudaSuccess) {
    st.why = "clearing the device request workspace failed";
    return TE_ERR_CUDA;
  }
  FpArgs a = filter_args(v, g, p, r.rough);
  a.mp = r.map_params;
  const Layers L{r.trav, r.slope, r.step, r.elev, r.rough};
  const PathArgs P = path_args(st, p, r.robot_slope);
  auto blocks = [](long long n, int per) { return (unsigned)std::max((n + per - 1) / per, 1LL); };
  size_t b1 = cub_bytes, b2 = cub_bytes, b3 = cub_bytes;
  k_req_paths<<<blocks(npaths, 128), 128, 0, s>>>(a, D);
  const bool at = a.pos != nullptr;  // maps at their own positions: the instantiations that read each map's tables
  const bool each = a.mp != nullptr;  // maps with parameters of their own: the instantiations that read each map's
  if (at) k_req_count<true><<<blocks(nposes + 1, 128), 128, 0, s>>>(a, D);
  else k_req_count<false><<<blocks(nposes + 1, 128), 128, 0, s>>>(a, D);
  cudaError_t e = cub::DeviceScan::ExclusiveSum(tmp, b1, (const long long*)D.cnt, D.gofs, (int)np1, s);
  k_req_cut<<<blocks(npaths, 128), 128, 0, s>>>(D);
  k_req_keys<<<blocks(nsort, 128), 128, 0, s>>>(D);
  if (e == cudaSuccess)
    e = cub::DeviceRadixSort::SortPairs(tmp, b2, (const unsigned short*)D.pkey, D.skey, (const int*)D.pidx, D.order, nsort, 0, 16, s);
  k_req_sorted<<<blocks(nposes + 1, 128), 128, 0, s>>>(D);
  if (e == cudaSuccess) e = cub::DeviceScan::ExclusiveSum(tmp, b3, (const int*)D.lcnt, D.lofs, (int)np1, s);
  if (at) k_req_list<true><<<blocks(nposes, 128), 128, 0, s>>>(a, D);
  else k_req_list<false><<<blocks(nposes, 128), 128, 0, s>>>(a, D);
  k_req_dedup<<<(unsigned)std::min<long long>(blocks((long long)nc, 256), 8LL * sms), 256, 0, s>>>(D);
  const unsigned ge = (unsigned)std::min<long long>(blocks((long long)nc, 4), 16LL * sms);
  const auto eval = at ? (each ? k_map_eval_circles_dev<true, true> : k_map_eval_circles_dev<true, false>)
                       : (each ? k_map_eval_circles_dev<false, true> : k_map_eval_circles_dev<false, false>);
  eval<<<ge, 128, 0, s>>>(a, L, P, D.keys, D.counters + 1, cache, D.recs);
  *launches = 12;  // nine kernels and three CUB calls, each counted as one launch (a CUB call runs two or more kernels)
  if (!r.plane) {
    k_req_replay<<<blocks(nmaps, 4), 128, 0, s>>>(a, D, cache);
  } else {  // a te_map's recorded layers: which keys' walks commit, then their visits
    unsigned char* const walked = (unsigned char*)base + o_walked;
    if (e == cudaSuccess) e = cudaMemsetAsync(walked, 0, nc, s);
    k_req_replay_rec<<<blocks(nmaps, 4), 128, 0, s>>>(a, D, cache, walked);
    const auto rec = at ? (each ? k_req_record<true, true> : k_req_record<true, false>)
                        : (each ? k_req_record<false, true> : k_req_record<false, false>);
    rec<<<ge, 128, 0, s>>>(a, L, P, D.keys, D.counters + 1, walked, r.plane);
    *launches += 2;
  }
  if (r.ucount) {
    const auto polys = at ? (each ? k_req_polygons<true, true> : k_req_polygons<true, false>)
                          : (each ? k_req_polygons<false, true> : k_req_polygons<false, false>);
    polys<<<blocks(npaths, 4), 128, 0, s>>>(a, L, P, D, circle_table());
    ++*launches;
  }
  if (e != cudaSuccess) { st.why = std::string("scan / sort failed: ") + cudaGetErrorString(e); return TE_ERR_CUDA; }
  return 0;
}

int launch_map_merge(const float* fresh, float* cache, float* out, size_t n, const int* slot, int nsel, int sms, cudaStream_t s) {
  const long long per_map = std::max<long long>((long long)sms * 8 / nsel, 1);
  const long long blocks = std::min<long long>((long long)((n + 255) / 256), per_map);
  k_map_merge<<<dim3((unsigned)std::max(blocks, 1LL), (unsigned)nsel), 256, 0, s>>>(cache, fresh, out, n, slot);
  return 0;
}

void launch_map_slots(const MapSlots& a, bool put, int sms, cudaStream_t s) {
  // 16-byte accesses when every map slot and every layer starts on a 16-byte boundary
  bool vec = a.cells % 4 == 0 && (reinterpret_cast<uintptr_t>(a.cache) & 15u) == 0;
  for (int l = 0; l < kMapSlotLayers; ++l)
    vec = vec && ((reinterpret_cast<uintptr_t>(a.src[l]) | reinterpret_cast<uintptr_t>(a.dst[l]) | reinterpret_cast<uintptr_t>(a.fill[l])) &
                  15u) == 0;
  const int V = vec ? 4 : 1;
  const long long per_map = std::max<long long>((long long)sms * 8 / a.nsel, 1);
  const long long bx = std::max(std::min<long long>((long long)((a.cells / V + 255) / 256), per_map), 1LL);
  const dim3 grid((unsigned)bx, (unsigned)std::min(a.nsel, 65535));
  if (put) {
    if (vec) k_map_slots<true, 4><<<grid, 256, 0, s>>>(a);
    else k_map_slots<true, 1><<<grid, 256, 0, s>>>(a);
  } else {
    if (vec) k_map_slots<false, 4><<<grid, 256, 0, s>>>(a);
    else k_map_slots<false, 1><<<grid, 256, 0, s>>>(a);
  }
}

}  // namespace te
