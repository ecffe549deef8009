// te_footprint_polygon.cu — TraversabilityMap::traversabilityFootprint(double footprintYaw): the polygonal footprint sweep of
// one yaw, of a list of yaws, or reduced over a list of yaws, after the predicate pass of te_footprint.cu (run_predicates).
// Compiled with --fmad=false: grid_map::Polygon::isInside is replayed in the reference's operand order.
#include "te_fp_device.cuh"

#include <algorithm>
#include <cmath>
#include <cstring>

namespace te {
namespace {

// Polygonal footprint sweep: TraversabilityMap::traversabilityFootprint(double footprintYaw), TraversabilityMap.cpp:239-305, with the
// polygon isTraversable (:592-645).  Every cell gets the footprint polygon placed at its centre; the value is 0 when a cell of the
// polygon fails isTraversableForFilters, otherwise the mean of t' over the polygon's cells (traversabilityDefault_ when it covers
// none).  The set of cells inside the polygon is the same offset pattern for every centre EXCEPT for offsets whose cell centre lies
// on (within rounding of) an edge: grid_map::Polygon::isInside decides those on absolute double coordinates, differently from
// centre to centre.  The host classifies the offsets once per polygon (launch_footprint_polygon): certain-in cells become per-column
// runs that are summed from the tile's prefix sums; the few uncertain offsets are decided per centre with the reference's own
// arithmetic — cooperatively when the decision does not depend on the centre's row (an edge parallel to the x axis through cell
// centres: the YAML footprint at 0.02 m has 92 such offsets), 32 offsets per warp pass.  One launch sweeps a list of polygons (the
// footprint at several yaws): a block stages its tile once and sweeps a group of them.
constexpr int PTR = 64, PTC = 16;  // tile of centres: rows x columns
constexpr int PMAXV = 16;          // polygon vertices
constexpr int PB = 130;            // pitch of a staged blocked-count column (uint16)
// Eigen::Quaternion::toRotationMatrix of (cos(yaw/2), 0, 0, sin(yaw/2)), upper-left 2 x 2
struct Rot2 {
  double r00, r01, r10, r11;
};
// One polygon of a sweep: the footprint placed with rotation R, its slices of the call's run and uncertain-offset tables, and its
// output layer (map m's starts m * rows * out_ncols cells into `out`).
struct PolyDesc {
  Rot2 R;
  int run0, nruns;    // runs[run0 .. run0 + nruns)
  int fz0, nfz;       // fz[fz0 .. fz0 + nfz)
  int ncert;          // number of certain cells (sum of the run lengths)
  float* out;
};
struct PolyArgs {
  int Lp;             // reach of the polygon in cells (<= 31), the same at every rotation
  int npts;
  int npoly;          // polygons of the launch
  int group;          // polygons per block: blockIdx.x = g * row_tiles + row tile sweeps polygons g * group .. (g + 1) * group - 1
  int row_tiles;
  const PolyDesc* desc;  // [npoly]
  const int* runs;    // (dj & 0xff) | (lo & 0xff) << 8 | (hi & 0xff) << 16: rows i+lo .. i+hi of column j+dj are certainly inside
  const int* fz;      // (di & 0xff) | (dj & 0xff) << 8 | flags << 16: uncertain offsets, sorted by (dj, di); flag bit 0: the decision
                      // depends on the centre's row; bit 1: same column as the previous entry, next row, neither depends on the row
  // Reduce mode (k_poly_tile<true>; the descriptors' `out` is unused): per centre, the value of the first polygon of the block's
  // group that minimises it (worst), of the first that maximises it (best) and that polygon's index (best_yaw); each null when not
  // wanted.  Group g writes at g * rstride cells (0 without a split; a split leaves the folding to k_poly_combine).
  float* worst;
  float* best;
  int* best_yaw;
  size_t rstride;
  double px[PMAXV], py[PMAXV];
};

// grid_map::Polygon::isInside for the polygon placed at (cx, cy): vertices = R * p + centre in the operand order of Eigen's
// Transform * vector (oracle: teo_footprint_polygon), crossing-number test over (v[i], v[i-1]).
__device__ bool poly_inside_d(const PolyArgs& Q, const Rot2& R, double cx, double cy, double ptx, double pty) {
  int cross = 0;
  const int last = Q.npts - 1;
  double jx = cx + ((R.r00 * Q.px[last] + R.r01 * Q.py[last]) + 0.0);
  double jy = cy + ((R.r10 * Q.px[last] + R.r11 * Q.py[last]) + 0.0);
  for (int k = 0; k < Q.npts; ++k) {
    const double ix = cx + ((R.r00 * Q.px[k] + R.r01 * Q.py[k]) + 0.0);
    const double iy = cy + ((R.r10 * Q.px[k] + R.r11 * Q.py[k]) + 0.0);
    if (((iy > pty) != (jy > pty)) && (ptx < (jx - ix) * (pty - iy) / (jy - iy) + ix)) ++cross;
    jx = ix;
    jy = iy;
  }
  return (cross & 1) != 0;
}

// The tile geometry (PTR x PTC centres, staging origin r0 - Lp, c0 - Lp) is part of the results: a sum over a run is a difference
// of the staged prefix sums, whose float32 rounding depends on where the staged column starts.  kReduce: reduce over the block's
// polygons in registers instead of storing a layer per polygon (PolyArgs::worst / best / best_yaw).  kAt: map z sits at its own
// position and reads its coordinate tables at A.X + z * A.xs, A.Y + z * A.ys.  kMaps (Q.npoly = 2, the polygons of each map):
// map z sweeps its own pair of polygons, desc[0] and desc[map_poly[z]], into map slot slot[z] of their layers (slot null: z);
// device arrays of one entry per map, unused otherwise.  kInv: the default is NaN or infinite, so it cannot go into the prefix sums
// (every sum below a column's first invalid cell would be non-finite); invalid cells are staged as 0 and counted in the high byte
// of the blocked counts (at most NR <= 126 of each per column), and a footprint that holds one gives the default, as the
// reference's sum does.  A and Q are taken by value: k_poly_tile then compiles to the code it had as a kernel of its own (by
// reference it does not).
template <bool kReduce, bool kAt, bool kMaps, bool kInv>
__device__ __forceinline__ void poly_tile(FpArgs A, PolyArgs Q, const float* __restrict__ trav,
                                          const unsigned char* __restrict__ blocked, const int* __restrict__ map_poly,
                                          const int* __restrict__ slot) {
  extern __shared__ double sP[];  // [NC][PS] prefix sums of t'; then [NC][PB] uint16 prefix counts of blocked cells
  const int Lr = Q.Lp, NR = PTR + 2 * Lr, NC = PTC + 2 * Lr, PS = NR + 1;
  unsigned short* sB = reinterpret_cast<unsigned short*>(sP + (size_t)NC * PS);
  // map blockIdx.z of the batch: its input-buffer columns start mb columns into the batch's, its output columns mbo
  const int mb = (int)blockIdx.z * A.in_ncols, mbo = (kMaps && slot ? slot[blockIdx.z] : (int)blockIdx.z) * A.out_ncols;
  if constexpr (kAt) {  // the map's coordinate tables
    A.X += (size_t)blockIdx.z * A.xs;
    A.Y += (size_t)blockIdx.z * A.ys;
  }
  const int tile_r = (int)blockIdx.x % Q.row_tiles, p0 = ((int)blockIdx.x / Q.row_tiles) * Q.group, p1 = min(p0 + Q.group, Q.npoly);
  const int r0 = tile_r * PTR, c0 = A.out_col0 + (int)blockIdx.y * PTC;
  const int rb = r0 - Lr, cb = c0 - Lr;
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  // ---- phase 1: prefix sums of t' and of the blocked flags, one warp per staged column.  NR <= 4 * 32 (Lp <= 31): a lane takes
  //      four consecutive rows, scans them in registers, the warp scans the lane totals.  Cells outside the map or the slab's
  //      buffer contribute 0, so the sums need no clipping.
  int anyb = 0;
  for (int cc = warp; cc < NC; cc += 8) {
    const int gcol = cb + cc, lb = gcol - A.in_col0;
    const bool col_ok = gcol >= 0 && gcol < A.cols_total && lb >= 0 && lb < A.in_ncols;
    const float* tcol = trav + (size_t)(mb + (col_ok ? lb : 0)) * A.rows;
    const unsigned char* bcol = blocked + (size_t)(mb + (col_ok ? lb : 0)) * A.rows;
    double v[4];
    int cb4[4];
    unsigned bw = 0;
#pragma unroll
    for (int m = 0; m < 4; ++m) {
      const int k = 4 * lane + m, row = rb + k;
      v[m] = 0.0;
      cb4[m] = 0;
      if (k < NR && col_ok && row >= 0 && row < A.rows) {
        const float t = __ldg(tcol + row);
        if constexpr (kInv) {
          v[m] = finitef(t) ? (double)t : 0.0;
          cb4[m] = (bcol[row] != 0 ? 1 : 0) | (finitef(t) ? 0 : 256);
          bw |= (unsigned)(cb4[m] != 0) << (8 * m);
        } else {
          v[m] = finitef(t) ? (double)t : A.tdefault;
          cb4[m] = bcol[row] != 0 ? 1 : 0;
          bw |= (unsigned)cb4[m] << (8 * m);
        }
      }
    }
    anyb |= (int)bw;
    v[1] += v[0]; v[2] += v[1]; v[3] += v[2];
    cb4[1] += cb4[0]; cb4[2] += cb4[1]; cb4[3] += cb4[2];
    double tot = v[3];
    int ctot = cb4[3];
#pragma unroll
    for (int d = 1; d < 32; d <<= 1) {
      const double o = __shfl_up_sync(0xffffffffu, tot, d);
      const int oc = __shfl_up_sync(0xffffffffu, ctot, d);
      if (lane >= d) { tot += o; ctot += oc; }
    }
    double before = __shfl_up_sync(0xffffffffu, tot, 1);
    int cbefore = __shfl_up_sync(0xffffffffu, ctot, 1);
    if (lane == 0) { before = 0.0; cbefore = 0; }
    double* pcol = sP + (size_t)cc * PS;
    unsigned short* ccol = sB + (size_t)cc * PB;
    if (lane == 0) { pcol[0] = 0.0; ccol[0] = 0; }
#pragma unroll
    for (int m = 0; m < 4; ++m) {
      const int k = 4 * lane + m;
      if (k < NR) { pcol[k + 1] = before + v[m]; ccol[k + 1] = (unsigned short)(cbefore + cb4[m]); }
    }
  }
  const bool tile_any = __syncthreads_or(anyb) != 0;
  // ---- phase 2: a warp is 32 consecutive rows of one column at a time (4 columns per warp), each centre swept for every polygon
  //      of the block's group
  const int i = r0 + (warp & 1) * 32 + lane;
  const int i0 = i - lane;
  if (i0 >= A.rows) return;
  const bool active = i < A.rows;
  const int ic = active ? i : A.rows - 1;
  const double cx = A.X[ic];
  const int k0 = ic - rb;
  const int mpoly = kMaps ? map_poly[blockIdx.z] : 0;
  for (int q = 0; q < PTC / 4; ++q) {
    const int j = c0 + (warp >> 1) * (PTC / 4) + q;
    if (j >= A.out_col0 + A.out_ncols) break;
    const double cy = A.Y[j];
    // certain cells: per-column runs from the prefix sums (cells outside the map were staged as t' = 0, not blocked)
    const double* pbase = sP + (size_t)(j - cb) * PS + k0;
    const unsigned short* bbase = sB + (size_t)(j - cb) * PB + k0;
    const bool interior = ic - Lr >= 0 && ic + Lr < A.rows && j - Lr >= max(0, A.in_col0) && j + Lr <= min(A.cols_total, A.in_col0 + A.in_ncols) - 1;
    // reduce mode: every value is finite (the callers reject a non-finite traversability_default), so the infinities lose to the
    // first polygon, and strict comparisons keep the earliest polygon of a tie with its own bits (-0.0 and +0.0 included)
    float worst = __int_as_float(0x7f800000), best = __int_as_float(0xff800000);
    int best_y = p0;
    for (int y = p0; y < p1; ++y) {
      const PolyDesc& D = Q.desc[kMaps ? (y == 0 ? 0 : mpoly) : y];
      const Rot2 R = D.R;
      const int* const runs = Q.runs + D.run0;
      const int* const fz = Q.fz + D.fz0;
      const int nruns = D.nruns, nfz = D.nfz;
      double t = 0.0;
      int n = 0, nblk = 0;
      int ninv = 0;  // kInv: invalid cells in the footprint
      if (interior) {  // no clipping anywhere: the cell count is the table's
        for (int r = 0; r < nruns; ++r) {
          const int w = __ldg(runs + r);
          const int dj = (int)(signed char)(w & 0xff), lo = (int)(signed char)((w >> 8) & 0xff), hi = (int)(signed char)((w >> 16) & 0xff);
          const double* pc = pbase + dj * PS;
          t += pc[hi + 1] - pc[lo];
          if (tile_any) {
            const unsigned short* bc = bbase + dj * PB;
            if constexpr (kInv) {
              const int d = (int)bc[hi + 1] - (int)bc[lo];
              nblk += d & 0xff;
              ninv += d >> 8;
            } else {
              nblk += (int)bc[hi + 1] - (int)bc[lo];
            }
          }
        }
        n = D.ncert;
      } else {
        for (int r = 0; r < nruns; ++r) {
          const int w = __ldg(runs + r);
          const int dj = (int)(signed char)(w & 0xff), lo = (int)(signed char)((w >> 8) & 0xff), hi = (int)(signed char)((w >> 16) & 0xff);
          const int b = j + dj, lb = b - A.in_col0;
          if (b < 0 || b >= A.cols_total || lb < 0 || lb >= A.in_ncols) continue;
          const int a0 = max(ic + lo, 0), a1 = min(ic + hi, A.rows - 1);
          if (a0 > a1) continue;
          const double* pc = pbase + dj * PS;
          t += pc[hi + 1] - pc[lo];
          n += a1 - a0 + 1;
          if (tile_any) {
            const unsigned short* bc = bbase + dj * PB;
            if constexpr (kInv) {
              const int d = (int)bc[hi + 1] - (int)bc[lo];
              nblk += d & 0xff;
              ninv += d >> 8;
            } else {
              nblk += (int)bc[hi + 1] - (int)bc[lo];
            }
          }
        }
      }
      // uncertain offsets, 32 per pass: lane l decides offset base + l when the decision is the same for every row of the column; the
      // offsets that came out inside and follow each other down a column are then summed as ONE run from the prefix sums
      for (int base = 0; base < nfz; base += 32) {
        const int idx = base + lane;
        int w = 0;
        bool cand = false;
        if (idx < nfz) {
          w = __ldg(fz + idx);
          const int di = (int)(signed char)(w & 0xff), dj = (int)(signed char)((w >> 8) & 0xff);
          if ((w >> 16) & 1) {
            cand = true;  // depends on the row: every lane decides for itself below
          } else {
            const int a = ic + di, b = j + dj;
            // the decision does not depend on the row, so any row's coordinates will do — but they must exist
            const int ar = min(max(a, 0), A.rows - 1), icr = ar - di;
            if (b >= 0 && b < A.cols_total && icr >= 0 && icr < A.rows) cand = poly_inside_d(Q, R, A.X[icr], cy, A.X[ar], A.Y[b]);
          }
        }
        unsigned m = __ballot_sync(0xffffffffu, cand);
        const unsigned ext = m & __ballot_sync(0xffffffffu, ((w >> 17) & 1) != 0);  // inside AND continues its predecessor down the column
        while (m) {
          const int src = __ffs((int)m) - 1;
          const unsigned tail = src == 31 ? 0u : (ext >> (src + 1));
          const int len = __ffs((int)~tail) - 1;  // further entries of the run (0..31 - src)
          m &= ~((len >= 31 ? 0xffffffffu : ((2u << len) - 1u)) << src);
          const int wv = __shfl_sync(0xffffffffu, w, src);
          const int di = (int)(signed char)(wv & 0xff), dj = (int)(signed char)((wv >> 8) & 0xff);
          const int b = j + dj, lb = b - A.in_col0;
          if (b < 0 || b >= A.cols_total || lb < 0 || lb >= A.in_ncols) continue;
          const int a0 = ic + di, a1 = a0 + len;
          const int a0c = max(a0, 0), a1c = min(a1, A.rows - 1);
          if (a0c > a1c) continue;
          if (((wv >> 16) & 1) && !poly_inside_d(Q, R, cx, cy, A.X[a0], A.Y[b])) continue;  // row-dependent entries never chain (len == 0)
          const int cc = b - cb;
          const double* pc = sP + (size_t)cc * PS + (a0 - rb);
          t += pc[len + 1] - pc[0];
          n += a1c - a0c + 1;
          if (tile_any) {
            const unsigned short* bc = sB + (size_t)cc * PB + (a0 - rb);
            if constexpr (kInv) {
              const int d = (int)bc[len + 1] - (int)bc[0];
              nblk += d & 0xff;
              ninv += d >> 8;
            } else {
              nblk += (int)bc[len + 1] - (int)bc[0];
            }
          }
        }
      }
      float result;
      if (nblk > 0) result = 0.0f;                       // :297 / :301
      else if (n == 0) result = (float)A.tdefault;       // :625-628
      else if (kInv && ninv > 0) result = (float)A.tdefault;  // the sum holds a non-finite default
      else result = (float)(t / (double)n);              // :630
      if constexpr (kReduce) {
        if (result < worst) worst = result;
        if (result > best) { best = result; best_y = y; }
      } else {
        if (active) D.out[(size_t)(mbo + j - A.out_col0) * A.rows + i] = result;
      }
    }
    if constexpr (kReduce) {
      if (active) {
        const size_t o = (size_t)(p0 / Q.group) * Q.rstride + (size_t)(mbo + j - A.out_col0) * A.rows + i;
        if (Q.worst) Q.worst[o] = worst;
        if (Q.best) Q.best[o] = best;
        if (Q.best_yaw) Q.best_yaw[o] = best_y;
      }
    }
  }
}

template <bool kReduce>
__global__ void __launch_bounds__(256) k_poly_tile(FpArgs A, PolyArgs Q, const float* __restrict__ trav, const unsigned char* __restrict__ blocked) {
  poly_tile<kReduce, false, false, false>(A, Q, trav, blocked, nullptr, nullptr);
}

// k_poly_tile<false> for a NaN or infinite traversability_default (the reductions refuse one).
__global__ void __launch_bounds__(256) k_poly_tile_inv(FpArgs A, PolyArgs Q, const float* __restrict__ trav, const unsigned char* __restrict__ blocked) {
  poly_tile<false, false, false, true>(A, Q, trav, blocked, nullptr, nullptr);
}

// The polygon layers a te_map keeps (launch_footprint_polygon with PolygonMaps): every map of the launch sweeps the identity and
// its own yaw's rotation on its own coordinate tables (kAt) or on the shared ones.
template <bool kAt>
__global__ void __launch_bounds__(256) k_poly_tile_maps(FpArgs A, PolyArgs Q, const float* __restrict__ trav, const unsigned char* __restrict__ blocked,
                                                        const int* __restrict__ map_poly, const int* __restrict__ slot) {
  poly_tile<false, kAt, true, false>(A, Q, trav, blocked, map_poly, slot);
}

template <bool kAt>
__global__ void __launch_bounds__(256) k_poly_tile_maps_inv(FpArgs A, PolyArgs Q, const float* __restrict__ trav,
                                                            const unsigned char* __restrict__ blocked, const int* __restrict__ map_poly,
                                                            const int* __restrict__ slot) {
  poly_tile<false, kAt, true, true>(A, Q, trav, blocked, map_poly, slot);
}

// Reduce mode after a yaw-group split: k_poly_tile left group g's partial reduction at g * n cells of each scratch array (sw: worst,
// sb: best, sk: best_yaw; sb is there when best or best_yaw is wanted).  The groups are runs of consecutive polygons in order, so
// folding them in group order with the same strict comparisons gives the first minimum / maximum over all polygons.
__global__ void k_poly_combine(const float* __restrict__ sw, const float* __restrict__ sb, const int* __restrict__ sk, int ngroups, size_t n,
                               float* worst, float* best, int* best_yaw) {
  for (size_t c = (size_t)blockIdx.x * blockDim.x + threadIdx.x; c < n; c += (size_t)gridDim.x * blockDim.x) {
    if (worst) {
      float w = sw[c];
      for (int g = 1; g < ngroups; ++g) {
        const float v = sw[(size_t)g * n + c];
        if (v < w) w = v;
      }
      worst[c] = w;
    }
    if (sb) {
      float b = sb[c];
      int k = sk ? sk[c] : 0;
      for (int g = 1; g < ngroups; ++g) {
        const float v = sb[(size_t)g * n + c];
        if (v > b) { b = v; if (sk) k = sk[(size_t)g * n + c]; }
      }
      if (best) best[c] = b;
      if (best_yaw) best_yaw[c] = k;
    }
  }
}

}  // namespace

int polygon_reach(const te_geometry* g, int npts, const double* pts_xy) {
  double r = 0.0;
  for (int k = 0; k < npts; ++k) r = std::max(r, std::hypot(pts_xy[2 * k], pts_xy[2 * k + 1]));
  return (int)std::ceil(r / g->resolution) + 1;
}

int footprint_polygon_halo(const te_geometry* g, const te_footprint_params* p, int npts, const double* pts_xy) {
  const int walk = (int)std::ceil(p->max_gap_width / g->resolution) + 1;
  return polygon_reach(g, npts, pts_xy) + std::max(4, 3 + 1 + walk);
}

namespace {
// Offsets (di, dj) of the cells inside the polygon placed at a cell centre, relative to that centre: certain-in cells as runs per
// column offset, cells within `tol` of a comparison of grid_map::Polygon::isInside as the uncertain list.
struct PolyTables {
  std::vector<int> runs, fz;
};
//
// The reference compares absolute doubles: vertex v + c (rounded) against cell centre c' with c, c' cell centres of coordinates up
// to M = |position| + half length + reach; cu = ulp(M).  A centre is (B + res * (-idx)) rounded with B common to the map, so
// c' - c is the lattice offset plus at most 2 cu (two products, two sums), and placing the vertex adds half a cu:
//   - y comparison v.y > pt.y: moved by at most 2.5 cu.  tol = max(1e-7 res, 4 cu).
//   - x threshold thr = (vj.x - vi.x) (pt.y - vi.y) / (vj.y - vi.y) + vi.x against pt.x: the three differences carry 1, 2.5 and
//     1 cu; with s = (vj.x - vi.x) / (vj.y - vi.y) and (pt.y - vi.y) / (vj.y - vi.y) in [0, 1] on a straddling edge, the quotient
//     moves by (1 + 3.5 |s|) cu to first order; placing vi.x (0.5 cu), rounding the final sum (0.5 cu) and pt.x against the
//     centre (2 cu) add 3 cu: (4 + 3.5 |s|) cu in all.  tol_x = max(tol, 8 (1 + |s|) cu), twice that first-order bound, covers
//     the second-order terms (|vj.y - vi.y| >= 1e3 tol >= 4e3 cu, or the edge is uncertain anyway).
// Near the origin 1e-7 res is the larger term, so the tables are what they always were; far out (a UTM or LV95 map) more offsets
// become uncertain and are decided per centre.
bool classify_polygon(double res, double cu, int Lp, int npts, const double* px, const double* py, const double R[4], PolyTables* out,
                      std::string* why) {
  std::vector<double> vx(npts), vy(npts);
  for (int k = 0; k < npts; ++k) {
    vx[k] = (R[0] * px[k] + R[1] * py[k]) + 0.0;
    vy[k] = (R[2] * px[k] + R[3] * py[k]) + 0.0;
  }
  const double tol = std::max(1e-7 * res, 4.0 * cu);
  out->runs.clear();
  out->fz.clear();
  for (int dj = -Lp; dj <= Lp; ++dj) {
    int run_lo = 0;
    bool in_run = false;
    for (int di = -Lp; di <= Lp + 1; ++di) {
      bool inside = false, fuzzy = false, row_dep = false;
      if (di <= Lp) {
        // cell centre relative to the polygon's centre: X decreases with the row index, Y with the column index
        const double ptx = -res * (double)di, pty = -res * (double)dj;
        int cross = 0;
        for (int i = 0, j = npts - 1; i < npts; j = i++) {
          // equal y (bitwise; per centre both get the same centre coordinate added): (v[i].y > pt.y) == (v[j].y > pt.y) always
          if (vy[i] == vy[j]) continue;
          const bool ui = std::fabs(vy[i] - pty) < tol, uj = std::fabs(vy[j] - pty) < tol;
          if (ui || uj) fuzzy = true;  // (v.y > pt.y) may fall either way: depends on the column pair only
          const bool ci = vy[i] > pty, cj = vy[j] > pty;
          if ((ci != cj) || ui || uj) {
            const double thr = (vx[j] - vx[i]) * (pty - vy[i]) / (vy[j] - vy[i]) + vx[i];
            const double tol_x = std::max(tol, 8.0 * (1.0 + std::fabs((vx[j] - vx[i]) / (vy[j] - vy[i]))) * cu);
            // the x comparison involves the centre's row; so does a threshold that is a quotient of two rounding-sized numbers
            if (std::fabs(ptx - thr) < tol_x || std::fabs(vy[j] - vy[i]) < 1e3 * tol) { fuzzy = true; row_dep = true; }
            if ((ci != cj) && ptx < thr) ++cross;
          }
        }
        inside = (cross & 1) != 0;
      }
      if (fuzzy) {
        if (out->fz.size() >= 4096) { *why = "footprint polygon has more than 4096 cells on its outline"; return false; }
        int chain = 0;
        if (!row_dep && !out->fz.empty()) {
          const int pw = out->fz.back();
          if ((int)(signed char)((pw >> 8) & 0xff) == dj && (int)(signed char)(pw & 0xff) == di - 1 && ((pw >> 16) & 1) == 0) chain = 1;
        }
        out->fz.push_back((di & 0xff) | ((dj & 0xff) << 8) | ((row_dep ? 1 : 0) << 16) | (chain << 17));
        inside = false;
      }
      if (inside && !in_run) { in_run = true; run_lo = di; }
      if (!inside && in_run) {
        in_run = false;
        out->runs.push_back((dj & 0xff) | ((run_lo & 0xff) << 8) | (((di - 1) & 0xff) << 16));
      }
    }
  }
  return true;
}

// Eigen::Quaternion::toRotationMatrix of AngleAxisd(yaw, UnitZ) = (w, 0, 0, z) = (cos(yaw/2), 0, 0, sin(yaw/2)), upper-left 2 x 2,
// in Eigen's operation order.  Yaw 0 gives w = 1, z = 0 exactly: the identity that traversability_x uses.
Rot2 yaw_rotation(double yaw) {
  const double w = std::cos(0.5 * yaw), z = std::sin(0.5 * yaw);
  const double tz = 2.0 * z, twz = tz * w, tzz = tz * z;
  return Rot2{1.0 - (0.0 + tzz), 0.0 - twz, 0.0 + twz, 1.0 - (0.0 + tzz)};
}

// Yaw groups of a k_poly_tile launch: a block sweeps a group of consecutive polygons of its tile.  Tiles alone fill an H100 from
// 4 * sms of them (at the largest reach two blocks are resident per SM: two waves); fewer tiles split the polygons into as many
// groups as bring the launch to 4 * sms blocks, at most one per polygon.  A group restages its tile, so larger groups save
// staging; which block sweeps a layer never changes its bits.
int polygon_groups(long long tiles, int npoly, int sms) {
  const long long want = std::max(1LL, (4LL * sms + tiles - 1) / tiles);
  return (int)std::min<long long>(npoly, want);
}
}  // namespace

// traversabilityFootprint(yaw) for every layer of `polys`: predicates once, the polygon tables of every rotation in one upload,
// then one k_poly_tile launch for all of them (and, in reduce mode with yaw groups, one k_poly_combine), or with `maps` one
// k_poly_tile_maps launch for each map's pair.
int launch_footprint_polygon(FootprintState& st, const SlabView& v, const te_geometry* g, const te_footprint_params* p, int npts,
                             const double* pts_xy, int npoly, const PolygonLayer* polys, const PolygonReduce* reduce,
                             const PolygonMaps* maps, const float* trav, const float* slope, const float* step, const float* rough,
                             const float* elev, int nmaps, int sms, cudaStream_t s, int* launches) {
  if (npts < 3 || npts > PMAXV) { st.why = "footprint polygon needs 3 to 16 vertices"; return TE_ERR_UNSUPPORTED; }
  if (npoly < (maps ? 2 : 1)) { st.why = "no polygon layer to sweep"; return TE_ERR_UNSUPPORTED; }
  if (maps && reduce) { st.why = "per-map polygons have no reduction"; return TE_ERR_UNSUPPORTED; }
  if (reduce && !reduce->worst && !reduce->best && !reduce->best_yaw) { st.why = "no reduction output"; return TE_ERR_UNSUPPORTED; }
  if (reduce && !std::isfinite(p->traversability_default)) { st.why = "reduction with a non-finite traversability_default"; return TE_ERR_UNSUPPORTED; }
  const int Lp = polygon_reach(g, npts, pts_xy);
  if (Lp > 31) { st.why = "footprint polygon reaches further than 31 cells from its centre"; return TE_ERR_UNSUPPORTED; }
  PolyArgs q{};
  q.Lp = Lp; q.npts = npts; q.npoly = npoly;
  for (int k = 0; k < npts; ++k) { q.px[k] = pts_xy[2 * k]; q.py[k] = pts_xy[2 * k + 1]; }
  // the call's table: npoly descriptors, then the runs of every polygon, then their uncertain offsets
  std::vector<PolyDesc> desc(npoly);
  std::vector<int> runs, fz;
  {
    PolyTables tb;
    const double cu = coord_ulp(v.coord_max + Lp * g->resolution);
    for (int k = 0; k < npoly; ++k) {
      PolyDesc& d = desc[k];
      d.R = yaw_rotation(polys[k].yaw);
      const double R[4] = {d.R.r00, d.R.r01, d.R.r10, d.R.r11};
      if (!classify_polygon(g->resolution, cu, Lp, npts, q.px, q.py, R, &tb, &st.why)) return TE_ERR_UNSUPPORTED;
      d.run0 = (int)runs.size(); d.nruns = (int)tb.runs.size();
      d.fz0 = (int)fz.size(); d.nfz = (int)tb.fz.size();
      d.ncert = 0;
      for (int rw : tb.runs) d.ncert += (int)(signed char)((rw >> 16) & 0xff) - (int)(signed char)((rw >> 8) & 0xff) + 1;
      d.out = polys[k].out;
      runs.insert(runs.end(), tb.runs.begin(), tb.runs.end());
      fz.insert(fz.end(), tb.fz.begin(), tb.fz.end());
    }
  }
  // with per-map polygons, each map's polygon index follows the tables
  const size_t nmp = maps ? (size_t)nmaps : 0;
  const size_t dbytes = sizeof(PolyDesc) * desc.size(), bytes = dbytes + sizeof(int) * (runs.size() + fz.size() + nmp);
  std::vector<char> blob(bytes);
  std::memcpy(blob.data(), desc.data(), dbytes);
  if (!runs.empty()) std::memcpy(blob.data() + dbytes, runs.data(), sizeof(int) * runs.size());
  if (!fz.empty()) std::memcpy(blob.data() + dbytes + sizeof(int) * runs.size(), fz.data(), sizeof(int) * fz.size());
  if (maps) std::memcpy(blob.data() + dbytes + sizeof(int) * (runs.size() + fz.size()), maps->poly_of, sizeof(int) * nmp);
  FpArgs a{};
  if (int rc = run_predicates(st, v, g, p, nmaps, trav, slope, step, rough, elev, nullptr, nullptr, nullptr, sms, s, &a)) return rc;
  if (st.poly.p && st.poly.cap < bytes) cudaStreamSynchronize(s);  // kernels of an earlier call may still read the old tables
  if (st.poly.reserve(bytes) != cudaSuccess) { st.why = "allocating the polygon tables failed"; return TE_ERR_CUDA; }
  if (cudaMemcpyAsync(st.poly.p, blob.data(), bytes, cudaMemcpyHostToDevice, s) != cudaSuccess) { st.why = "polygon table upload failed"; return TE_ERR_CUDA; }
  q.desc = (const PolyDesc*)st.poly.p;
  q.runs = (const int*)((const char*)st.poly.p + dbytes);
  q.fz = q.runs + runs.size();
  if (maps) q.npoly = 2;  // per map: the identity and the map's own rotation
  const size_t smem = sizeof(double) * (size_t)(PTC + 2 * Lp) * (PTR + 2 * Lp + 1) + (size_t)(PTC + 2 * Lp) * (PB * 2);
  if (!st.poly_attr) {
    const size_t smax = sizeof(double) * (size_t)(PTC + 62) * (PTR + 63) + (size_t)(PTC + 62) * (PB * 2);
    if (cudaFuncSetAttribute(k_poly_tile<false>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smax) != cudaSuccess ||
        cudaFuncSetAttribute(k_poly_tile<true>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smax) != cudaSuccess ||
        cudaFuncSetAttribute(k_poly_tile_maps<false>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smax) != cudaSuccess ||
        cudaFuncSetAttribute(k_poly_tile_maps<true>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smax) != cudaSuccess ||
        cudaFuncSetAttribute(k_poly_tile_inv, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smax) != cudaSuccess ||
        cudaFuncSetAttribute(k_poly_tile_maps_inv<false>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smax) != cudaSuccess ||
        cudaFuncSetAttribute(k_poly_tile_maps_inv<true>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smax) != cudaSuccess) {
      st.why = "cudaFuncSetAttribute(max dynamic shared memory) failed"; return TE_ERR_CUDA;
    }
    st.poly_attr = true;
  }
  q.row_tiles = (v.rows + PTR - 1) / PTR;
  const int col_tiles = (v.out_ncols + PTC - 1) / PTC;
  const int ngroups = polygon_groups((long long)q.row_tiles * col_tiles * nmaps, q.npoly, sms);
  q.group = (q.npoly + ngroups - 1) / ngroups;
  const int nsplit = (q.npoly + q.group - 1) / q.group;  // groups actually launched
  const int nblocks_x = q.row_tiles * nsplit;
  const dim3 grid((unsigned)nblocks_x, (unsigned)col_tiles, (unsigned)nmaps);
  const bool inv = !std::isfinite(a.tdefault);  // the reductions refuse such a default (footprint_polygon_common)
  if (maps) {
    const auto kern = inv ? (a.pos ? k_poly_tile_maps_inv<true> : k_poly_tile_maps_inv<false>)
                          : (a.pos ? k_poly_tile_maps<true> : k_poly_tile_maps<false>);
    kern<<<grid, 256, smem, s>>>(a, q, trav, (const unsigned char*)st.block.p, q.fz + fz.size(), maps->slot);
    if (launches) *launches = 3;
    return 0;
  }
  if (!reduce) {
    (inv ? k_poly_tile_inv : k_poly_tile<false>)<<<grid, 256, smem, s>>>(a, q, trav, (const unsigned char*)st.block.p);
    if (launches) *launches = 3;
    return 0;
  }
  // Reduce mode.  Without a split the sweep writes the outputs.  With one, each group writes its partial results to st.reduce:
  // the split only happens below 4 * sms tiles, so that is under (4 * sms + tiles) * PTR * PTC cells per array.
  const size_t n = (size_t)nmaps * v.out_ncols * v.rows;
  if (nsplit == 1) {
    q.worst = reduce->worst; q.best = reduce->best; q.best_yaw = reduce->best_yaw;
    k_poly_tile<true><<<grid, 256, smem, s>>>(a, q, trav, (const unsigned char*)st.block.p);
    if (launches) *launches = 3;
    return 0;
  }
  const bool want_best = reduce->best || reduce->best_yaw;
  const size_t per = (size_t)nsplit * n, sbytes = sizeof(float) * per * ((reduce->worst ? 1 : 0) + (want_best ? 1 : 0) + (reduce->best_yaw ? 1 : 0));
  if (st.reduce.p && st.reduce.cap < sbytes) cudaStreamSynchronize(s);  // kernels of an earlier call may still use the old scratch
  if (st.reduce.reserve(sbytes) != cudaSuccess) { st.why = "allocating the reduction scratch failed"; return TE_ERR_CUDA; }
  float* next = (float*)st.reduce.p;
  if (reduce->worst) { q.worst = next; next += per; }
  if (want_best) { q.best = next; next += per; }
  if (reduce->best_yaw) q.best_yaw = (int*)next;
  q.rstride = n;
  k_poly_tile<true><<<grid, 256, smem, s>>>(a, q, trav, (const unsigned char*)st.block.p);
  const int cblocks = (int)std::min<size_t>((n + 255) / 256, (size_t)sms * 8);
  k_poly_combine<<<cblocks, 256, 0, s>>>(q.worst, q.best, q.best_yaw, nsplit, n, reduce->worst, reduce->best, reduce->best_yaw);
  if (launches) *launches = 4;
  return 0;
}

}  // namespace te
