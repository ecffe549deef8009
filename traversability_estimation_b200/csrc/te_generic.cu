// te_generic.cu — the "literal" kernels: every cell is computed with the reference's own operand
// order in IEEE double (this translation unit is compiled with --fmad=false so no multiply-add is
// contracted).  They serve three purposes:
//   1. TE_KERNEL_GENERIC: any window radius / resolution / algorithm, no shape specialisation;
//   2. the certified slow path of the fused stencil (te_fused.cu appends the few cells whose fp32
//      result cannot be certified to a work list that k_fixup_cells recomputes here);
//   3. the stand-alone filter entry points (te_normals / te_step / te_roughness / te_slope).
//
// Reference arithmetic restated (paths relative to the reference repository):
//   normals   grid_map::NormalVectorsFilter area method (robot_filter_parameter.yaml:3-9)
//   slope     traversability_estimation_filters/src/SlopeFilter.cpp:59-89
//   step      traversability_estimation_filters/src/StepFilter.cpp:102-182
//   roughness traversability_estimation_filters/src/RoughnessFilter.cpp:73-132
//   fuse      grid_map::MathExpressionFilter (robot_filter_parameter.yaml:29-33)
#include <algorithm>
#include <cstdint>

#include "te_device.cuh"
#include "te_kernels.h"

namespace te {
namespace {

struct ElevAccess {
  const float* __restrict__ e;
  int rows, col0, ncols, cols_total;
  // Value at global cell (a, b); NaN when outside the map, outside the slab, or not finite.
  __device__ __forceinline__ float operator()(int a, int b) const {
    if (a < 0 || a >= rows || b < 0 || b >= cols_total) return nanf_();
    const int lb = b - col0;
    if (lb < 0 || lb >= ncols) return nanf_();
    const float v = __ldg(e + (size_t)lb * rows + a);
    return finitef(v) ? v : nanf_();
  }
};

// CircleIterator membership (grid_map_core CircleIterator::isInside): squared distance of the two
// cell centres in double, inclusive.
template <class F>
__device__ __forceinline__ void for_circle(const SlabView& v, int i, int j, double r2, int R, F&& f) {
  const int a0 = max(0, i - R), a1 = min(v.rows - 1, i + R);
  const int b0 = max(0, j - R), b1 = min(v.cols_total - 1, j + R);
  const double cx = v.X[i], cy = v.Y[j];
  // not unrolled: a literal cell runs this loop nest a dozen times with different bodies, and the code of one cell is executed
  // once — compact loops keep it inside the instruction cache (the tier-3 kernel is bound by instruction fetch otherwise)
#pragma unroll 1
  for (int a = a0; a <= a1; ++a) {
    const double dx = v.X[a] - cx;
    const double dx2 = dx * dx;
#pragma unroll 1
    for (int b = b0; b <= b1; ++b) {
      const double dy = v.Y[b] - cy;
      if (dx2 + dy * dy <= r2) f(a, b);
    }
  }
}

// Rank of a 3x3 as Eigen::FullPivHouseholderQR reports it with its default threshold.
__device__ int qr_rank3(const double cov[3][3]) {
  double m[3][3];
  for (int r = 0; r < 3; ++r)
    for (int c = 0; c < 3; ++c) m[r][c] = cov[r][c];
  const double eps = 2.220446049250313e-16;
  const double precision = eps * 3.0;
  double biggest = 0.0, maxpivot = 0.0;
  int nonzero = 3;
  double diag[3] = {0.0, 0.0, 0.0};
  for (int k = 0; k < 3; ++k) {
    int pr = k, pc = k;
    double big = -1.0;
    for (int c = k; c < 3; ++c)
      for (int r = k; r < 3; ++r) {
        const double a = fabs(m[r][c]);
        if (a > big) { big = a; pr = r; pc = c; }
      }
    if (k == 0) biggest = big;
    if (fabs(big) <= fabs(biggest) * precision) { nonzero = k; break; }
    if (pr != k)
      for (int c = 0; c < 3; ++c) { const double t = m[k][c]; m[k][c] = m[pr][c]; m[pr][c] = t; }
    if (pc != k)
      for (int r = 0; r < 3; ++r) { const double t = m[r][k]; m[r][k] = m[r][pc]; m[r][pc] = t; }
    double tail2 = 0.0;
    for (int r = k + 1; r < 3; ++r) tail2 += m[r][k] * m[r][k];
    const double c0 = m[k][k];
    double beta, tau;
    double ess[3] = {0.0, 0.0, 0.0};
    if (tail2 <= 2.2250738585072014e-308) {
      tau = 0.0;
      beta = c0;
    } else {
      beta = sqrt(c0 * c0 + tail2);
      if (c0 >= 0.0) beta = -beta;
      for (int r = k + 1; r < 3; ++r) ess[r] = m[r][k] / (c0 - beta);
      tau = (beta - c0) / beta;
    }
    m[k][k] = beta;
    diag[k] = beta;
    if (fabs(beta) > maxpivot) maxpivot = fabs(beta);
    for (int c = k + 1; c < 3; ++c) {
      double tmp = m[k][c];
      for (int r = k + 1; r < 3; ++r) tmp += ess[r] * m[r][c];
      m[k][c] -= tau * tmp;
      for (int r = k + 1; r < 3; ++r) m[r][c] -= tau * ess[r] * tmp;
    }
  }
  const double threshold = maxpivot * (eps * 3.0);
  int rank = 0;
  for (int k = 0; k < nonzero; ++k)
    if (fabs(diag[k]) > threshold) ++rank;
  return rank;
}

// Cyclic Jacobi on a symmetric 3x3 in double; returns eigenvalues and unit eigenvectors (columns).
__device__ void jacobi3(const double ain[3][3], double eval[3], double evec[3][3]) {
  double a[3][3];
  for (int r = 0; r < 3; ++r)
    for (int c = 0; c < 3; ++c) { a[r][c] = ain[r][c]; evec[r][c] = (r == c) ? 1.0 : 0.0; }
  for (int sweep = 0; sweep < 64; ++sweep) {
    const double off = fabs(a[0][1]) + fabs(a[0][2]) + fabs(a[1][2]);
    if (off == 0.0) break;
#pragma unroll
    for (int p = 0; p < 2; ++p)
#pragma unroll
      for (int q = p + 1; q < 3; ++q) {
        const double apq = a[p][q];
        if (apq == 0.0) continue;
        const double g = 100.0 * fabs(apq);
        if (sweep > 3 && fabs(a[p][p]) + g == fabs(a[p][p]) && fabs(a[q][q]) + g == fabs(a[q][q])) {
          a[p][q] = a[q][p] = 0.0;
          continue;
        }
        const double h = a[q][q] - a[p][p];
        double t;
        if (fabs(h) + g == fabs(h)) {
          t = apq / h;
        } else {
          const double theta = 0.5 * h / apq;
          t = 1.0 / (fabs(theta) + sqrt(theta * theta + 1.0));
          if (theta < 0.0) t = -t;
        }
        const double c = 1.0 / sqrt(t * t + 1.0), s = t * c;
#pragma unroll
        for (int k = 0; k < 3; ++k) {
          const double akp = a[k][p], akq = a[k][q];
          a[k][p] = c * akp - s * akq;
          a[k][q] = s * akp + c * akq;
        }
#pragma unroll
        for (int k = 0; k < 3; ++k) {
          const double apk = a[p][k], aqk = a[q][k];
          a[p][k] = c * apk - s * aqk;
          a[q][k] = s * apk + c * aqk;
        }
        a[p][q] = a[q][p] = 0.0;
#pragma unroll
        for (int k = 0; k < 3; ++k) {
          const double vkp = evec[k][p], vkq = evec[k][q];
          evec[k][p] = c * vkp - s * vkq;
          evec[k][q] = s * vkp + c * vkq;
        }
      }
  }
  for (int k = 0; k < 3; ++k) eval[k] = a[k][k];
}

// NormalVectorsFilter area method at one cell whose elevation is finite.
template <class Acc>
__device__ void normal_literal(const SlabView& v, const ChainDev& p, const Acc& E, int i, int j, double n[3]) {
  n[0] = 0.0; n[1] = 0.0; n[2] = 1.0;
  if (p.alg == 0) {
    double sx = 0.0, sy = 0.0, sz = 0.0;
    int cnt = 0;
    for_circle(v, i, j, p.rn2, p.Rn, [&](int a, int b) {
      const float z = E(a, b);
      if (!finitef(z)) return;
      sx += v.X[a]; sy += v.Y[b]; sz += (double)z;
      ++cnt;
    });
    const double mx = sx / (double)cnt, my = sy / (double)cnt, mz = sz / (double)cnt;
    double cov[3][3] = {{0.0, 0.0, 0.0}, {0.0, 0.0, 0.0}, {0.0, 0.0, 0.0}};
    for_circle(v, i, j, p.rn2, p.Rn, [&](int a, int b) {
      const float z = E(a, b);
      if (!finitef(z)) return;
      const double d0 = v.X[a] - mx, d1 = v.Y[b] - my, d2 = (double)z - mz;
      cov[0][0] += d0 * d0; cov[0][1] += d0 * d1; cov[0][2] += d0 * d2;
      cov[1][1] += d1 * d1; cov[1][2] += d1 * d2; cov[2][2] += d2 * d2;
    });
    cov[1][0] = cov[0][1]; cov[2][0] = cov[0][2]; cov[2][1] = cov[1][2];
    if (qr_rank3(cov) >= 3) {
      double eval[3], evec[3][3];
      jacobi3(cov, eval, evec);
      int s = 0;
      double sv = 1.7976931348623157e308;
      for (int k = 0; k < 3; ++k)
        if (eval[k] < sv) { sv = eval[k]; s = k; }
      n[0] = evec[0][s]; n[1] = evec[1][s]; n[2] = evec[2][s];
    }
  } else {
    double s[3] = {0.0, 0.0, 0.0};
    double ss[3][3] = {{0.0, 0.0, 0.0}, {0.0, 0.0, 0.0}, {0.0, 0.0, 0.0}};
    int cnt = 0;
    for_circle(v, i, j, p.rn2, p.Rn, [&](int a, int b) {
      const float z = E(a, b);
      if (!finitef(z)) return;
      const double d[3] = {v.X[a], v.Y[b], (double)z};
      for (int r = 0; r < 3; ++r) {
        s[r] += d[r];
        for (int c = 0; c < 3; ++c) ss[r][c] += d[r] * d[c];
      }
      ++cnt;
    });
    if (cnt >= 3) {
      double cov[3][3];
      for (int r = 0; r < 3; ++r)
        for (int c = 0; c < 3; ++c) cov[r][c] = ss[r][c] / (double)cnt - (s[r] / (double)cnt) * (s[c] / (double)cnt);
      double eval[3], evec[3][3];
      jacobi3(cov, eval, evec);
      int lo = 0;
      for (int k = 1; k < 3; ++k)
        if (eval[k] < eval[lo]) lo = k;
      // second smallest eigenvalue
      double mid = 1.7976931348623157e308;
      for (int k = 0; k < 3; ++k)
        if (k != lo && eval[k] < mid) mid = eval[k];
      if (mid > 1e-8) { n[0] = evec[0][lo]; n[1] = evec[1][lo]; n[2] = evec[2][lo]; }
    }
  }
  const double along = p.axis == 0 ? n[0] : (p.axis == 1 ? n[1] : n[2]);
  if (along < 0.0) { n[0] = -n[0]; n[1] = -n[1]; n[2] = -n[2]; }
}

__device__ __forceinline__ float slope_literal(float nz, double crit) {
  if (!finitef(nz)) return nanf_();
  const double s = acos((double)nz);
  return (float)(s < crit ? 1.0 - s / crit : 0.0);
}

__device__ float step_height_literal(const SlabView& v, const ChainDev& p, const ElevAccess& E, int i, int j) {
  if (!finitef(E(i, j))) return nanf_();
  bool init = false;
  double hmax = 0.0, hmin = 0.0;
  for_circle(v, i, j, p.r1sq, p.R1, [&](int a, int b) {
    const float z = E(a, b);
    if (!finitef(z)) return;
    const double h = (double)z;
    if (!init) { hmax = hmin = h; init = true; return; }
    if (h > hmax) hmax = h;
    if (h < hmin) hmin = h;
  });
  return init ? (float)(hmax - hmin) : nanf_();
}

__device__ float step_literal(const SlabView& v, const ChainDev& p, const ElevAccess& E, int i, int j) {
  int nCells = 0;
  double stepMax = 0.0;
  bool any = false;
  for_circle(v, i, j, p.r2sq, p.R2, [&](int a, int b) {
    const float sh = step_height_literal(v, p, E, a, b);
    if (!finitef(sh)) return;
    any = true;
    if ((double)sh > stepMax) stepMax = (double)sh;
    if ((double)sh > p.step_crit) ++nCells;
  });
  if (!any) return nanf_();
  const double step = fmin(stepMax, (double)nCells / (double)p.ncrit * stepMax);
  return (float)(step < p.step_crit ? 1.0 - step / p.step_crit : 0.0);
}

template <class Acc>
__device__ float roughness_literal(const SlabView& v, const ChainDev& p, const Acc& E, int i, int j,
                                   float fnx, float fny, float fnz) {
  if (!finitef(fnx)) return nanf_();
  double sx = 0.0, sy = 0.0, sz = 0.0;
  unsigned long long cnt = 0;
  for_circle(v, i, j, p.rr2, p.Rr, [&](int a, int b) {
    const float z = E(a, b);
    if (!finitef(z)) return;
    sx += v.X[a]; sy += v.Y[b]; sz += (double)z;
    ++cnt;
  });
  const double mx = sx / (double)cnt, my = sy / (double)cnt, mz = sz / (double)cnt;
  const double nx = fnx, ny = fny, nz = fnz;
  const double plane = mx * nx + my * ny + mz * nz;
  double sum = 0.0;
  for_circle(v, i, j, p.rr2, p.Rr, [&](int a, int b) {
    const float z = E(a, b);
    if (!finitef(z)) return;
    const double d = nx * v.X[a] + ny * v.Y[b] + nz * (double)z - plane;
    sum += d * d;
  });
  const double rough = sqrt(sum / (double)(cnt - 1ull));  // cnt == 1 -> 0/0 -> NaN -> 0.0 below
  return (float)(rough < p.rough_crit ? 1.0 - rough / p.rough_crit : 0.0);
}

// The 7 x 7 neighbourhood of one cell fetched up front (49 independent loads) so that the literal arithmetic of a
// lone fix-up cell is not a chain of dependent memory latencies.
struct ElevWindow {
  float z[7][7];
  int i0, j0;
  __device__ __forceinline__ void fill(const ElevAccess& E, int i, int j) {
    i0 = i - 3;
    j0 = j - 3;
#pragma unroll
    for (int b = 0; b < 7; ++b)
#pragma unroll
      for (int a = 0; a < 7; ++a) z[b][a] = E(i0 + a, j0 + b);
  }
  __device__ __forceinline__ float operator()(int a, int b) const {  // dynamic index: the array lives in (L1-cached) local memory
    const unsigned da = (unsigned)(a - i0), db = (unsigned)(b - j0);
    return (da < 7u && db < 7u) ? z[db][da] : nanf_();
  }
};

__device__ __forceinline__ ElevAccess make_access(const SlabView& v, const float* e) {
  return ElevAccess{e, v.rows, v.in_col0, v.in_ncols, v.cols_total};
}

// One cell of the whole chain.  The fix-up pass of the fused stencil recomputes only the part it
// could not certify (normals/slope/roughness and/or step) and always re-fuses.
__device__ void chain_cell_literal(const SlabView& v, const ChainDev& p, const float* elev, int i, int j,
                                   ChainOut o, bool do_normals, bool do_step, bool use_window = false) {
  const ElevAccess E = make_access(v, elev);
  const size_t oc = (size_t)(j - v.out_col0) * v.rows + i;
  float s, r, t;
  if (do_normals) {
    float fnx = nanf_(), fny = nanf_(), fnz = nanf_();
    if (use_window && p.Rn <= 3 && p.Rr <= 3) {
      ElevWindow Wn;
      Wn.fill(E, i, j);
      // the coordinates of the neighbourhood too: the window loops then run on local data only
      double Xl[7], Yl[7];
#pragma unroll
      for (int k = 0; k < 7; ++k) {
        Xl[k] = v.X[min(max(i - 3 + k, 0), v.rows - 1)];
        Yl[k] = v.Y[min(max(j - 3 + k, 0), v.cols_total - 1)];
      }
      SlabView vl = v;
      vl.X = Xl - (i - 3);
      vl.Y = Yl - (j - 3);
      if (finitef(Wn(i, j))) {
        double n[3];
        normal_literal(vl, p, Wn, i, j, n);
        fnx = (float)n[0]; fny = (float)n[1]; fnz = (float)n[2];
      }
      s = slope_literal(fnz, p.slope_crit);
      r = roughness_literal(vl, p, Wn, i, j, fnx, fny, fnz);
    } else {
      if (finitef(E(i, j))) {
        double n[3];
        normal_literal(v, p, E, i, j, n);
        fnx = (float)n[0]; fny = (float)n[1]; fnz = (float)n[2];
      }
      s = slope_literal(fnz, p.slope_crit);
      r = roughness_literal(v, p, E, i, j, fnx, fny, fnz);
    }
    o.slope[oc] = s;
    o.rough[oc] = r;
    if (o.nx) o.nx[oc] = fnx;
    if (o.ny) o.ny[oc] = fny;
    if (o.nz) o.nz[oc] = fnz;
  } else {
    s = o.slope[oc];
    r = o.rough[oc];
  }
  if (do_step) {
    t = step_literal(v, p, E, i, j);
    o.step[oc] = t;
  } else {
    t = o.step[oc];
  }
  o.trav[oc] = __fmul_rn(p.fuse_w, __fadd_rn(__fadd_rn(s, t), r));
}

__global__ void __launch_bounds__(128) k_chain_generic(SlabView v, ChainDev p, const float* __restrict__ elev, ChainOut o) {
  const long long total = (long long)v.rows * v.out_ncols;
  for (long long c = (long long)blockIdx.x * blockDim.x + threadIdx.x; c < total; c += (long long)gridDim.x * blockDim.x) {
    const int i = (int)(c % v.rows);
    const int j = v.out_col0 + (int)(c / v.rows);
    chain_cell_literal(v, p, elev, i, j, o, true, true);
  }
}

// Certified slow path of the fused stencil: recompute the listed cells (j_local*rows+i | flags<<30).
__global__ void __launch_bounds__(128) k_fixup_cells(SlabView v, ChainDev p, const float* __restrict__ elev, ChainOut o,
                                                     const unsigned int* __restrict__ list,
                                                     const unsigned int* __restrict__ count, unsigned int cap,
                                                     unsigned int* __restrict__ zero_next) {
  asm volatile("griddepcontrol.wait;" ::: "memory");  // programmatic dependent launch: tier 2 has finished and flushed its list
  if (zero_next && blockIdx.x == 0) zero_next[threadIdx.x] = 0u;  // the counter block of the next chain call (blockDim.x == 128 words)
  unsigned int n = *count;
  if (n > cap) n = cap;
  // A literal cell is ~40 us of serial, branchy double-precision code (half of it instruction fetch).  The usual handful of cells gets one warp each
  // (lane 0 works): no divergence between cells with different sweep counts, and the cells run on different SMs.
  // Long lists (degenerate maps, e.g. exact planes everywhere) fall back to one cell per thread.
  const unsigned int nthreads = gridDim.x * blockDim.x, tid = blockIdx.x * blockDim.x + threadIdx.x;
  const bool sparse = n <= (nthreads >> 5);
  if (sparse && (threadIdx.x & 31u) != 0u) return;
  for (unsigned int k = sparse ? (tid >> 5) : tid; k < n; k += sparse ? (nthreads >> 5) : nthreads) {
    const unsigned int w = list[k];
    const unsigned int c = w & 0x3fffffffu;  // bit 30: normals part, bit 31: step part
    const unsigned int map_cells = (unsigned)v.rows * (unsigned)v.out_ncols;
    const unsigned int mapi = c / map_cells, cl = c - mapi * map_cells;  // batched launches index cells across maps
    const int i = (int)(cl % (unsigned)v.rows);
    const int j = v.out_col0 + (int)(cl / (unsigned)v.rows);
    ChainOut om = o;
    const size_t off = (size_t)mapi * map_cells;
    om.slope += off; om.step += off; om.rough += off; om.trav += off;
    if (om.nx) { om.nx += off; om.ny += off; om.nz += off; }
    SlabView vm = v;  // the cell's map's coordinate tables (the same tables for every map unless the maps sit at their own positions)
    vm.X += (size_t)mapi * v.xs;
    vm.Y += (size_t)mapi * v.ys;
    chain_cell_literal(vm, p, elev + (size_t)mapi * v.rows * v.in_ncols, i, j, om, (w >> 30) & 1u, (w >> 31) & 1u, true);
  }
}

__global__ void __launch_bounds__(128) k_normals(SlabView v, ChainDev p, const float* __restrict__ elev, float* nx, float* ny, float* nz) {
  const long long total = (long long)v.rows * v.out_ncols;
  const ElevAccess E = make_access(v, elev);
  for (long long c = (long long)blockIdx.x * blockDim.x + threadIdx.x; c < total; c += (long long)gridDim.x * blockDim.x) {
    const int i = (int)(c % v.rows);
    const int j = v.out_col0 + (int)(c / v.rows);
    float a = nanf_(), b = nanf_(), d = nanf_();
    if (finitef(E(i, j))) {
      double n[3];
      normal_literal(v, p, E, i, j, n);
      a = (float)n[0]; b = (float)n[1]; d = (float)n[2];
    }
    nx[c] = a; ny[c] = b; nz[c] = d;
  }
}

__global__ void __launch_bounds__(256) k_slope(long long total, double crit, const float* __restrict__ nz, float* __restrict__ out) {
  for (long long c = (long long)blockIdx.x * blockDim.x + threadIdx.x; c < total; c += (long long)gridDim.x * blockDim.x)
    out[c] = slope_literal(__ldg(nz + c), crit);
}

__constant__ double c_acos14[15] = {3.139129045303817e-05,  -0.0002719939971935411, 0.0011120542916517797, -0.002896219765138688,
                                    0.005523167239593235,   -0.008503457350174303,  0.01149382355518035,   -0.01466134286289636,
                                    0.018621724287455857,   -0.024366397045309886,  0.03368046433967888,   -0.050792762643682245,
                                    0.08904862081826843,    -0.21460183657961013,   1.5707963267948457};

// The stand-alone SlopeFilter as a stream (8 B/cell).  acos in double as sqrt(1 - |x|) * P14(|x|) — a Chebyshev interpolant of
// acos(x)/sqrt(1 - x) on [0, 1], |error| <= 5.1e-14 rad against a 40-digit reference — instead of the library acos (~100
// instructions).  The result is CERTIFIED, not trusted: the layer value 1 - theta/critical is rounded to float32 here only when it
// stands clear (1e-12, 20 times the polynomial's error) of the float32 rounding boundaries and theta of the branch point
// theta == critical; the ~3 cells in 1e5 that do not are recomputed with the literal expression (SlopeFilter.cpp:74-81), so the
// layer is bit-identical to the literal kernel's (a degree-12 fit with a wider band was slower: its fall-backs diverge a fifth
// of the warps).  Four cells per thread, 16-byte accesses.
__device__ __forceinline__ float slope_stream(float x, double crit, double inv_crit, double band) {
  if (!finitef(x)) return nanf_();                      // no surface normal: the layer stays NaN (SlopeFilter.cpp:71)
  const double a = fabs((double)x);
  // coefficients as constant-bank operands of the DFMAs: as 64-bit literals they cost two UMOV each (28 of ~80 instructions per cell)
  double p = fma(a, c_acos14[0], c_acos14[1]);
#pragma unroll
  for (int k = 2; k < 15; ++k) p = fma(p, a, c_acos14[k]);
  double th = sqrt(1.0 - a) * p;
  if (x < 0.0f) th = 3.141592653589793 - th;
  const double v = fma(-th, inv_crit, 1.0);
  const float f = (float)v;
  // |v - f| against half a float32 ulp of f (exponent arithmetic on f's bits): within `band` of it, v sits on a rounding boundary
  const unsigned fb = __float_as_uint(f);
  float half_ulp = __uint_as_float(((fb >> 23) & 0xffu) > 26u ? ((fb & 0x7f800000u) - (24u << 23)) : 0u);
  if ((fb & 0x007fffffu) == 0u && v < (double)f) half_ulp *= 0.5f;  // below a power of two the float32 spacing halves
  const double r = fabs(v - (double)f);
  const bool sure = a <= 1.0 && fabs(th - crit) > band && fabs(r - (double)half_ulp) > band && f > 1e-30f;
  if (th >= crit + band) return 0.0f;                   // beyond the critical slope (clear of the branch point)
  if (!sure) return slope_literal(x, crit);             // also |x| > 1 (acos is NaN: the comparison is false -> 0.0)
  return f;
}
__global__ void __launch_bounds__(256) k_slope_stream(long long total4, double crit, double inv_crit, const float4* __restrict__ nz,
                                                      float4* __restrict__ out) {
  const double band = 1e-12 * fmax(1.0, inv_crit);
  for (long long c = (long long)blockIdx.x * blockDim.x + threadIdx.x; c < total4; c += (long long)gridDim.x * blockDim.x) {
    const float4 v = __ldg(nz + c);
    float4 r;
    r.x = slope_stream(v.x, crit, inv_crit, band);
    r.y = slope_stream(v.y, crit, inv_crit, band);
    r.z = slope_stream(v.z, crit, inv_crit, band);
    r.w = slope_stream(v.w, crit, inv_crit, band);
    out[c] = r;
  }
}

__global__ void __launch_bounds__(128) k_step(SlabView v, ChainDev p, const float* __restrict__ elev, float* out) {
  const long long total = (long long)v.rows * v.out_ncols;
  const ElevAccess E = make_access(v, elev);
  for (long long c = (long long)blockIdx.x * blockDim.x + threadIdx.x; c < total; c += (long long)gridDim.x * blockDim.x) {
    const int i = (int)(c % v.rows);
    const int j = v.out_col0 + (int)(c / v.rows);
    out[c] = step_literal(v, p, E, i, j);
  }
}

__global__ void __launch_bounds__(128) k_roughness(SlabView v, ChainDev p, const float* __restrict__ elev, const float* __restrict__ nx,
                                                   const float* __restrict__ ny, const float* __restrict__ nz, float* out) {
  const long long total = (long long)v.rows * v.out_ncols;
  const ElevAccess E = make_access(v, elev);
  for (long long c = (long long)blockIdx.x * blockDim.x + threadIdx.x; c < total; c += (long long)gridDim.x * blockDim.x) {
    const int i = (int)(c % v.rows);
    const int j = v.out_col0 + (int)(c / v.rows);
    out[c] = roughness_literal(v, p, E, i, j, __ldg(nx + c), __ldg(ny + c), __ldg(nz + c));
  }
}

inline int grid_for(long long total, int block, int sms) {
  long long g = (total + block - 1) / block;
  const long long cap = (long long)sms * 16;
  if (g > cap) g = cap;
  if (g < 1) g = 1;
  return (int)g;
}

}  // namespace

void launch_chain_generic(const SlabView& v, const ChainDev& p, const float* elev, const ChainOut& o, int sms, cudaStream_t s) {
  const long long total = (long long)v.rows * v.out_ncols;
  k_chain_generic<<<grid_for(total, 128, sms), 128, 0, s>>>(v, p, elev, o);
}

void launch_fixup(const SlabView& v, const ChainDev& p, const float* elev, const ChainOut& o, const unsigned int* list,
                  const unsigned int* count, unsigned int cap, unsigned int* zero_next, int sms, cudaStream_t s, bool pdl) {
  cudaLaunchConfig_t cfg{};
  cfg.gridDim = dim3((unsigned)(sms * 4));
  cfg.blockDim = dim3(128);
  cfg.stream = s;
  cudaLaunchAttribute at{};
  at.id = cudaLaunchAttributeProgrammaticStreamSerialization;
  at.val.programmaticStreamSerializationAllowed = 1;
  cfg.attrs = &at;
  cfg.numAttrs = pdl ? 1 : 0;
  cudaLaunchKernelEx(&cfg, k_fixup_cells, v, p, elev, o, list, count, cap, zero_next);
}

void launch_normals(const SlabView& v, const ChainDev& p, const float* elev, float* nx, float* ny, float* nz, int sms, cudaStream_t s) {
  const long long total = (long long)v.rows * v.out_ncols;
  k_normals<<<grid_for(total, 128, sms), 128, 0, s>>>(v, p, elev, nx, ny, nz);
}

void launch_slope(long long total, double crit, const float* nz, float* out, int sms, cudaStream_t s) {
  const bool aligned = ((reinterpret_cast<uintptr_t>(nz) | reinterpret_cast<uintptr_t>(out)) & 15u) == 0;
  if (crit > 0.0 && aligned && total >= 4) {
    const long long total4 = total / 4;
    const int grid = (int)std::min<long long>((total4 + 255) / 256, (long long)sms * 32);
    k_slope_stream<<<std::max(grid, 1), 256, 0, s>>>(total4, crit, 1.0 / crit, reinterpret_cast<const float4*>(nz),
                                                     reinterpret_cast<float4*>(out));
    const long long done = total4 * 4;
    if (done < total) k_slope<<<1, 32, 0, s>>>(total - done, crit, nz + done, out + done);
    return;
  }
  k_slope<<<grid_for(total, 256, sms), 256, 0, s>>>(total, crit, nz, out);
}

void launch_step(const SlabView& v, const ChainDev& p, const float* elev, float* out, int sms, cudaStream_t s) {
  const long long total = (long long)v.rows * v.out_ncols;
  k_step<<<grid_for(total, 128, sms), 128, 0, s>>>(v, p, elev, out);
}

void launch_roughness(const SlabView& v, const ChainDev& p, const float* elev, const float* nx, const float* ny, const float* nz,
                      float* out, int sms, cudaStream_t s) {
  const long long total = (long long)v.rows * v.out_ncols;
  k_roughness<<<grid_for(total, 128, sms), 128, 0, s>>>(v, p, elev, nx, ny, nz, out);
}

}  // namespace te
