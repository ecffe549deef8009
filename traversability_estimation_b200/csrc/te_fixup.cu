// te_fixup.cu — second tier of the fused stencil's certification ladder.
//
// Tier 1 (te_fused.cu) is fp32 with a closed form that assumes a full, valid disk window.  Cells it
// cannot certify land on a work list.  This tier recomputes them in fp64 on window-centred
// coordinates with validity-aware moments (map borders, NaN holes), which is accurate to ~1e-13 —
// far inside one float32 ulp — and escalates to tier 3 (the literal kernel in te_generic.cu, which
// replays the reference's own operand order on absolute coordinates) only where even that cannot
// decide: numerically rank-deficient scatter matrices (the reference's FullPivHouseholderQR rank
// test), ill-conditioned eigenvectors, or n_z within 1e-9 of a float32 rounding boundary.
#include <algorithm>

#include "te_fused.h"

namespace te {
namespace {

struct Elev {
  const float* __restrict__ e;
  int rows, col0, ncols, cols_total;
  __device__ __forceinline__ float operator()(int a, int b) const {
    if (a < 0 || a >= rows || b < 0 || b >= cols_total) return nanf_();
    const int lb = b - col0;
    if (lb < 0 || lb >= ncols) return nanf_();
    const float v = __ldg(e + (size_t)lb * rows + a);
    return finitef(v) ? v : nanf_();
  }
};

// step_height of cell (a,b): pass 1 of StepFilter.cpp:112-144 with the integer window description.
__device__ float step_height_t2(const FixupArgs& A, const Elev& E, int a, int b) {
  const float zc = E(a, b);
  if (!finitef(zc)) return nanf_();
  const unsigned rm = A.rowmask ? A.rowmask[a] : 0u, cm = A.colmask ? A.colmask[b] : 0u;
  float mn = zc, mx = zc;
#pragma unroll
  for (int l = -2; l <= 2; ++l) {
    const int w = A.w1[l < 0 ? -l : l];
    for (int k = -w; k <= w; ++k) {
      const float z = E(a + k, b + l);
      if (finitef(z)) { mn = fminf(mn, z); mx = fmaxf(mx, z); }
    }
  }
  if (A.tip1) {
    const float t0 = (rm & 1u) ? E(a - 2, b) : nanf_(), t1 = (rm & 2u) ? E(a + 2, b) : nanf_();
    const float t2 = (cm & 1u) ? E(a, b - 2) : nanf_(), t3 = (cm & 2u) ? E(a, b + 2) : nanf_();
    mn = fminf(fminf(mn, t0), fminf(t1, fminf(t2, t3)));  // fminf/fmaxf skip NaN operands
    mx = fmaxf(fmaxf(mx, t0), fmaxf(t1, fmaxf(t2, t3)));
  }
  return (float)((double)mx - (double)mn);
}

// pass 2 of StepFilter.cpp:147-178.  Out of line and with its arguments BY VALUE: the step part is needed for the rare cells an
// infinite elevation reaches, and a reference to the kernel parameters would force them into local memory for every thread.
__device__ __noinline__ float step_t2(const FixupArgs A, const Elev E, int i, int j) {
  const unsigned rm = A.rowmask ? A.rowmask[i] : 0u, cm = A.colmask ? A.colmask[j] : 0u;
  double stepMax = 0.0;
  int n = 0;
  bool any = false;
  auto visit = [&](int a, int b) {
    const float sh = step_height_t2(A, E, a, b);
    if (!finitef(sh)) return;
    any = true;
    if ((double)sh > stepMax) stepMax = (double)sh;
    if ((double)sh > A.step_crit) ++n;
  };
  for (int l = -2; l <= 2; ++l) {
    const int w = A.w2[l < 0 ? -l : l];
    for (int k = -w; k <= w; ++k) visit(i + k, j + l);
  }
  if (A.tip2) {
    if (rm & 4u) visit(i - 2, j);
    if (rm & 8u) visit(i + 2, j);
    if (cm & 4u) visit(i, j - 2);
    if (cm & 8u) visit(i, j + 2);
  }
  if (!any) return nanf_();
  const double step = fmin(stepMax, (double)n / (double)A.ncrit * stepMax);
  return (float)(step < A.step_crit ? 1.0 - step / A.step_crit : 0.0);
}

// 1/n, correctly rounded, for the valid-cell counts a 5 x 5 window can have (constant memory: indexed dynamically)
__constant__ double c_rcp[26] = {0.0,      1.0 / 1,  1.0 / 2,  1.0 / 3,  1.0 / 4,  1.0 / 5,  1.0 / 6,  1.0 / 7,  1.0 / 8,
                                 1.0 / 9,  1.0 / 10, 1.0 / 11, 1.0 / 12, 1.0 / 13, 1.0 / 14, 1.0 / 15, 1.0 / 16, 1.0 / 17,
                                 1.0 / 18, 1.0 / 19, 1.0 / 20, 1.0 / 21, 1.0 / 22, 1.0 / 23, 1.0 / 24, 1.0 / 25};

// acos on [0,1] in float32: sqrt(1-x) * P7(x), the same polynomial tier 1 evaluates (te_fused.cu acos2; max abs error 2.2e-7,
// max rel. error 1.7e-7 — 1 - x is exact, so the relative accuracy holds down to theta -> 0).  The argument is the float32 n_z
// the reference reads back from the layer (SlopeFilter.cpp:74).
__device__ __forceinline__ float acos_t2(float x) {
  const float u = 1.0f - x;
  float p = fmaf(x, -0.0011488182935863733f, 0.006254698149859905f);
  p = fmaf(p, x, -0.016484638676047325f);
  p = fmaf(p, x, 0.03044925443828106f);
  p = fmaf(p, x, -0.05000271648168564f);
  p = fmaf(p, x, 0.08894557505846024f);
  p = fmaf(p, x, -0.21459604799747467f);
  p = fmaf(p, x, 1.570796251296997f);
  return sqrtf(u) * p;
}

// Normals + slope + roughness of one cell in fp64 on centred coordinates.  Returns false when the
// result cannot be certified at this tier.
// `why` receives the reason of an escalation (1 degenerate full window, 2 rank of a full window, 3 eigen-gap of a full window,
// 4 no convergence, 5 rank of a partial window, 6 conditioning of a partial window, 7 null eigenvector, 8 n_z == 0,
// 9 n_z on a float32 rounding boundary) in its low byte and the number of valid window cells in the next one.
// SHAPE: the window's cells as a 25-bit mask (bit (l+2)*5 + (k+2)) known at compile time — the two shapes the fused stencil is
// instantiated for — so that cells outside the disk cost nothing (no load, no select, no bit test); 0 = take it from A.wn.
constexpr unsigned shape_mask(int w0, int w1, int w2) {
  auto col = [](int w) { return w >= 2 ? 0x1fu : w == 1 ? 0x0eu : w == 0 ? 0x04u : 0u; };
  return (col(w2)) | (col(w1) << 5) | (col(w0) << 10) | (col(w1) << 15) | (col(w2) << 20);
}
constexpr unsigned SHAPE_A = shape_mask(2, 2, 1), SHAPE_B = shape_mask(1, 1, -1);

template <unsigned SHAPE>
__device__ bool normals_t2(const FixupArgs& A, const Elev& E, int i, int j, float& fnx, float& fny, float& fnz, float& slope,
                           float& rough, unsigned& why) {
  const float zc = E(i, j);
  if (!finitef(zc)) {  // hole: no normal, slope and roughness stay NaN (SlopeFilter.cpp:71, RoughnessFilter.cpp:84)
    fnx = fny = fnz = slope = rough = nanf_();
    return true;
  }
  // Gather the 5 x 5 neighbourhood with 25 unconditional, independent loads and accumulate the four moments that involve z on
  // the fly (no array: nothing lives in local memory).  A cell that is outside the map / window / buffer or not finite is
  // replaced by the centre value (its deviation is an exact zero) and stays out of the validity mask (bit (l+2)*5 + (k+2)).
  unsigned mask = 0;
  double sw = 0, suw = 0, svw = 0, sww = 0;
  {
    const int lb0 = j - A.in_col0;
    const double dzc = (double)zc;
    unsigned shape = SHAPE;  // cells of the disk window
    if (SHAPE == 0u) {
#pragma unroll
      for (int l = -2; l <= 2; ++l) {
        const int w = A.wn[l < 0 ? -l : l];
        shape |= (w >= 2 ? 0x1fu : w == 1 ? 0x0eu : w == 0 ? 0x04u : 0u) << ((l + 2) * 5);
      }
    }
    float v[5][5];
    if (i >= 2 && i + 2 < A.rows && j >= 2 && j + 2 < A.cols_total && lb0 >= 2 && lb0 + 2 < A.in_ncols) {
      const float* base = E.e + (size_t)lb0 * A.rows + i;  // interior cell: no clamping
#pragma unroll
      for (int l = -2; l <= 2; ++l)
#pragma unroll
        for (int k = -2; k <= 2; ++k)
          v[l + 2][k + 2] = (SHAPE == 0u || ((SHAPE >> ((l + 2) * 5 + (k + 2))) & 1u)) ? __ldg(base + (ptrdiff_t)l * A.rows + k) : 0.0f;
    } else {
#pragma unroll
      for (int l = -2; l <= 2; ++l) {
        const int b = j + l, lb = lb0 + l;
        const bool col_ok = b >= 0 && b < A.cols_total && lb >= 0 && lb < A.in_ncols;
        const float* col = E.e + (size_t)min(max(lb, 0), A.in_ncols - 1) * A.rows;
#pragma unroll
        for (int k = -2; k <= 2; ++k) {
          const int a = i + k;
          if (SHAPE != 0u && !((SHAPE >> ((l + 2) * 5 + (k + 2))) & 1u)) { v[l + 2][k + 2] = 0.0f; continue; }
          const float x = __ldg(col + min(max(a, 0), A.rows - 1));
          v[l + 2][k + 2] = (col_ok && a >= 0 && a < A.rows) ? x : nanf_();
        }
      }
    }
#pragma unroll
    for (int l = -2; l <= 2; ++l) {
      double cs = 0.0, ck = 0.0;  // column sums of d and k*d
#pragma unroll
      for (int k = -2; k <= 2; ++k) {
        const unsigned bitm = 1u << ((l + 2) * 5 + (k + 2));
        if (SHAPE != 0u && !(SHAPE & bitm)) continue;  // not a cell of the window: folded away after unrolling
        const bool ok = finitef(v[l + 2][k + 2]) && (shape & bitm) != 0u;
        mask |= ok ? bitm : 0u;
        const double d = (double)(ok ? v[l + 2][k + 2] : zc) - dzc;  // invalid cells: exact zero
        cs += d;
        if (k != 0) ck = fma((double)k, d, ck);
        sww = fma(d, d, sww);
      }
      sw += cs;
      suw += ck;
      if (l != 0) svw = fma((double)l, cs, svw);
    }
    suw *= -A.res;  // u = -res*k, v = -res*l
    svw *= -A.res;
  }
  // The moments of the cell offsets depend only on WHICH cells are valid: integer sums over the 25-bit validity mask, exact.
  constexpr unsigned KM = 0x108421u, LM = 0x1fu;  // cells of row offset k = -2 / of column offset l = -2
  const int k_m2 = __popc(mask & KM), k_m1 = __popc(mask & (KM << 1)), k_p1 = __popc(mask & (KM << 3)), k_p2 = __popc(mask & (KM << 4));
  const int l_m2 = __popc(mask & LM), l_m1 = __popc(mask & (LM << 5)), l_p1 = __popc(mask & (LM << 15)), l_p2 = __popc(mask & (LM << 20));
  auto bit = [](int k, int l) { return 1u << ((l + 2) * 5 + (k + 2)); };
  const unsigned kl_p1 = bit(1, 1) | bit(-1, -1), kl_m1 = bit(1, -1) | bit(-1, 1);
  const unsigned kl_p2 = bit(2, 1) | bit(1, 2) | bit(-2, -1) | bit(-1, -2), kl_m2 = bit(2, -1) | bit(-1, 2) | bit(-2, 1) | bit(1, -2);
  const unsigned kl_p4 = bit(2, 2) | bit(-2, -2), kl_m4 = bit(2, -2) | bit(-2, 2);
  const int ik = 2 * (k_p2 - k_m2) + (k_p1 - k_m1), il = 2 * (l_p2 - l_m2) + (l_p1 - l_m1);
  const int ikk = 4 * (k_p2 + k_m2) + (k_p1 + k_m1), ill = 4 * (l_p2 + l_m2) + (l_p1 + l_m1);
  const int ikl = (__popc(mask & kl_p1) - __popc(mask & kl_m1)) + 2 * (__popc(mask & kl_p2) - __popc(mask & kl_m2)) +
                  4 * (__popc(mask & kl_p4) - __popc(mask & kl_m4));
  const double res2 = A.res * A.res;
  const int cnt = __popc(mask);
  const double su = -A.res * (double)ik, sv = -A.res * (double)il;
  const double suu = res2 * (double)ikk, svv = res2 * (double)ill, suv = res2 * (double)ikl;
  double nx = 0.0, ny = 0.0, nz = 1.0;
  const double rn = c_rcp[cnt];  // 1/n, correctly rounded
  const double mu = su * rn, mv = sv * rn, mw = sw * rn;
  // scatter matrix sum (p - mean)(p - mean)^T
  const double xx = fma(-su, mu, suu), xy = fma(-su, mv, suv), xz = fma(-su, mw, suw);
  const double yy = fma(-sv, mv, svv), yz = fma(-sv, mw, svw), zz = fma(-sw, mw, sww);
  if (cnt >= 3 && zz > 0.0) {
    double bx, by, bz;
    if (cnt == A.n_full_i) {
      // full disk window: scatter = [[a,0,p],[0,a,q],[p,q,c]] (sums of u, v, uv vanish by symmetry) and
      // the eigen-problem collapses to 2x2 — robust even when two eigenvalues nearly coincide
      const double a = 0.5 * (xx + yy), g2 = fma(xz, xz, yz * yz);
      const double h = 0.5 * (a - zz), hh = fma(h, h, g2);
      const double D = sqrt(hh);
      const double dph = D + fabs(h);
      why = 1u | ((unsigned)cnt << 8);
      if (!(dph > 0.0)) return false;
      const double qq = g2 / dph;
      const double m = h >= 0.0 ? dph : qq;           // a - lambda0
      const double lam = (h >= 0.0 ? zz : a) - qq;     // lambda0
      const double big = fmax(a, zz);
      why = 2u | ((unsigned)cnt << 8);
      if (!(lam > 1e-9 * big)) return false;           // rank: the literal QR decides (tier 3)
      why = 3u | ((unsigned)cnt << 8);
      if (!(fmin(2.0 * D, m) > 1e-7 * big)) return false;
      bx = -xz; by = -yz; bz = m;
    } else {
      const double c2 = xx + yy + zz;
      const double c1 = xx * yy + xx * zz + yy * zz - xy * xy - xz * xz - yz * yz;
      const double c0 = xx * (yy * zz - yz * yz) - xy * (xy * zz - yz * xz) + xz * (xy * yz - yy * xz);
      // smallest root of p(l) = -l^3 + c2 l^2 - c1 l + c0 (three real non-negative roots): Halley from 0 converges monotonically
      // from below and cubically — three or four iterations where Newton took six to ten, one division each
      double lam = 0.0, dp = -c1;
      bool conv = false;
#pragma unroll 1
      for (int it = 0; it < 40; ++it) {
        const double pv = fma(fma(c2 - lam, lam, -c1), lam, c0);
        dp = fma(fma(-3.0, lam, 2.0 * c2), lam, -c1);
        const double hpp = fma(-3.0, lam, c2);                   // p''/2
        const double den = fma(dp, dp, -pv * hpp);               // p'^2 - p p''/2  (> 0 below the smallest root)
        if (!(den > 0.0)) break;
        const double step = pv * dp / den;                       // Halley: p p' / (p'^2 - p p''/2), negative (p > 0 > p')
        lam -= step;
        if (fabs(step) <= 1e-15 * c2) { conv = true; break; }
      }
      dp = fma(fma(-3.0, lam, 2.0 * c2), lam, -c1);
      // rank: lambda0 at the reference's rank-threshold scale -> the literal QR decides (tier 3);
      // conditioning: |p'(lambda0)| = (l1 - l0)(l2 - l0) must leave the cross products accurate
      why = (!conv ? 4u : !(lam > 1e-9 * c2) ? 5u : 6u) | ((unsigned)cnt << 8);
      if (!conv || !(lam > 1e-9 * c2) || !(fabs(dp) > 1e-4 * c2 * c2)) return false;
      const double ax = xx - lam, ay = yy - lam, az = zz - lam;
      // eigenvector = largest cross product of two rows of (S - lambda0 I)
      const double v0x = xy * yz - xz * ay, v0y = xz * xy - ax * yz, v0z = ax * ay - xy * xy;  // r0 x r1
      const double v1x = xy * az - xz * yz, v1y = xz * xz - ax * az, v1z = ax * yz - xy * xz;  // r0 x r2
      const double v2x = ay * az - yz * yz, v2y = yz * xz - xy * az, v2z = xy * yz - ay * xz;  // r1 x r2
      const double q0 = v0x * v0x + v0y * v0y + v0z * v0z, q1 = v1x * v1x + v1y * v1y + v1z * v1z, q2 = v2x * v2x + v2y * v2y + v2z * v2z;
      bx = v0x; by = v0y; bz = v0z;
      double bq = q0;
      if (q1 > bq) { bx = v1x; by = v1y; bz = v1z; bq = q1; }
      if (q2 > bq) { bx = v2x; by = v2y; bz = v2z; bq = q2; }
    }
    const double bq = fma(bx, bx, fma(by, by, bz * bz));
    why = 7u | ((unsigned)cnt << 8);
    if (!(bq > 0.0)) return false;
    const double inv = rsqrt(bq);
    nx = bx * inv; ny = by * inv; nz = bz * inv;
    if (nz < 0.0) { nx = -nx; ny = -ny; nz = -nz; }
    why = 8u | ((unsigned)cnt << 8);
    if (nz == 0.0) return false;
    // float32 rounding of n_z: where acos amplifies one ulp beyond the tolerance (theta < ~0.02 rad at crit = 1 rad, up to
    // just past crit for small crit: A.nz_check) the rounding must be certain: escalate when n_z is within A.nz_guard ulps of a
    // rounding boundary (make_fixup_args: 100 x the error the reference's absolute-coordinate arithmetic can carry into its own n_z)
    if (nz > A.nz_check) {
      const float f = (float)nz;
      const float up = __uint_as_float(__float_as_uint(f) + 1u), dn = __uint_as_float(__float_as_uint(f) - 1u);
      const double bu = 0.5 * ((double)f + (double)up), bd = 0.5 * ((double)f + (double)dn);
      // the reference's error grows with the cell's own s = 1 - n_z: nz_guard holds for s <= 2e-4
      const double guard = A.nz_guard * fmax(1.0, (1.0 - nz) * 5e3) * (bu - bd);
      why = 9u | ((unsigned)cnt << 8);
      if (fabs(nz - bu) < guard || fabs(nz - bd) < guard) return false;
    }
  }
  fnx = (float)nx; fny = (float)ny; fnz = (float)nz;
  // layer = x < crit ? 1 - x/crit : 0 in double, narrowed on store (SlopeFilter.cpp:74-81); 1/crit is a host-side constant
  const double th = (double)acos_t2(fminf(fnz, 1.0f));
  slope = (float)(th < A.slope_crit ? fma(-th, A.inv_slope_crit, 1.0) : 0.0);
  // roughness with the float32 normal (RoughnessFilter.cpp:108-117): the sum over the window of (N . (p - mean))^2 is the
  // quadratic form N^T S N of the scatter matrix already at hand (the reference sums it point by point; the quadratic form
  // loses at most ~1e-16 * |S| absolutely, ~1e-12 of the layer value)
  const double NX = fnx, NY = fny, NZ = fnz;
  const double sum = fmax(NX * (NX * xx + 2.0 * (NY * xy + NZ * xz)) + NY * (NY * yy + 2.0 * NZ * yz) + NZ * NZ * zz, 0.0);
  if (cnt >= 2) {
    const double r = sqrt(sum * c_rcp[cnt - 1]);
    rough = (float)(r < A.rough_crit ? fma(-r, A.inv_rough_crit, 1.0) : 0.0);
  } else {
    rough = 0.0f;  // one point: 0/0 = NaN -> comparison false -> 0.0 (RoughnessFilter.cpp:117-124)
  }
  return true;
}

template <unsigned SHAPE>
__global__ void __launch_bounds__(128, 8) k_fixup_t2(FixupArgs A, const float* __restrict__ elev, ChainOut o,
                                                  const unsigned* __restrict__ list, const unsigned* __restrict__ count,
                                                  unsigned cap, unsigned* list3, unsigned* count3, unsigned cap3) {
  asm volatile("griddepcontrol.launch_dependents;");   // tier 3 may be set up while this grid runs
  asm volatile("griddepcontrol.wait;" ::: "memory");   // programmatic dependent launch: the fused kernel has finished and flushed its list
  unsigned n = *count;
  if (n > cap) n = cap;
  for (unsigned k = blockIdx.x * blockDim.x + threadIdx.x; k < n; k += gridDim.x * blockDim.x) {
    const unsigned w = list[k];
    if (w == LIST_INVALID) continue;  // padding of a warp's chunk tail
    const unsigned c = w & 0x3fffffffu;
    const unsigned mapi = c / A.map_cells, cl = c - mapi * A.map_cells;
    const int i = (int)(cl % (unsigned)A.rows);
    const int j = A.out_col0 + (int)(cl / (unsigned)A.rows);
    const Elev E{elev + (size_t)mapi * A.in_map_stride, A.rows, A.in_col0, A.in_ncols, A.cols_total};
    const bool do_n = (w >> 30) & 1u, do_s = (w >> 31) & 1u;
    float s, r, t;
    bool escalate = false;
    unsigned why = 0;
    if (do_n) {
      float fx, fy, fz;
      if (normals_t2<SHAPE>(A, E, i, j, fx, fy, fz, s, r, why)) {
        o.slope[c] = s;
        o.rough[c] = r;
        if (o.nx) { o.nx[c] = fx; o.ny[c] = fy; o.nz[c] = fz; }
      } else {
        escalate = true;
      }
    } else {
      s = o.slope[c];
      r = o.rough[c];
    }
    if (do_s) {
      if (A.rowmask_stride | A.colmask_stride) {  // the maps sit at their own positions: the cell's map's masks
        FixupArgs Am = A;
        Am.rowmask += (size_t)mapi * A.rowmask_stride;
        Am.colmask += (size_t)mapi * A.colmask_stride;
        t = step_t2(Am, E, i, j);
      } else {
        t = step_t2(A, E, i, j);
      }
      o.step[c] = t;
    } else {
      t = o.step[c];
    }
    if (escalate) {
      const unsigned idx = atomicAdd(count3, 1u);
      if (idx < cap3) list3[idx] = c | (1u << 30);  // tier 3 redoes the normals part and re-fuses
      else atomicExch(count3 + 1, 1u);              // cannot happen: list3 holds every cell of the launch
      atomicAdd(count3 + 4 + (why & 15u), 1u);       // diagnostics (te_get_escalation_stats): by reason ...
      atomicAdd(count3 + 20 + min((why >> 8) & 31u, 25u), 1u);  // ... and by number of valid window cells
    } else {
      o.trav[c] = __fmul_rn(A.fuse_w, __fadd_rn(__fadd_rn(s, t), r));
    }
  }
}

}  // namespace

void launch_fixup_t2(const FixupArgs& a, const float* elev, const ChainOut& o, const unsigned* list, const unsigned* count,
                     unsigned cap, unsigned* list3, unsigned* count3, unsigned cap3, int sms, cudaStream_t s, bool pdl) {
  cudaLaunchConfig_t cfg{};
  // one listed cell per thread up to ~1.2 M threads (latency hidden by occupancy), grid-stride beyond; small launches get a grid in
  // proportion to their cell count (about 3 % of the cells are listed) so that a 2048^2 map does not pay for 9 472 blocks
  const unsigned long long want = ((unsigned long long)cap3 / 32ull + 127ull) / 128ull;  // cap3 = cells of the launch (all maps)
  cfg.gridDim = dim3((unsigned)std::min<unsigned long long>((unsigned long long)sms * 64ull, std::max<unsigned long long>(want, (unsigned long long)sms * 2ull)));
  cfg.blockDim = dim3(128);
  cfg.stream = s;
  cudaLaunchAttribute at{};
  at.id = cudaLaunchAttributeProgrammaticStreamSerialization;
  at.val.programmaticStreamSerializationAllowed = 1;
  cfg.attrs = &at;
  cfg.numAttrs = pdl ? 1 : 0;
  const bool is_a = a.wn[0] == 2 && a.wn[1] == 2 && a.wn[2] == 1, is_b = a.wn[0] == 1 && a.wn[1] == 1 && a.wn[2] == -1;
  if (is_a) cudaLaunchKernelEx(&cfg, k_fixup_t2<SHAPE_A>, a, elev, o, list, count, cap, list3, count3, cap3);
  else if (is_b) cudaLaunchKernelEx(&cfg, k_fixup_t2<SHAPE_B>, a, elev, o, list, count, cap, list3, count3, cap3);
  else cudaLaunchKernelEx(&cfg, k_fixup_t2<0u>, a, elev, o, list, count, cap, list3, count3, cap3);
}

}  // namespace te
