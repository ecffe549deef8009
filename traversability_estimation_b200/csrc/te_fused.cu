// te_fused.cu — the fused chain stencil for sm_90a (H100).
//
// One launch computes, for every cell of a column slab, what the reference's six-filter chain
// (robot_filter_parameter.yaml:2-37) computes — normals -> slope, step (both passes), roughness,
// weighted sum — reading `elevation` once and writing the four output layers once; no
// intermediate layer (surface normals, step_height) ever reaches HBM.
//
// Execution model (DESIGN.md §"fused stencil"):
//   * The layer is column-major, row index contiguous.  A WARP owns a strip of 64 rows (two adjacent
//     rows per lane, so all arithmetic is issued on row pairs) and marches along the
//     column index.  Warps are autonomous: each has its own TMA ring (4 stages x 5 columns x 68 rows,
//     NaN out-of-bounds fill so map borders look like invalid cells), its own mbarriers and a tiny
//     step_height exchange buffer; there is no __syncthreads in the kernel.  Work units are (60-row strip,
//     column segment) pairs popped from a device queue, long segments first (plan_levels).
//   * Everything a lane needs from columns other than the arriving one lives in registers as
//     five-deep rings indexed at compile time (the march is unrolled by 5 = ring depth = TMA chunk).
//   * Surface normals use the closed form of the 3x3 eigen-problem that holds for a full disk window
//     (scatter matrix [[a,0,p],[0,a,q],[p,q,c]]); moments are accumulated from per-column run sums
//     centred on the run's own middle cell and re-centred on the output cell, so fp32 never sees a
//     cancellation larger than the window's own elevation spread.
//   * fp32 results are CERTIFIED, not trusted: a cell whose window holds an invalid cell (NaN
//     poisoning of the moments / of the NaN-propagating min-max), whose n_z lies too close to a
//     float32 rounding boundary where acos amplifies it, whose scatter matrix is numerically
//     rank-deficient, or whose roughness cancels too far, is appended to a work list and recomputed
//     in fp64 on centred coordinates (te_fixup.cu: k_fixup_t2), which hands what it cannot decide
//     either to the literal double-precision kernel (te_generic.cu: k_fixup_cells).
#include <cuda.h>
#include <cuda_runtime.h>

#include <cmath>
#include <cstdio>
#include <cstdlib>
#include <cstring>

#include "te_fused.h"
#include "te_grid.cuh"

namespace te {
namespace {

constexpr int SROWS = 64;          // rows a warp holds (two adjacent rows per lane): step_height rows
constexpr int OROWS = 60;          // rows a warp produces (lanes 1..30); pitch of the strips
constexpr int EROWS = SROWS + 4;   // staged elevation rows (2 more each side for the step_height rows)
constexpr int CH = 5;              // columns per TMA chunk = unroll factor = ring depth
constexpr int NST = 4;             // TMA ring stages per warp
constexpr int STAGE_BYTES = 1408;  // EROWS*CH*4 = 1360, padded so every stage is 128-byte aligned
constexpr int SHBUF_BYTES = 272;   // 2 pad + 64 + 2 pad floats (264 bytes), 16-byte aligned
constexpr int NSHB = 3;            // step_height exchange buffers: buffer PH % 3, so the address is a compile-time offset, consecutive
                                   // steps never share a buffer and a buffer is rewritten two steps (= one __syncwarp) after it was read
constexpr int STAGE_PAD = EROWS * CH * 4;  // first byte of a stage TMA does not write: 5 x 4 column-mask bytes of the chunk live there
// The run-sum and column-statistics rings live in shared memory instead of registers (one 8-byte element per lane and slot:
// conflict-free), which brings the kernel under the 168 registers that a third warp per scheduler needs (the register file is
// four 16 K partitions), so 12 warps fit per SM: k_chain_fused is compiled with __maxnreg__(168).
// RING_REG1: bit mask of rings (RingId) whose age-1 read comes from the register the value was put in one step earlier instead
// of from shared memory (one more live register pair per ring, one LDS.64 less per step): A2 B2 Q2 C1MN C1MX S3MX S3C.  ShapeA
// takes 168 / 166 registers without / with the normals outputs, two LDS per march step fewer than 0xF8 (the same without S3MX S3C).
constexpr unsigned RING_REG1 = 0x3F8;
enum RingId { R_A1, R_B1, R_Q1, R_A2, R_B2, R_Q2, R_C1MN, R_C1MX, R_S3MX, R_S3C, NRING };
constexpr int RING_BYTES = NRING * 5 * 32 * 8;
constexpr int WARP_SMEM_BYTES = NST * STAGE_BYTES + (NSHB * SHBUF_BYTES + 48 + 127) / 128 * 128 + RING_BYTES;  // 5632 + 896 + 12800: 151 * 128; 12 warps = 226.5 KB
constexpr int WARPS_PER_CTA = 12;
static_assert(WARPS_PER_CTA * WARP_SMEM_BYTES <= 232448, "the warps of a CTA must fit the 227 KB of dynamic shared memory");
constexpr int WARP_AUX_OFF = NST * STAGE_BYTES + NSHB * SHBUF_BYTES;  // mbarriers (NST x 8 bytes), then the work-list cursor (8 bytes)
constexpr int WARP_RING_OFF = WARP_SMEM_BYTES - RING_BYTES;
constexpr unsigned FULL = 0xffffffffu;

constexpr int NLVL = 4;            // levels of the work queue
constexpr unsigned LIST_CHUNK = 512u;  // work-list entries a warp reserves at a time (an append adds at most 64)

typedef unsigned long long f2;  // two packed floats in one aligned register pair (see below)

// The kernel parameter block.  Some members are read by no kernel (half_a, kp, invN, ..., k_1p5, k_0375, k_m03125); they stay,
// in this order, on purpose: the layout decides where each constant sits in the parameter bank, and removing members changes
// how ptxas schedules k_chain_fused's constant loads.
struct FusedArgs {
  int rows, cols_total;
  int in_col0, in_ncols, out_col0, out_ncols;
  int nstrips;
  // work queue: units are (level, map, column segment, strip); levels hold ever shorter segments so the
  // warps that pop the queue last finish close together
  int lvl_unit0[NLVL + 1];      // first unit of each level; [NLVL] = number of units
  int lvl_col0[NLVL + 1];       // first output column (relative to out_col0) of each level
  int lvl_len[NLVL];            // segment length of each level
  int lvl_nseg[NLVL];           // segments per map of each level
  unsigned* queue;              // zeroed before the launch; warps pop unit ids past their first one
  int nmaps;                    // independent maps stored back to back (te_chain_batched); 1 otherwise
  unsigned map_cells;           // rows * out_ncols: output cells per map
  float half_a;     // 0.5 * res^2 * K2 / N   (Cxx = Cyy of a full window is a = 2*half_a)
  float a_cov;
  float kp;         // -res / N         (Cxz = kp * sum k*w)
  float invN;       // 1 / N
  float n_over_nm1; // N / (N-1)
  float rough_thr;  // (0.2 / crit_rough)^2 * (N-1)/N : lambda0 below rough_thr*cmag^2 cannot be certified
  float slope_crit, inv_slope_crit, minv_slope_crit;
  float step_crit, inv_step_crit, minv_step_crit, inv_ncrit;
  float step_cmp;   // largest float <= critical step (double): `h > step_cmp` in float == `(double)h > critical` (StepFilter.cpp:165)
  float rough_crit, inv_rough_crit, minv_rough_crit;
  float fuse_w;
  float cond_k;     // eigen-gap / scale ratio below which the fp32 eigenvector is not trusted
  // constants of the row-pair arithmetic, one float each: both halves of a pair operation take the same constant-bank word
  // as a direct FFMA/FADD/FMUL operand, so a constant costs no load and no register
  float k_invN, k_kp, k_half_a, k_nnm1, k_rough_thr, k_m0, k_m1;
  float k_inv_ncrit, k_fuse_w;
  float k_1em5, k_1em10a, k_mcond, k_2p24, k_7p1em6, k_2em6, k_bmargin;
  float k_one, k_two, k_half, k_1p5, k_0375, k_m03125, k_p0, k_p1, k_p2, k_p3, k_p4, k_p5, k_p6, k_p7;
  const unsigned char* rowmask;  // per global row: bit0/1 pass-1 tips (-2,0)/(+2,0); bit2/3 pass-2 tips
  const unsigned char* colmask;  // per global column, same bits for (0,-2)/(0,+2)
  unsigned rowmask_stride, colmask_stride;  // map m's masks start m * stride bytes in (0: every map at one position)
  float* slope;
  float* step;
  float* rough;
  float* trav;
  float* nx;
  float* ny;
  float* nz;
  unsigned* list;
  unsigned* count;
  unsigned cap;
  float k_nz_check;  // s = 1 - n_z below which the float32 rounding of n_z is certified: nz_check_limit(slope_crit)
};

// ---------------------------------------------------------------------------------------------
// paired f32 arithmetic: .x = row i, .y = row i+1 of the lane
// ---------------------------------------------------------------------------------------------
// An f2 lives in one 64-bit register pair; lo()/hi() only name the halves.  sm_90 has no packed
// f32x2 instructions, so every pair operation is two scalar round-to-nearest instructions (never
// contracted), which round each half exactly as a packed instruction would.
__device__ __forceinline__ f2 mk(float x, float y) {
  f2 r;
  asm("mov.b64 %0, {%1, %2};" : "=l"(r) : "f"(x), "f"(y));
  return r;
}
__device__ __forceinline__ float lo(f2 v) {
  float a, b;
  asm("mov.b64 {%0, %1}, %2;" : "=f"(a), "=f"(b) : "l"(v));
  return a;
}
__device__ __forceinline__ float hi(f2 v) {
  float a, b;
  asm("mov.b64 {%0, %1}, %2;" : "=f"(a), "=f"(b) : "l"(v));
  return b;
}
__device__ __forceinline__ f2 add2(f2 a, f2 b) { return mk(__fadd_rn(lo(a), lo(b)), __fadd_rn(hi(a), hi(b))); }
__device__ __forceinline__ f2 sub2(f2 a, f2 b) { return mk(__fsub_rn(lo(a), lo(b)), __fsub_rn(hi(a), hi(b))); }
__device__ __forceinline__ f2 mul2(f2 a, f2 b) { return mk(__fmul_rn(lo(a), lo(b)), __fmul_rn(hi(a), hi(b))); }
__device__ __forceinline__ f2 fma2(f2 a, f2 b, f2 c) { return mk(__fmaf_rn(lo(a), lo(b), lo(c)), __fmaf_rn(hi(a), hi(b), hi(c))); }
// a scalar constant k (a FusedArgs member) as one operand of both halves; the operand order of each scalar instruction is
// the one the pair form with a broadcast constant had, so the results are the same bits
__device__ __forceinline__ f2 mul2c(f2 a, float k) { return mk(__fmul_rn(lo(a), k), __fmul_rn(hi(a), k)); }
__device__ __forceinline__ f2 sub2c(f2 a, float k) { return mk(__fsub_rn(lo(a), k), __fsub_rn(hi(a), k)); }
__device__ __forceinline__ f2 csub2(float k, f2 a) { return mk(__fsub_rn(k, lo(a)), __fsub_rn(k, hi(a))); }
__device__ __forceinline__ f2 fma2c(f2 a, f2 b, float k) { return mk(__fmaf_rn(lo(a), lo(b), k), __fmaf_rn(hi(a), hi(b), k)); }
__device__ __forceinline__ f2 fma2k(f2 a, float k, f2 c) { return mk(__fmaf_rn(lo(a), k, lo(c)), __fmaf_rn(hi(a), k, hi(c))); }
__device__ __forceinline__ f2 kfma2(float k, f2 b, f2 c) { return mk(__fmaf_rn(k, lo(b), lo(c)), __fmaf_rn(k, hi(b), hi(c))); }
__device__ __forceinline__ f2 fma2kc(f2 a, float k, float c) { return mk(__fmaf_rn(lo(a), k, c), __fmaf_rn(hi(a), k, c)); }
__device__ __forceinline__ f2 kmul2(float k, f2 b) { return mk(__fmul_rn(k, lo(b)), __fmul_rn(k, hi(b))); }
__device__ __forceinline__ f2 bc(float v) { return mk(v, v); }
__device__ __forceinline__ f2 neg2(f2 a) { return a ^ 0x8000000080000000ull; }
// -a for both rows, written as two scalar negations: ptxas folds each into the operand modifier of the consuming
// FFMA/FADD/FMUL, so the negation costs no instruction (an integer XOR would cost two).
__device__ __forceinline__ f2 negf2(f2 a) { return mk(-lo(a), -hi(a)); }

// Three-input min/max with IEEE minNum/maxNum semantics: NaN operands are skipped, which is
// exactly how the reference's step filter treats invalid cells (StepFilter.cpp:126,159); the result is
// NaN only when every operand is.  Excluded on-circle tips are passed as NaN.  Two chained FMNMX (sm_90
// has no three-input form).
__device__ __forceinline__ float max3n(float a, float b, float c) {
  float r;
  asm("{ .reg .f32 t; max.f32 t, %1, %2; max.f32 %0, t, %3; }" : "=f"(r) : "f"(a), "f"(b), "f"(c));
  return r;
}
__device__ __forceinline__ float min3n(float a, float b, float c) {
  float r;
  asm("{ .reg .f32 t; min.f32 t, %1, %2; min.f32 %0, t, %3; }" : "=f"(r) : "f"(a), "f"(b), "f"(c));
  return r;
}
// 1.0f / 0.0f comparison result in one instruction (FSET.BF)
__device__ __forceinline__ float gtf(float a, float b) {
  float r;
  asm("set.gt.f32.f32 %0, %1, %2;" : "=f"(r) : "f"(a), "f"(b));
  return r;
}
// max(fma(a, b, 1), 0) for a*b <= 0 in one instruction (FFMA.SAT clamps to [0, 1]; NaN -> +0 exactly like fmaxf(NaN, 0))
__device__ __forceinline__ float fma_sat1(float a, float b) {
  float r;
  asm("fma.rn.sat.f32 %0, %1, %2, 0f3F800000;" : "=f"(r) : "f"(a), "f"(b));
  return r;
}
__device__ __forceinline__ float rcp_a(float x) {
  float r;
  asm("rcp.approx.ftz.f32 %0, %1;" : "=f"(r) : "f"(x));
  return r;
}
__device__ __forceinline__ float sqrt_a(float x) {
  float r;
  asm("sqrt.approx.ftz.f32 %0, %1;" : "=f"(r) : "f"(x));
  return r;
}

// ---------------------------------------------------------------------------------------------
// shared memory / mbarrier / TMA (per-warp pipelines), all on 32-bit shared addresses
// ---------------------------------------------------------------------------------------------
__device__ __forceinline__ unsigned smem_u32(const void* p) { return (unsigned)__cvta_generic_to_shared(p); }
__device__ __forceinline__ f2 lds64(unsigned a) {
  f2 v;
  asm volatile("ld.shared.b64 %0, [%1];" : "=l"(v) : "r"(a));
  return v;
}
__device__ __forceinline__ void sts64(unsigned a, float x, float y) {
  asm volatile("st.shared.v2.f32 [%0], {%1, %2};" ::"r"(a), "f"(x), "f"(y) : "memory");
}
__device__ __forceinline__ void sts64(unsigned a, f2 v) {
  asm volatile("st.shared.b64 [%0], %1;" ::"r"(a), "l"(v) : "memory");
}
__device__ __forceinline__ void mbar_init(unsigned bar, int count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(bar), "r"(count));
}
__device__ __forceinline__ void mbar_expect_tx(unsigned bar, unsigned bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(bar), "r"(bytes) : "memory");
}
__device__ __forceinline__ void mbar_wait(unsigned bar, unsigned parity) {
  unsigned ok = 0;
  while (!ok) {
    asm volatile(
        "{ .reg .pred p; mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2; selp.u32 %0, 1, 0, p; }"
        : "=r"(ok)
        : "r"(bar), "r"(parity)
        : "memory");
  }
}
__device__ __forceinline__ void tma_load_3d(unsigned dst, const CUtensorMap* map, int c0, int c1, int c2, unsigned bar) {
  asm volatile(
      "cp.async.bulk.tensor.3d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%2, %3, %4}], [%5];" ::"r"(dst),
      "l"(map), "r"(c0), "r"(c1), "r"(c2), "r"(bar)
      : "memory");
}

// ---------------------------------------------------------------------------------------------
// Window shapes within reach 2 (half-width per |column offset|; -1 = column not in the window).
// TIP = the four offsets (+-2,0),(0,+-2) lie exactly ON the circle and are decided per row/column
// from the double-precision tables (rowmask/colmask), SURVEY.md Appendix C.1.
// ---------------------------------------------------------------------------------------------
template <int WN0_, int WN1_, int WN2_, int W10_, int W11_, int W12_, bool TIP1_, int W20_, int W21_, int W22_, bool TIP2_>
struct Shape {
  static constexpr int WN0 = WN0_, WN1 = WN1_, WN2 = WN2_;
  static constexpr int W10 = W10_, W11 = W11_, W12 = W12_;
  static constexpr bool TIP1 = TIP1_;
  static constexpr int W20 = W20_, W21 = W21_, W22 = W22_;
  static constexpr bool TIP2 = TIP2_;
  static constexpr bool NEED_N1 = (WN0_ == 1 || WN1_ == 1 || WN2_ == 1);
  static constexpr bool NEED_N2 = (WN0_ == 2 || WN1_ == 2 || WN2_ == 2);
  static constexpr bool MASKS = TIP1_ || TIP2_;
};

template <int W>
__device__ __forceinline__ float colmin_w(const float* z, int r) {  // z[r+2] is the centre row
  if constexpr (W == 0) return z[r + 2];
  else if constexpr (W == 1) return min3n(z[r + 1], z[r + 2], z[r + 3]);
  else return min3n(min3n(z[r + 1], z[r + 2], z[r + 3]), z[r], z[r + 4]);
}
template <int W>
__device__ __forceinline__ float colmax_w(const float* z, int r) {
  if constexpr (W == 0) return z[r + 2];
  else if constexpr (W == 1) return max3n(z[r + 1], z[r + 2], z[r + 3]);
  else return max3n(max3n(z[r + 1], z[r + 2], z[r + 3]), z[r], z[r + 4]);
}
// count (as float) of rows whose flag f[] is set
template <int W>
__device__ __forceinline__ float colcnt_w(const float* f, int r) {
  float c = f[r + 2];
  if constexpr (W >= 1) c += f[r + 1] + f[r + 3];
  if constexpr (W >= 2) c += f[r] + f[r + 4];
  return c;
}

// Per-lane register state.  Rings are indexed by the arrival phase of the column (0..4).
template <class S>
struct Lane {
  f2 e[5];                           // own-row elevation
  f2 a1[5], b1[5], q1[5];            // three-row run sums centred on the run's middle cell
  f2 a2[5], b2[5], q2[5];            // five-row run sums
  f2 c1mn[5], c1mx[5];               // pass-1 column min/max of width W11 (columns l = +-1)
  f2 p1mn[5], p1mx[5];               // pass-1 centre column (width W10 + masked tips)
  f2 sh[5];                          // own-row step_height
  f2 s3mx[5], s3c[5];                // pass-2 column max / count of width W21
  f2 pcmx[5], pcc[5];                // pass-2 centre column
  f2 dslope[5], drough[5];           // slope / roughness layers waiting for the step layer
  unsigned dflag[5];                 // certification flags of the normals stage (bit0 row x, bit1 row y)
};

// Ring access.  A value is written to its register slot and stored to shared memory; every read of a slot other than the one
// written in this very step comes from shared memory, so the register copy dies with the step.  The RING_REG1 rings also read
// the slot written one step earlier from its register, which then lives one step longer.
template <int RID, int SLOT, class CT>
__device__ __forceinline__ void ring_put(const CT& C, f2 (&reg)[5], f2 v) {
  reg[SLOT] = v;
  C.rg[(RID * 5 + SLOT) * 32] = v;
}
template <int RID, int SLOT, int S0, class CT>
__device__ __forceinline__ f2 ring_get(const CT& C, const f2 (&reg)[5]) {
  constexpr bool age1_in_reg = ((RING_REG1 >> RID) & 1u) != 0u && SLOT == (S0 + 4) % 5;
  if constexpr (SLOT != S0 && !age1_in_reg) return C.rg[(RID * 5 + SLOT) * 32];
  else return reg[SLOT];
}
template <int W, int SLOT, int S0, class CT, class S>
__device__ __forceinline__ f2 runA(const CT& C, const Lane<S>& L) {
  if constexpr (W == 2) return ring_get<R_A2, SLOT, S0>(C, L.a2);
  else if constexpr (W == 1) return ring_get<R_A1, SLOT, S0>(C, L.a1);
  else return 0ull;
}
template <int W, int SLOT, int S0, class CT, class S>
__device__ __forceinline__ f2 runB(const CT& C, const Lane<S>& L) {
  if constexpr (W == 2) return ring_get<R_B2, SLOT, S0>(C, L.b2);
  else if constexpr (W == 1) return ring_get<R_B1, SLOT, S0>(C, L.b1);
  else return 0ull;
}
template <int W, int SLOT, int S0, class CT, class S>
__device__ __forceinline__ f2 runQ(const CT& C, const Lane<S>& L) {
  if constexpr (W == 2) return ring_get<R_Q2, SLOT, S0>(C, L.q2);
  else if constexpr (W == 1) return ring_get<R_Q1, SLOT, S0>(C, L.q1);
  else return 0ull;
}

struct Normal2 {
  f2 nx, ny, nz, slope, rough;
  unsigned flag;  // bit0: row x, bit1: row y could not be certified
};

// acos on [0,1] for both rows: sqrt(1-x) * P7(x) (Abramowitz-Stegun 4.4.46 form, coefficients refitted for
// relative error; float32 evaluation: max abs error 2.2e-7, max rel. error 1.7e-7).  Branch-free.
__device__ __forceinline__ f2 acos2(const FusedArgs& A, f2 x) {
  const f2 u = csub2(A.k_one, x);
  const f2 sq = mk(sqrt_a(lo(u)), sqrt_a(hi(u)));
  f2 p = fma2kc(x, A.k_p7, A.k_p6);
  p = fma2c(p, x, A.k_p5);
  p = fma2c(p, x, A.k_p4);
  p = fma2c(p, x, A.k_p3);
  p = fma2c(p, x, A.k_p2);
  p = fma2c(p, x, A.k_p1);
  p = fma2c(p, x, A.k_p0);
  return mul2(sq, p);
}

// h >= 0 ? a : b as one FSEL on a comparison ptxas shares between the selects of a row (a C conditional becomes a MOV and a
// predicated MOV)
__device__ __forceinline__ float sel_ge0(float h, float a, float b) {
  float r;
  asm("{ .reg .pred p; setp.ge.f32 p, %1, 0f00000000; selp.f32 %0, %2, %3, p; }" : "=f"(r) : "f"(h), "f"(a), "f"(b));
  return r;
}
// NaN-propagating min (a NaN margin must fail the certification)
__device__ __forceinline__ float min2n(float a, float b) {
  float r;
  asm("min.NaN.f32 %0, %1, %2;" : "=f"(r) : "f"(a), "f"(b));
  return r;
}
// Closed-form smallest eigenpair of the scatter matrix [[a,0,p],[0,a,q],[p,q,c]] of a full disk
// window for both rows of the lane, slope and roughness layers, and the certification of all of it.
// D = sqrt(hh) (MUFU.SQRT) and g2 / dph (MUFU.RCP) carry a relative error of 2^-23 without a Newton correction, which what they
// feed tolerates: lambda0 is certified against 1e-5 cmag, s = 1 - n_z against a relative error budget of 2.5e-6, and
// theta = atan(g/m) moves by sin(theta) cos(theta) eps.
__device__ __forceinline__ Normal2 finish_normal2(const FusedArgs& A, f2 Sw, f2 Sk, f2 Sl, f2 Sww, f2 ec) {
  Normal2 o;
  const f2 mw = mul2c(Sw, A.k_invN);
  const f2 c = fma2(negf2(mw), mw, mul2c(Sww, A.k_invN));  // Czz = Sww/N - (Sw/N)^2
  const f2 p = mul2c(Sk, A.k_kp), q = mul2c(Sl, A.k_kp);               // Cxz, Cyz
  const f2 g2 = fma2(p, p, mul2(q, q));
  const f2 h = fma2kc(negf2(c), A.k_half, A.k_half_a);                  // (a - c)/2
  const f2 hh = fma2(h, h, g2);
  const f2 D = mk(sqrt_a(lo(hh)), sqrt_a(hi(hh)));
  const float h0 = lo(h), h1 = hi(h);
  const f2 dph = add2(D, mk(fabsf(h0), fabsf(h1)));
  const f2 rq = mk(rcp_a(lo(dph)), rcp_a(hi(dph)));
  const f2 qq = mul2(g2, rq);
  const f2 m = mk(sel_ge0(h0, lo(dph), lo(qq)), sel_ge0(h1, hi(dph), hi(qq)));  // a - lambda0
  const f2 cmag = mk(sel_ge0(h0, lo(c), A.a_cov), sel_ge0(h1, hi(c), A.a_cov));
  const f2 lam0 = sub2(cmag, qq);                                  // smallest eigenvalue
  const f2 m2 = mul2(m, m);
  const f2 nn = add2(m2, g2);
  // n_z = 1 - s with s = g^2 / (N (m + N)), N = sqrt(m^2 + g^2), for every inclination (the identity 1 - m/N =
  // (N^2 - m^2) / (N (N + m)); no cancellation, relative error of s ~4.5e-7 from MUFU.SQRT and MUFU.RCP)
  const f2 Nn = mk(sqrt_a(lo(nn)), sqrt_a(hi(nn)));
  const f2 den = mul2(Nn, add2(m, Nn));
  const f2 rden = mk(rcp_a(lo(den)), rcp_a(hi(den)));
  const f2 s = mul2(g2, rden);
  const f2 nz = csub2(A.k_one, s);  // s >= 0: n_z <= 1; the subtraction rounds n_z to float32 exactly like the reference's layer
  {
    const f2 rn = mk(rcp_a(lo(Nn)), rcp_a(hi(Nn)));  // only the instantiation that stores the normals keeps this
    o.nx = mul2(negf2(p), rn);
    o.ny = mul2(negf2(q), rn);
  }
  // roughness = sqrt(lambda0 * N/(N-1)); lambda0 is a difference of two terms of size cmag
  const f2 rr2 = mul2c(lam0, A.k_nnm1);
  const f2 r = mk(sqrt_a(fmaxf(lo(rr2), 0.f)), sqrt_a(fmaxf(hi(rr2), 0.f)));
  const f2 thr = mul2c(mul2(cmag, cmag), A.k_rough_thr);
  // ---- certification (packed margins; a NaN margin fails) ----------------------------------------------------------
  // rank / roughness: lambda0 must stand clear of its cancellation error (1e-5 cmag), of the reference's rank-threshold
  // region (1e-10 a) and of what the roughness tolerance allows (thr); conditioning: the eigen-gap min(2D, m) against
  // the matrix scale.  Invalid windows (NaN/Inf moments) fail through NaN; exactly flat windows (Sww == 0) are exact;
  // holes (invalid centre) need no second opinion.
  const f2 lbase = fma2kc(cmag, A.k_1em5, A.k_1em10a);
  const f2 t1 = sub2(lam0, mk(fmaxf(lo(lbase), lo(thr)), fmaxf(hi(lbase), hi(thr))));
  // the eigen-gap is min(2D, a - lambda0) = a - lambda0 = m: m = D + h <= 2D because D = sqrt(h^2 + g^2) >= |h|
  const f2 t2 = fma2k(mk(fmaxf(A.a_cov, lo(c)), fmaxf(A.a_cov, hi(c))), A.k_mcond, m);
  const f2 inval = sub2(ec, ec);
  // a row fails unless its margin is positive or its window is exactly flat, and a hole is never flagged; the comparisons
  // are combined with non-short-circuit & so that they stay predicate logic (no branch, no bytes of bools to repack)
  const bool fail0 = !(min2n(lo(t1), lo(t2)) > 0.f) & (lo(Sww) != 0.f) & (lo(inval) == 0.f);
  const bool fail1 = !(min2n(hi(t1), hi(t2)) > 0.f) & (hi(Sww) != 0.f) & (hi(inval) == 0.f);
  unsigned flag = (unsigned)fail0 | ((unsigned)fail1 << 1);
  // where acos amplifies one ulp of n_z beyond half the slope layer's tolerance (s < k_nz_check: theta < 0.012 rad at crit
  // >= 1 rad, every theta up to just past crit below crit ~0.35 rad) certify its float32 rounding.
  // n_z = 1 - s is rounded to float32 with spacing 2^-24: flag when s, known to relative error eps, may sit on the other
  // side of a rounding boundary (eps: the first moments carry <= 2.5e-6*sqrt(Sww) absolute error).  Both rows at once.
  const bool cx = lo(s) < A.k_nz_check && lo(Sww) > 0.f, cy = hi(s) < A.k_nz_check && hi(Sww) > 0.f;
  if (cx || cy) {
    const f2 qv = mul2c(s, A.k_2p24);
    const f2 fr = sub2(qv, mk(floorf(lo(qv)), floorf(hi(qv))));
    const f2 gm2 = fma2(Sk, Sk, mul2(Sl, Sl));
    const f2 ratio = mul2(Sww, mk(rcp_a(fmaxf(lo(gm2), 1e-36f)), rcp_a(fmaxf(hi(gm2), 1e-36f))));
    const f2 eps = fma2kc(mk(sqrt_a(lo(ratio)), sqrt_a(hi(ratio))), A.k_7p1em6, A.k_2em6);
    const f2 bound = fma2c(qv, eps, A.k_bmargin);
    const f2 dist = sub2c(fr, A.k_half);
    if (cx && fabsf(lo(dist)) <= lo(bound)) flag |= 1u;
    if (cy && fabsf(hi(dist)) <= hi(bound)) flag |= 2u;
  }
  const f2 theta = acos2(A, nz);
  // layer = x < crit ? 1 - x/crit : 0  ==  max(1 - x/crit, 0)  ==  sat(1 - x/crit) for x >= 0
  // a hole (invalid centre: NaN, or Inf - Inf) has no normal: slope and roughness stay NaN
  // (SlopeFilter.cpp:71, RoughnessFilter.cpp:84) and the cell is not flagged
  o.nz = add2(nz, inval);
  o.slope = add2(mk(fma_sat1(lo(theta), A.minv_slope_crit), fma_sat1(hi(theta), A.minv_slope_crit)), inval);
  o.rough = add2(mk(fma_sat1(lo(r), A.minv_rough_crit), fma_sat1(hi(r), A.minv_rough_crit)), inval);
  o.flag = flag;
  return o;
}

// Rare paths kept out of line so that the five unrolled march phases stay small.
//
// Work-list append.  A warp owns a private chunk of LIST_CHUNK list entries at a time and fills it without atomics; only when an
// append does not fit into what is left of the chunk does lane 0 reserve the next chunk from the global cursor (count[0]) — one
// returning atomic per ~LIST_CHUNK flagged cells instead of one per flagged march step, so the march does not wait on L2 atomics.
// The unused tail of a chunk is padded with LIST_INVALID, which the consumers skip; count[1] tallies the flagged cells themselves
// (fire-and-forget reduction).  The chunk cursor of a warp lives in its shared-memory block (warp-uniform, rare path).
__device__ __noinline__ void append_flagged(unsigned* count, unsigned* list, unsigned cap, unsigned lstate, int lane, unsigned cell,
                                            unsigned fl) {
  const unsigned fl0 = (fl & 1u) | ((fl >> 1) & 2u), fl1 = ((fl >> 1) & 1u) | ((fl >> 2) & 2u);  // per row: bit0 normals, bit1 step
  const unsigned b0 = __ballot_sync(FULL, fl0 != 0u), b1 = __ballot_sync(FULL, fl1 != 0u);
  const unsigned n = (unsigned)(__popc(b0) + __popc(b1));
  unsigned base, pos;
  asm volatile("ld.shared.v2.u32 {%0, %1}, [%2];" : "=r"(base), "=r"(pos) : "r"(lstate) : "memory");
  if (pos + n > LIST_CHUNK) {  // also the first append of a warp (pos starts at LIST_CHUNK)
    for (unsigned i = pos + lane; i < LIST_CHUNK; i += 32) list[base + i] = LIST_INVALID;
    if (lane == 0) base = atomicAdd(count, LIST_CHUNK);
    base = __shfl_sync(FULL, base, 0);
    pos = 0;
    if (base + LIST_CHUNK > cap) {  // cannot happen with the capacity fused_list_capacity() prescribes; never write past the list
      if (lane == 0) {
        atomicExch(count + 2, 1u);
        asm volatile("st.shared.v2.u32 [%0], {%1, %2};" ::"r"(lstate), "r"(0u), "r"(LIST_CHUNK) : "memory");
      }
      __syncwarp();
      return;
    }
  }
  const unsigned lower = (1u << lane) - 1u;
  if (fl0) list[base + pos + __popc(b0 & lower)] = cell | (fl0 << 30);
  if (fl1) list[base + pos + __popc(b0) + __popc(b1 & lower)] = (cell + 1u) | (fl1 << 30);
  if (lane == 0) {
    asm volatile("st.shared.v2.u32 [%0], {%1, %2};" ::"r"(lstate), "r"(base), "r"(pos + n) : "memory");
    atomicAdd(count + 1, n);  // result unused: a reduction
  }
  __syncwarp();
}
// End of a warp's work: pad what is left of its chunk.
__device__ __noinline__ void finish_list(unsigned* list, unsigned lstate, int lane) {
  unsigned base, pos;
  asm volatile("ld.shared.v2.u32 {%0, %1}, [%2];" : "=r"(base), "=r"(pos) : "r"(lstate) : "memory");
  for (unsigned i = pos + lane; i < LIST_CHUNK; i += 32) list[base + i] = LIST_INVALID;
}
__device__ __noinline__ void store_normals(float* pnx, float* pny, float* pnz, bool ok, unsigned oc, f2 nx, f2 ny, f2 nz) {
  if (!ok) return;
  *reinterpret_cast<f2*>(pnx + oc) = nx;
  *reinterpret_cast<f2*>(pny + oc) = ny;
  *reinterpret_cast<f2*>(pnz + oc) = nz;
}

// Column tips of a chunk (CH march steps; column `cb` arrives at phase 0).  Lane ph < CH writes the word of phase ph into the
// padding of the chunk's TMA stage: byte 0/1 = pass-1 tips (0,-2)/(0,+2) of column js = cb + ph - 2, byte 2/3 = pass-2 tips of
// column jo = cb + ph - 4; 0x00 where the on-circle offset belongs to the window (colmask bit set), 0xff where it does not.
// `colmask` is the unit's map's table.
__device__ __forceinline__ void fill_colmask(const FusedArgs& A, const unsigned char* colmask, unsigned stage_addr, int cb, int lane) {
  if (lane < CH) {
    const int js = cb + lane - 2, jo = js - 2;
    const unsigned x = (js >= 0 && js < A.cols_total) ? colmask[js] : 0u;
    const unsigned y = (jo >= 0 && jo < A.cols_total) ? colmask[jo] : 0u;
    const unsigned w = ((x & 1u) ? 0u : 0xffu) | ((x & 2u) ? 0u : 0xff00u) | ((y & 4u) ? 0u : 0xff0000u) | ((y & 8u) ? 0u : 0xff000000u);
    asm volatile("st.shared.u32 [%0], %1;" ::"r"(stage_addr + STAGE_PAD + lane * 4), "r"(w) : "memory");
  }
}

template <class S>
struct StepCtx {
  const FusedArgs& A;
  unsigned e_base;    // shared address of stage 0 of the warp's TMA ring
  unsigned e_lane;    // shared address of the lane's first staged row in stage 0 / column 0
  unsigned sh_lane;   // shared address of the lane's first step_height row in buffer 0
  int lane;
  int s0;             // first row held by the warp (strip row 0 = output row -2)
  int q0, q1;         // output columns of the unit
  f2 tipU1, tipD1;    // pass-1 row tips: +0.0 where the on-circle offset (-2,0)/(+2,0) belongs to the window, NaN where not
  f2 tipU2, tipD2;    // same for pass 2
  f2 cntU2, cntD2;    // pass-2 row tips as count weights: 1.0 where the offset belongs to the window, 0.0 where not
  f2* rg;             // the lane's element of ring 0 / slot 0 in shared memory (rings are 32 lanes x 8 bytes apart)
  unsigned lstate;    // shared address of the warp's work-list cursor {chunk base, entries used}
  unsigned oc;        // running output element offset (column jo, lane's first row); a launch covers < 2^30 cells.  It runs
                      // 8 columns ahead of the first store of a unit (wraps below zero; never dereferenced then)
  unsigned out_len;   // output columns of the unit (q1 - q0) the lane stores: 0 unless it produces output rows (lanes 1..30
                      // inside the map), so that one unsigned compare per step decides a store
};

// One march step: column ce = q0 - 4 + t arrives.  PH = t % 5.
template <class S, int PH, bool KN>
__device__ __forceinline__ void march_step(StepCtx<S>& C, Lane<S>& L, int t, unsigned stage) {
  const FusedArgs& A = C.A;
  constexpr int S0 = PH, S1 = (PH + 4) % 5, S2 = (PH + 3) % 5, S3 = (PH + 2) % 5, S4 = (PH + 1) % 5;  // slot of age 0..4
  const int ce = C.q0 - 4 + t;
  const unsigned oc = C.oc;  // element offset of column jo = ce - 4, lane's first row
  C.oc += (unsigned)A.rows;
  // ---- stage A: the arriving elevation column -------------------------------------------------
  float z[6];
  f2 ZM2, Z0, ZP2;
  {
    const unsigned a = C.e_lane + stage * STAGE_BYTES + PH * (EROWS * 4);
    ZM2 = lds64(a); Z0 = lds64(a + 8); ZP2 = lds64(a + 16);
    z[0] = lo(ZM2); z[1] = hi(ZM2); z[2] = lo(Z0); z[3] = hi(Z0); z[4] = lo(ZP2); z[5] = hi(ZP2);
  }
  L.e[S0] = Z0;
  if constexpr (S::NEED_N1 || S::NEED_N2) {
    // the row pairs (z1,z2) and (z3,z4) straddle two registers pairs: scalar subtractions land in aligned pairs without moves
    const f2 D1 = mk(__fsub_rn(z[3], z[2]), __fsub_rn(z[4], z[3])), Dm1 = mk(__fsub_rn(z[1], z[2]), __fsub_rn(z[2], z[3]));
    const f2 A1 = add2(D1, Dm1);
    const f2 B1 = mk(__fsub_rn(z[3], z[1]), __fsub_rn(z[4], z[2]));
    const f2 Q1 = fma2(D1, D1, mul2(Dm1, Dm1));
    if constexpr (S::NEED_N1) { ring_put<R_A1, S0>(C, L.a1, A1); ring_put<R_B1, S0>(C, L.b1, B1); ring_put<R_Q1, S0>(C, L.q1, Q1); }
    if constexpr (S::NEED_N2) {
      const f2 D2 = sub2(ZP2, Z0), Dm2 = sub2(ZM2, Z0);
      ring_put<R_A2, S0>(C, L.a2, add2(A1, add2(D2, Dm2)));
      ring_put<R_B2, S0>(C, L.b2, fma2k(sub2(ZP2, ZM2), A.k_two, B1));
      ring_put<R_Q2, S0>(C, L.q2, fma2(D2, D2, fma2(Dm2, Dm2, Q1)));
    }
  }
  {
    float cmn[2], cmx[2], pmn[2], pmx[2];
    // excluded on-circle tips become NaN (x + NaN), included ones pass through (x + 0): both rows in one FADD2
    f2 TU = 0ull, TD = 0ull;
    if constexpr (S::TIP1) { TU = add2(ZM2, C.tipU1); TD = add2(ZP2, C.tipD1); }
    // the three-row windows of the two rows, {z1,z2,z3} and {z2,z3,z4}, share min/max(z2, z3): one FMNMX each instead of
    // two (minNum/maxNum are associative and commutative: a total order in which -0 < +0, NaN operands skipped)
    const float mn23 = fminf(z[2], z[3]), mx23 = fmaxf(z[2], z[3]);
    const float lo3r[2] = {fminf(z[1], mn23), fminf(mn23, z[4])}, hi3r[2] = {fmaxf(z[1], mx23), fmaxf(mx23, z[4])};
#pragma unroll
    for (int r = 0; r < 2; ++r) {
      const float lo3 = lo3r[r], hi3 = hi3r[r];
      if constexpr (S::W11 == 1) { cmn[r] = lo3; cmx[r] = hi3; }
      else if constexpr (S::W11 >= 0) { cmn[r] = colmin_w<(S::W11 < 0 ? 0 : S::W11)>(z, r); cmx[r] = colmax_w<(S::W11 < 0 ? 0 : S::W11)>(z, r); }
      else { cmn[r] = cmx[r] = 0.f; }
      float mn = lo3, mx = hi3;
      if constexpr (S::W10 == 2) {
        mn = min3n(mn, z[r], z[r + 4]);
        mx = max3n(mx, z[r], z[r + 4]);
      } else if constexpr (S::TIP1) {
        const float tu = r ? hi(TU) : lo(TU), td = r ? hi(TD) : lo(TD);
        mn = min3n(mn, tu, td);
        mx = max3n(mx, tu, td);
      }
      pmn[r] = mn;
      pmx[r] = mx;
    }
    ring_put<R_C1MN, S0>(C, L.c1mn, mk(cmn[0], cmn[1])); ring_put<R_C1MX, S0>(C, L.c1mx, mk(cmx[0], cmx[1]));
    L.p1mn[S0] = mk(pmn[0], pmn[1]); L.p1mx[S0] = mk(pmx[0], pmx[1]);
  }
  if (t < 4) return;  // rings not primed yet
  // ---- stage B: step_height of column js = ce - 2 (ages: js+1 -> 1, js -> 2, js-1 -> 3) ---------
  const unsigned shcol = C.sh_lane + (PH % NSHB) * SHBUF_BYTES;
  // column tips of this step: one broadcast word from the stage's padding, a byte per tip (0x00 = inside the window,
  // 0xff = excluded); replicated into all four bytes it is +0.0 or a NaN to add to the tip value (see fill_colmask)
  unsigned cmw = 0u;
  if constexpr (S::MASKS) asm volatile("ld.shared.u32 %0, [%1];" : "=r"(cmw) : "r"(C.e_base + stage * STAGE_BYTES + (STAGE_PAD + PH * 4)));
  f2 V0;
  {
    float mn2[2], mx2[2];
    f2 c1mnA = 0ull, c1mnB = 0ull, c1mxA = 0ull, c1mxB = 0ull;
    if constexpr (S::W11 >= 0) {
      c1mnA = ring_get<R_C1MN, S1, S0>(C, L.c1mn); c1mnB = ring_get<R_C1MN, S3, S0>(C, L.c1mn);
      c1mxA = ring_get<R_C1MX, S1, S0>(C, L.c1mx); c1mxB = ring_get<R_C1MX, S3, S0>(C, L.c1mx);
    }
    f2 TL1 = L.e[S4], TR1 = L.e[S0];
    if constexpr (S::TIP1) {
      TL1 = add2(TL1, bc(__uint_as_float(__byte_perm(cmw, 0u, 0x0000))));
      TR1 = add2(TR1, bc(__uint_as_float(__byte_perm(cmw, 0u, 0x1111))));
    }
#pragma unroll
    for (int r = 0; r < 2; ++r) {
      auto R = [&](f2 v) { return r ? hi(v) : lo(v); };
      float mn = R(L.p1mn[S2]), mx = R(L.p1mx[S2]);
      if constexpr (S::W11 >= 0) {
        mn = min3n(mn, R(c1mnA), R(c1mnB));
        mx = max3n(mx, R(c1mxA), R(c1mxB));
      }
      if constexpr (S::W12 == 0 || S::TIP1) {
        const float tl = R(TL1), tr = R(TR1);
        mn = min3n(mn, tl, tr);
        mx = max3n(mx, tl, tr);
      }
      mn2[r] = mn;
      mx2[r] = mx;
    }
    // centre gate (StepFilter.cpp:113): an invalid centre (NaN, or Inf: Inf - Inf) leaves step_height NaN
    const f2 zc = L.e[S2];
    V0 = add2(sub2(mk(mx2[0], mx2[1]), mk(mn2[0], mn2[1])), sub2(zc, zc));
    sts64(shcol + 8, V0);  // buffer row 0 is strip row -2
  }
  __syncwarp();
  float v[6], f[6];
  f2 SU = 0ull, SD = 0ull;
  {
    const f2 VM2 = lds64(shcol), VP2 = lds64(shcol + 16);
    if constexpr (S::TIP2) { SU = add2(VM2, C.tipU2); SD = add2(VP2, C.tipD2); }
    v[0] = lo(VM2); v[1] = hi(VM2); v[2] = lo(V0); v[3] = hi(V0); v[4] = lo(VP2); v[5] = hi(VP2);
#pragma unroll
    for (int k = 0; k < 6; ++k) f[k] = gtf(v[k], A.step_cmp);
  }
  {
    float smx[2], pmx[2], sc[2];
    const float fmid = f[2] + f[3];
    const float c3[2] = {f[1] + fmid, fmid + f[4]};  // counts are small integers: any association is exact
    f2 PC = mk(c3[0], c3[1]);
    const float vx23 = fmaxf(v[2], v[3]);  // shared by the windows of both rows, as in stage A
    const float hi3r[2] = {fmaxf(v[1], vx23), fmaxf(vx23, v[4])};
#pragma unroll
    for (int r = 0; r < 2; ++r) {
      const float hi3 = hi3r[r];
      if constexpr (S::W21 == 1) { smx[r] = hi3; sc[r] = c3[r]; }
      else if constexpr (S::W21 >= 0) { smx[r] = colmax_w<(S::W21 < 0 ? 0 : S::W21)>(v, r); sc[r] = colcnt_w<(S::W21 < 0 ? 0 : S::W21)>(f, r); }
      else { smx[r] = 0.f; sc[r] = 0.f; }
      float mx = hi3;
      if constexpr (S::W20 == 2) {
        mx = max3n(mx, v[r], v[r + 4]);
      } else if constexpr (S::TIP2) {
        const float tu = r ? hi(SU) : lo(SU), td = r ? hi(SD) : lo(SD);
        mx = max3n(mx, tu, td);
      }
      pmx[r] = mx;
    }
    if constexpr (S::W20 == 2) {
      PC = add2(PC, add2(mk(f[0], f[1]), mk(f[4], f[5])));
    } else if constexpr (S::TIP2) {  // NaN > crit is false
      PC = fma2(mk(f[0], f[1]), C.cntU2, fma2(mk(f[4], f[5]), C.cntD2, PC));  // the tips' flags exist already: weight them (0/1, exact)
    }
    L.sh[S0] = V0;
    ring_put<R_S3MX, S0>(C, L.s3mx, mk(smx[0], smx[1])); ring_put<R_S3C, S0>(C, L.s3c, mk(sc[0], sc[1]));
    L.pcmx[S0] = mk(pmx[0], pmx[1]); L.pcc[S0] = PC;
  }
  // ---- normals / slope / roughness of column jn = ce - 2 (ages: l = 2 - age) -------------------
  const int jn = ce - 2;
  if (jn >= C.q0 && jn < C.q1) {
    const f2 ec = L.e[S2];
    f2 Sw = runA<S::WN0, S2, S0>(C, L), Sk = runB<S::WN0, S2, S0>(C, L), Sww = runQ<S::WN0, S2, S0>(C, L);
    f2 Sl = 0ull;
    if constexpr (S::WN1 >= 0) {
      const f2 dR = sub2(L.e[S1], ec), dL = sub2(L.e[S3], ec);
      const f2 aR = runA<S::WN1, S1, S0>(C, L), aL = runA<S::WN1, S3, S0>(C, L);
      const f2 tR = kfma2(A.k_m1, dR, aR), tL = kfma2(A.k_m1, dL, aL);
      Sw = add2(Sw, add2(tR, tL));
      Sl = sub2(tR, tL);
      Sk = add2(Sk, add2(runB<S::WN1, S1, S0>(C, L), runB<S::WN1, S3, S0>(C, L)));
      Sww = add2(Sww, fma2(dR, add2(aR, tR), runQ<S::WN1, S1, S0>(C, L)));
      Sww = add2(Sww, fma2(dL, add2(aL, tL), runQ<S::WN1, S3, S0>(C, L)));
    }
    if constexpr (S::WN2 >= 0) {
      const f2 dR = sub2(L.e[S0], ec), dL = sub2(L.e[S4], ec);
      const f2 aR = runA<S::WN2, S0, S0>(C, L), aL = runA<S::WN2, S4, S0>(C, L);
      const f2 tR = kfma2(A.k_m0, dR, aR), tL = kfma2(A.k_m0, dL, aL);
      Sw = add2(Sw, add2(tR, tL));
      Sl = kfma2(A.k_two, sub2(tR, tL), Sl);
      Sk = add2(Sk, add2(runB<S::WN2, S0, S0>(C, L), runB<S::WN2, S4, S0>(C, L)));
      Sww = add2(Sww, fma2(dR, add2(aR, tR), runQ<S::WN2, S0, S0>(C, L)));
      Sww = add2(Sww, fma2(dL, add2(aL, tL), runQ<S::WN2, S4, S0>(C, L)));
    }
    // row index grows toward -x and column index toward -y: kp carries that sign and 1/N
    const Normal2 n = finish_normal2(A, Sw, Sk, Sl, Sww, ec);
    L.dslope[S0] = n.slope;
    L.drough[S0] = n.rough;
    L.dflag[S0] = n.flag;
    if constexpr (KN)  // column jn is two columns ahead of the column the step layer is stored for
      store_normals(A.nx, A.ny, A.nz, (unsigned)(t - 6) < C.out_len, oc + 2u * (unsigned)A.rows, n.nx, n.ny, n.nz);
  }
  if (t < 8) return;
  // ---- stage C: step layer of column jo = ce - 4 and the fuse ----------------------------------
  if (ce - 4 >= C.q1) return;
  const bool st_ok = (unsigned)(t - 8) < C.out_len;  // column jo = ce - 4 = q0 + t - 8 belongs to the unit
  {
    float mx2[2];
    f2 TL2 = L.sh[S4], TR2 = L.sh[S0];
    if constexpr (S::TIP2) {
      TL2 = add2(TL2, bc(__uint_as_float(__byte_perm(cmw, 0u, 0x2222))));
      TR2 = add2(TR2, bc(__uint_as_float(__byte_perm(cmw, 0u, 0x3333))));
    }
    f2 s3mxA = 0ull, s3mxB = 0ull;
    if constexpr (S::W21 >= 0) { s3mxA = ring_get<R_S3MX, S1, S0>(C, L.s3mx); s3mxB = ring_get<R_S3MX, S3, S0>(C, L.s3mx); }
    f2 CNT = L.pcc[S2];
    if constexpr (S::W21 >= 0) CNT = add2(CNT, add2(ring_get<R_S3C, S1, S0>(C, L.s3c), ring_get<R_S3C, S3, S0>(C, L.s3c)));
    if constexpr (S::W22 == 0 || S::TIP2)
      CNT = add2(CNT, add2(mk(gtf(lo(TL2), A.step_cmp), gtf(hi(TL2), A.step_cmp)), mk(gtf(lo(TR2), A.step_cmp), gtf(hi(TR2), A.step_cmp))));
#pragma unroll
    for (int r = 0; r < 2; ++r) {
      auto R = [&](f2 x) { return r ? hi(x) : lo(x); };
      float mx = R(L.pcmx[S2]);
      if constexpr (S::W21 >= 0) mx = max3n(mx, R(s3mxA), R(s3mxB));
      if constexpr (S::W22 == 0 || S::TIP2) mx = max3n(mx, R(TL2), R(TR2));
      mx2[r] = mx;
    }
    const f2 MX = mk(mx2[0], mx2[1]);
    const f2 stepMax = mk(fmaxf(mx2[0], 0.0f), fmaxf(mx2[1], 0.0f));
    const f2 prod = mul2(mul2c(CNT, A.k_inv_ncrit), stepMax);
    const f2 st = mk(fminf(lo(stepMax), lo(prod)), fminf(hi(stepMax), hi(prod)));
    // st < crit ? 1 - st/crit : 0 ; no finite step_height in the window (mx is NaN) -> layer stays NaN (StepFilter.cpp:169)
    const f2 outv = add2(mk(fma_sat1(lo(st), A.minv_step_crit), fma_sat1(hi(st), A.minv_step_crit)), sub2(MX, MX));  // mx NaN (or Inf - Inf) keeps the layer NaN
    const f2 sl = L.dslope[S2], ro = L.drough[S2];
    const unsigned nf = L.dflag[S2];
    const f2 tr = kmul2(A.k_fuse_w, add2(add2(sl, outv), ro));
    if (st_ok) {
      *reinterpret_cast<f2*>(A.slope + oc) = sl;
      *reinterpret_cast<f2*>(A.rough + oc) = ro;
      *reinterpret_cast<f2*>(A.step + oc) = outv;
      *reinterpret_cast<f2*>(A.trav + oc) = tr;
    }
    // certified slow path: append flagged cells (bit 30: normals part, bit 31: step part).  An infinite elevation that reached
    // the step window (maxNum skips NaN: the larger row maximum is +Inf iff one of them is) is sorted out there as well.
    const bool any_inf = fmaxf(mx2[0], mx2[1]) > 3.0e38f;
    if (__any_sync(FULL, st_ok && (nf != 0u || any_inf))) {
      const unsigned sflag = (mx2[0] > 3.0e38f ? 1u : 0u) | (mx2[1] > 3.0e38f ? 2u : 0u);
      append_flagged(A.count, A.list, A.cap, C.lstate, C.lane, oc, st_ok ? (nf | (sflag << 2)) : 0u);  // bits 0/1: normals part of row x/y, bits 2/3: step part
    }
  }
}

template <class S, bool KN>
__global__ void __maxnreg__(168) k_chain_fused(const __grid_constant__ CUtensorMap map, FusedArgs A) {
  extern __shared__ __align__(128) unsigned char smem_raw[];
  const int warp = __shfl_sync(FULL, (int)(threadIdx.x >> 5), 0);  // provably warp-uniform: uniform datapath for the control flow
  const int lane = threadIdx.x & 31;
  const unsigned wbase = smem_u32(smem_raw) + warp * WARP_SMEM_BYTES;
  const unsigned ering = wbase;
  const unsigned shbuf = wbase + NST * STAGE_BYTES;
  const unsigned bar0 = wbase + WARP_AUX_OFF;
  if (lane == 0) {
    for (int s = 0; s < NST; ++s) mbar_init(bar0 + 8 * s, 1);
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }
  __syncwarp();

  asm volatile("griddepcontrol.launch_dependents;");  // tier 2 (a programmatic dependent launch) may be set up while this grid runs
  const int total_warps = gridDim.x * WARPS_PER_CTA;
  const int gwarp = blockIdx.x * WARPS_PER_CTA + warp;
  const int nunits = A.lvl_unit0[NLVL];
  unsigned kglob = 0;  // chunks consumed so far by this warp (stage = kglob % NST, parity = (kglob / NST) & 1)

  Lane<S> L{};  // the warm-up steps of a unit read ring slots before they are written (results discarded)
  StepCtx<S> C{A, ering, ering + lane * 8u, shbuf + lane * 8u, lane, 0, 0, 0, 0ull, 0ull, 0ull, 0ull, 0ull, 0ull,
               reinterpret_cast<f2*>(smem_raw + warp * WARP_SMEM_BYTES + WARP_RING_OFF) + lane,
               bar0 + 8 * NST, 0u, 0u};
  if (lane == 0) asm volatile("st.shared.v2.u32 [%0], {%1, %2};" ::"r"(C.lstate), "r"(0u), "r"(LIST_CHUNK) : "memory");  // no chunk yet
  __syncwarp();

  int unit = gwarp;  // the first unit is static, the rest come from the queue
  while (unit < nunits) {
    int next = 0;
    if (lane == 0) next = total_warps + (int)atomicAdd(A.queue, 1u);  // consumed after this unit: the latency hides behind it
    int u0 = A.lvl_unit0[0], c0 = A.lvl_col0[0], c1 = A.lvl_col0[1], len = A.lvl_len[0], ns = A.lvl_nseg[0];
    if (unit >= A.lvl_unit0[1]) { u0 = A.lvl_unit0[1]; c0 = A.lvl_col0[1]; c1 = A.lvl_col0[2]; len = A.lvl_len[1]; ns = A.lvl_nseg[1]; }
    if (unit >= A.lvl_unit0[2]) { u0 = A.lvl_unit0[2]; c0 = A.lvl_col0[2]; c1 = A.lvl_col0[3]; len = A.lvl_len[2]; ns = A.lvl_nseg[2]; }
    if (unit >= A.lvl_unit0[3]) { u0 = A.lvl_unit0[3]; c0 = A.lvl_col0[3]; c1 = A.lvl_col0[4]; len = A.lvl_len[3]; ns = A.lvl_nseg[3]; }
    const int u = unit - u0, upm = A.nstrips * ns;
    const int mapi = u / upm, um = u - mapi * upm;
    const int strip = um % A.nstrips, seg = um / A.nstrips;
    C.s0 = strip * OROWS - 2;
    C.q0 = A.out_col0 + c0 + seg * len;
    C.q1 = min(C.q0 + len, A.out_col0 + c1);
    const int nsteps = (C.q1 - C.q0) + 8;
    const int nchunks = (nsteps + CH - 1) / CH;
    const int row0 = C.s0 + 2 * lane;
    C.out_len = (lane >= 1 && lane <= 30 && row0 < A.rows) ? (unsigned)(C.q1 - C.q0) : 0u;
    C.oc = (unsigned)mapi * A.map_cells + (unsigned)(C.q0 - A.out_col0 - 8) * (unsigned)A.rows + (unsigned)row0;
    // the unit's map's mask tables (one per map when the maps sit at their own positions): looked up once per unit
    const unsigned char* const colmask = A.colmask + (size_t)mapi * A.colmask_stride;
    if constexpr (S::MASKS) {
      const unsigned char* const rowmask = A.rowmask + (size_t)mapi * A.rowmask_stride;
      const unsigned rm0 = (row0 >= 0 && row0 < A.rows) ? rowmask[row0] : 0u;
      const unsigned rm1 = (row0 + 1 >= 0 && row0 + 1 < A.rows) ? rowmask[row0 + 1] : 0u;
      const float qn = __int_as_float(0x7fc00000);
      C.tipU1 = mk((rm0 & 1u) ? 0.f : qn, (rm1 & 1u) ? 0.f : qn);
      C.tipD1 = mk((rm0 & 2u) ? 0.f : qn, (rm1 & 2u) ? 0.f : qn);
      C.tipU2 = mk((rm0 & 4u) ? 0.f : qn, (rm1 & 4u) ? 0.f : qn);
      C.tipD2 = mk((rm0 & 8u) ? 0.f : qn, (rm1 & 8u) ? 0.f : qn);
      C.cntU2 = mk((rm0 & 4u) ? 1.f : 0.f, (rm1 & 4u) ? 1.f : 0.f);
      C.cntD2 = mk((rm0 & 8u) ? 1.f : 0.f, (rm1 & 8u) ? 1.f : 0.f);
    }
    __syncwarp();  // every lane is done with the previous unit's smem
    const unsigned kbase = kglob;
    if (lane == 0) {
      for (int k = 0; k < NST - 2 && k < nchunks; ++k) {
        const unsigned st = (kbase + k) % NST;
        mbar_expect_tx(bar0 + 8 * st, EROWS * CH * 4);
        tma_load_3d(ering + st * STAGE_BYTES, &map, C.s0 - 2, (C.q0 - 4 + CH * k) - A.in_col0, mapi, bar0 + 8 * st);
      }
    }
    // column masks of the first chunk
    if constexpr (S::MASKS) fill_colmask(A, colmask, ering + (kbase % NST) * STAGE_BYTES, C.q0 - 4, lane);
    for (int kc = 0; kc < nchunks; ++kc) {
      const unsigned st = (kbase + kc) % NST;
      __syncwarp();  // all lanes finished the previous chunk: its predecessor's stage may be refilled
      if (lane == 0 && kc + NST - 2 < nchunks) {
        const unsigned sn = (kbase + kc + NST - 2) % NST;
        mbar_expect_tx(bar0 + 8 * sn, EROWS * CH * 4);
        tma_load_3d(ering + sn * STAGE_BYTES, &map, C.s0 - 2, (C.q0 - 4 + CH * (kc + NST - 2)) - A.in_col0, mapi, bar0 + 8 * sn);
      }
      if constexpr (S::MASKS) fill_colmask(A, colmask, ering + ((kbase + kc + 1) % NST) * STAGE_BYTES, C.q0 - 4 + CH * (kc + 1), lane);  // next chunk's
      mbar_wait(bar0 + 8 * st, ((kbase + kc) / NST) & 1u);
      const int t0 = kc * CH;
      march_step<S, 0, KN>(C, L, t0 + 0, st);
      march_step<S, 1, KN>(C, L, t0 + 1, st);
      march_step<S, 2, KN>(C, L, t0 + 2, st);
      march_step<S, 3, KN>(C, L, t0 + 3, st);
      march_step<S, 4, KN>(C, L, t0 + 4, st);
    }
    kglob += nchunks;
    unit = __shfl_sync(FULL, next, 0);
  }
  finish_list(A.list, C.lstate, lane);
}

// ---------------------------------------------------------------------------------------------
// host side
// ---------------------------------------------------------------------------------------------
struct WindowClass {
  int w[3] = {-1, -1, -1};
  bool tips_on_circle = false;  // exactly {(+-2,0),(0,+-2)} undecidable
  bool ok = true;               // representable within reach 2
  int n = 0;                    // certain cells
  int k2 = 0;                   // sum of k^2 over certain cells
};

// The window offsets within 4 cells, classified against the circle of `radius` as the fused kernel needs them.  The reference
// decides membership on absolute cell centres (CircleIterator: dx * dx + dy * dy <= r2 with dx = X[a] - X[i]); dx is the lattice
// offset plus at most 2 cu, cu = ulp of the largest |coordinate| (te_footprint.cu's launch_footprint derives it), which moves
// dx^2 + dy^2 by up to 4 sqrt(2) r cu near the circle.  An offset closer to the circle than tol = max(1e-9 r2, 8 r cu) is "on" it:
// the tips the mask tables decide per row and column, anything else not representable.  Near the origin 1e-9 r2 is the larger
// term, so the YAML shapes and their outputs are unchanged; far out a radius in the band leaves the fused kernel.
WindowClass classify(double radius, double res, double cu) {
  WindowClass c;
  const double r2 = radius * radius;
  const double tol = std::max(1e-9 * r2, 8.0 * radius * cu) + 1e-300;
  for (int l = -4; l <= 4; ++l)
    for (int k = -4; k <= 4; ++k) {
      const double d2 = (double)(k * k + l * l) * res * res;
      const bool in = d2 < r2 - tol, on = std::fabs(d2 - r2) <= tol;
      if (!in && !on) continue;
      if (std::abs(k) > 2 || std::abs(l) > 2) { c.ok = false; continue; }
      if (on) {
        if ((k == 0 && std::abs(l) == 2) || (l == 0 && std::abs(k) == 2)) c.tips_on_circle = true;
        else c.ok = false;
        continue;
      }
      c.w[std::abs(l)] = std::max(c.w[std::abs(l)], std::abs(k));
      ++c.n;
      c.k2 += k * k;
    }
  return c;
}

// s = 1 - n_z below which the float32 rounding of n_z has to be certain (finish_normal2's k_nz_check; tier 2 widens its guard
// band to it).  One float32 ulp of n_z (2^-24 on [0.5, 1)) moves theta = acos(n_z) by ~2^-24 / sin(theta) and the slope layer
// 1 - theta/crit by that over crit, while the layer's tolerance 1e-5 |layer| + 1e-6 does not scale with crit; and away from a
// rounding boundary the fp32 n_z may be several ulps off (s carries the relative error of the moments), which near theta = crit,
// where the tolerance is 1e-6, the layer does not absorb either once crit < 1 rad.  So below 1 rad the band is every theta up to
// just past crit (2 % and 4 ulps of n_z past it, where the layer could otherwise step across its 0 branch): inside it a cell is
// either rounded exactly like the reference or flagged.  From 1 rad up it stays the 7.2e-5 (theta = 0.012 rad) calibrated at
// the YAML's crit = 1 rad (DESIGN.md §4.1: worst slope error 0.45 x tolerance on the 8192^2 map), so the YAML outputs keep every
// bit; there one ulp moves the layer by at most half its tolerance above the band.  s < 0.48: n_z > 0.5, the 2^-24 spacing the
// check assumes.  tests/test_kernel_constants_cpu.py restates this and checks it against every float32 n_z.
double nz_check_limit(double crit) {
  if (!(crit < 1.0)) return 7.2e-5;
  const double t = 1.02 * crit + std::ldexp(1.0, -22) / std::sin(crit);
  const double sh = std::sin(0.5 * t);
  return std::max(7.2e-5, 2.0 * sh * sh);  // 1 - cos(t) without cancellation
}

// roughness_critical of the YAML, where the roughness certification (rough_k = 0.06) was calibrated
constexpr double ROUGH_CRIT_YAML = 0.05;

// 1/step_crit as the kernel multiplies it (step layer = sat(1 - st * m)): for a step_critical_cells that is not a power of two,
// rounded up from float32(1/crit) until every st that may stand for a reference step >= crit gives st * m >= 1, i.e. exactly the
// reference's 0 branch (StepFilter.cpp:172-176): CNT * (1/ncrit) * stepMax carries up to three float32 roundings, so st may lie
// 4 ulps below crit.  A reference step below crit whose st passes that bound has a layer below 2.4e-7, inside the tolerance of
// 0.  With a power of two only the last product rounds; m stays float32(1/crit), so that the YAML outputs (0.12, 4 cells) keep
// every bit.  There the 0 branch is exact where st >= the smallest float >= crit, but CNT * stepMax / ncrit with CNT not a multiple
// of ncrit (3/4 stepMax at the YAML's 4 cells) can round to float32(crit) < crit where the reference's double step is >= crit: a
// layer of ~1e-7 instead of 0, at the YAML values too (a 1e-9 m wide window of stepMax at 0.12 m).  Open: deciding the branch
// exactly (the residual of the exact CNT * (1/ncrit) times stepMax) costs march-step instructions at the 168-register limit.
float step_layer_scale(double crit, int ncrit) {
  float m = (float)(1.0 / crit);
  if (ncrit > 0 && (ncrit & (ncrit - 1)) == 0) return m;
  float lo = (float)(crit * (1.0 - std::ldexp(4.0, -24)));
  if ((double)lo > crit * (1.0 - std::ldexp(4.0, -24))) lo = std::nextafterf(lo, 0.0f);
  while ((double)lo * (double)m < 1.0) m = std::nextafterf(m, INFINITY);  // the product of two floats is exact in double
  return m;
}

using ShapeA = Shape<2, 2, 1, 1, 1, -1, true, 1, 1, -1, true>;    // YAML radii at 0.02 m
using ShapeB = Shape<1, 1, -1, 1, 0, -1, false, 1, 0, -1, false>; // YAML radii at 0.03 m (fixture)

int match_shape(const WindowClass& n, const WindowClass& s1, const WindowClass& s2) {
  auto is = [](const WindowClass& c, int a, int b, int d, bool tip) {
    return c.ok && c.w[0] == a && c.w[1] == b && c.w[2] == d && c.tips_on_circle == tip;
  };
  if (is(n, 2, 2, 1, false) && is(s1, 1, 1, -1, true) && is(s2, 1, 1, -1, true)) return 0;
  if (is(n, 1, 1, -1, false) && is(s1, 1, 0, -1, false) && is(s2, 1, 0, -1, false)) return 1;
  return -1;
}

typedef CUresult (*PFN_encodeTiled)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*, const cuuint64_t*,
                                    const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave, CUtensorMapSwizzle,
                                    CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

PFN_encodeTiled get_encode() {
  static PFN_encodeTiled fn = nullptr;
  if (!fn) {
    void* p = nullptr;
    cudaDriverEntryPointQueryResult qres;
    if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &qres) == cudaSuccess &&
        qres == cudaDriverEntryPointSuccess)
      fn = reinterpret_cast<PFN_encodeTiled>(p);
  }
  return fn;
}

// Splits the output columns of every map into up to NLVL runs of segments, longest segments first.  A warp
// pops (segment, strip) units in that order, so the last units handed out are short and the warps finish
// within one short unit of each other.  Each unit pays 8 warm-up columns (cheap: the later stages are
// skipped), so the bulk of the map stays in longer segments (about eight long units per warp).
void plan_levels(FusedArgs& a, int out_ncols, int nmaps, int total_warps) {
  const double share = (double)a.nstrips * out_ncols * nmaps / (double)total_warps;  // strip-columns per warp
  const int len0 = std::min(128, std::max(16, (int)std::lround(share / 8.0 / 8.0) * 8));
  int len[NLVL] = {len0, std::max(16, len0 * 3 / 8 / 8 * 8), 16, 16};
  double frac[NLVL] = {0.80, 0.15, 0.05, 0.0};
  if (len0 == 16) { frac[0] = 1.0; frac[1] = frac[2] = 0.0; }
  if (share >= 400.0 && (long long)a.nstrips * nmaps <= total_warps / 4) {
    // Large single maps: ONE long unit per warp first — as many segments per strip as give every warp (at most) one unit, over
    // three quarters of the columns, so that a warp pays its 8 warm-up columns once for most of its work — then the tapering
    // tail (24- and 16-column segments) that evens out the warps' different speeds.  8192^2 on an H100 (132 SMs): 11 segments
    // of 552 columns per strip (1 507 units on 1 584 warps).
    const int nseg0 = (int)(total_warps / ((long long)a.nstrips * nmaps));
    const int l0 = (int)(0.75 * out_ncols / nseg0) / 8 * 8;
    if (l0 >= 128) {
      len[0] = l0; len[1] = 24; len[2] = 16;
      frac[0] = (double)l0 * nseg0 / out_ncols; frac[1] = 0.20; frac[2] = 1.0 - frac[0] - frac[1];
      if (frac[2] < 0.0) { frac[1] = 1.0 - frac[0]; frac[2] = 0.0; }
    }
  }
  if (share < 100.0) {
    // Small launches (a warp's share is a couple of units at most): the tapering queue has nothing to balance and the whole-unit
    // quantisation decides — the kernel lasts rounds(len) units of len full march steps + 8 warm-up steps (which skip the later
    // stages: ~0.45 of a step each) + ~4 steps of TMA pipeline fill, where rounds = ceil(units / warps).  Take the single segment
    // length that minimises that (2048^2: 44 columns, one round, instead of 16 columns: three rounds; an 8192 x 1024 slab of the
    // 8-GPU tiling: 88 columns, one round, instead of five rounds of 16).
    int best_len = 16;
    double best_cost = 1e300;
    for (int l = 8; l <= 160; l += 4) {
      const long long units = (long long)a.nstrips * ((out_ncols + l - 1) / l) * nmaps;
      const long long rounds = (units + total_warps - 1) / total_warps;
      const double cost = (double)rounds * (l + 8 * 0.45 + 4);
      if (cost < best_cost - 1e-9) { best_cost = cost; best_len = l; }
    }
    len[0] = best_len;
    frac[0] = 1.0; frac[1] = frac[2] = 0.0;
  }
#ifdef TE_CALIBRATION
  const char* e = std::getenv("TE_FUSED_SEGS");  // calibration builds only (tools/dev_segs.sh): "len:frac,len:frac,..."
#else
  const char* e = nullptr;
#endif
  if (e && *e) {
    for (int i = 0; i < NLVL; ++i) { len[i] = 16; frac[i] = 0.0; }
    int i = 0, l = 0, n = 0;
    double f = 0.0;
    while (i < NLVL && std::sscanf(e, "%d:%lf%n", &l, &f, &n) >= 2) {
      len[i] = std::max(8, l);
      frac[i] = f;
      ++i;
      e += n;
      if (*e == ',') ++e;
    }
  }
  int col = 0, unit = 0;
  double cum = 0.0;
  for (int i = 0; i < NLVL; ++i) {
    cum += frac[i];
    int end = (i == NLVL - 1 || cum >= 1.0) ? out_ncols : (int)std::lround(cum * out_ncols);
    end = std::min(std::max(end, col), out_ncols);
    bool later = false;
    for (int j = i + 1; j < NLVL; ++j) later = later || frac[j] > 0.0;
    if (!later) end = out_ncols;
    const int ncol = end - col;
    a.lvl_unit0[i] = unit;
    a.lvl_col0[i] = col;
    a.lvl_len[i] = len[i];
    a.lvl_nseg[i] = (ncol + len[i] - 1) / len[i];
    unit += a.nstrips * a.lvl_nseg[i] * nmaps;
    col = end;
  }
  a.lvl_unit0[NLVL] = unit;
  a.lvl_col0[NLVL] = out_ncols;
}

template <class S, bool KN>
int launch_shape(FusedState& st, const CUtensorMap& map, const FusedArgs& a, int sms, cudaStream_t s) {
  const int smem = WARPS_PER_CTA * WARP_SMEM_BYTES;
  bool& attr_set = st.smem_attr[st.shape_id * 2 + (KN ? 1 : 0)];
  if (!attr_set) {
    if (cudaFuncSetAttribute(k_chain_fused<S, KN>, cudaFuncAttributeMaxDynamicSharedMemorySize, smem) != cudaSuccess) {
      st.why = "cudaFuncSetAttribute(max dynamic shared memory) failed";
      return 1;
    }
    attr_set = true;
  }
  const int nunits = a.lvl_unit0[NLVL];
  int grid = std::min(sms, (nunits + WARPS_PER_CTA - 1) / WARPS_PER_CTA);
  if (grid < 1) grid = 1;
  k_chain_fused<S, KN><<<grid, WARPS_PER_CTA * 32, smem, s>>>(map, a);
  return 0;
}

}  // namespace

size_t fused_list_capacity(size_t cells, int sms) {
  // every flagged cell once, plus the padding of chunk tails (an append of up to 64 entries that does not fit opens a new
  // chunk: at most 63 of LIST_CHUNK entries lost per chunk) and one open chunk per warp
  return cells + cells / 7 + (size_t)sms * WARPS_PER_CTA * LIST_CHUNK + LIST_CHUNK;
}

void fused_plan(int rows, int out_ncols, int nmaps, int sms, int out[19]) {
  FusedArgs a{};
  a.nstrips = (rows + OROWS - 1) / OROWS;
  plan_levels(a, out_ncols, nmaps, sms * WARPS_PER_CTA);
  out[0] = a.nstrips;
  out[1] = NLVL;
  for (int i = 0; i < NLVL; ++i) {
    out[2 + 4 * i] = a.lvl_unit0[i];
    out[3 + 4 * i] = a.lvl_col0[i];
    out[4 + 4 * i] = a.lvl_len[i];
    out[5 + 4 * i] = a.lvl_nseg[i];
  }
  out[2 + 4 * NLVL] = a.lvl_unit0[NLVL];
}

void FusedState::release() {
  rowmask.release();
  colmask.release();
  valid = false;
}

void fused_mask_bits(const te_chain_params* p, const double* P, int n, unsigned char* out) {
  const double r1sq = p->step_first_radius * p->step_first_radius, r2sq = p->step_second_radius * p->step_second_radius;
  for (int i = 0; i < n; ++i) {
    unsigned b = 0;
    if (i - 2 >= 0) {
      const double d = P[i - 2] - P[i];
      if (d * d + 0.0 <= r1sq) b |= 1u;
      if (d * d + 0.0 <= r2sq) b |= 4u;
    }
    if (i + 2 < n) {
      const double d = P[i + 2] - P[i];
      if (d * d + 0.0 <= r1sq) b |= 2u;
      if (d * d + 0.0 <= r2sq) b |= 8u;
    }
    out[i] = (unsigned char)b;
  }
}

bool fused_eligible(FusedState& st, const std::vector<double>& X, const std::vector<double>& Y, const te_geometry* g,
                    const te_chain_params* p, double coord_max, cudaStream_t stream) {
  const double cu = coord_ulp(coord_max + 4.0 * g->resolution);
  if (st.valid && std::memcmp(&st.key_geo, g, sizeof(*g)) == 0 && std::memcmp(&st.key_par, p, sizeof(*p)) == 0 && st.key_cu == cu)
    return st.shape_id >= 0;
  st.valid = false;
  st.shape_id = -1;
  st.key_geo = *g;
  st.key_par = *p;
  st.key_cu = cu;
  auto no = [&](const char* why) {
    st.why = why;
    st.valid = true;
    return false;
  };
  if (p->normals_algorithm != TE_NORMALS_FIXTURE) return no("normals algorithm is not the fixture-pinned one");
  if (p->normals_positive_axis != 2) return no("normal_vector_positive_axis is not z");
  if (g->rows % 4 != 0) return no("row count is not a multiple of 4 (TMA needs 16-byte column pitch)");
  if (!(p->slope_critical > 0.0) || !(p->step_critical > 0.0) || !(p->roughness_critical > 0.0)) return no("a critical value is zero");
  const double res = g->resolution;
  const WindowClass wn = classify(p->normals_radius, res, cu), wr = classify(p->roughness_radius, res, cu);
  const WindowClass w1 = classify(p->step_first_radius, res, cu), w2 = classify(p->step_second_radius, res, cu);
  if (!wn.ok || wn.tips_on_circle) return no("normals window not representable (reach > 2 cells or on-circle offsets)");
  if (!wr.ok || wr.tips_on_circle || std::memcmp(wn.w, wr.w, sizeof(wn.w)) != 0) return no("roughness window differs from the normals window");
  const int id = match_shape(wn, w1, w2);
  if (id < 0) return no("no fused instantiation for these window shapes");
  // on-circle tip membership, decided exactly like CircleIterator does (double, absolute positions)
  std::vector<unsigned char>&rm = st.h_rowmask, &cm = st.h_colmask;  // owned by the state: the uploads below are asynchronous
  rm.assign(g->rows, 0);
  cm.assign(g->cols, 0);
  fused_mask_bits(p, X.data(), g->rows, rm.data());
  fused_mask_bits(p, Y.data(), g->cols, cm.data());
  // Kernels of an earlier asynchronous call may still read the tables: the overwrite is ordered after them on the context
  // stream (a reallocation waits for the stream first).
  auto upload = [&](DevBuf& d, const std::vector<unsigned char>& h) {
    if (d.p && d.cap < h.size() && cudaStreamSynchronize(stream) != cudaSuccess) return false;
    return d.reserve(h.size()) == cudaSuccess &&
           cudaMemcpyAsync(d.p, h.data(), h.size(), cudaMemcpyHostToDevice, stream) == cudaSuccess;
  };
  if (!upload(st.rowmask, rm) || !upload(st.colmask, cm)) return no("mask table upload failed");
  if (cudaStreamSynchronize(stream) != cudaSuccess) return no("mask table upload failed");  // the host copies are reused
  st.shape_id = id;
  st.valid = true;
  st.why.clear();
  return true;
}

void make_fixup_args(const FusedState& st, const SlabView& v, const ChainDev& p, const MapMasks* mm, FixupArgs* out) {
  const WindowClass wn = classify(p.rn, v.res, st.key_cu), w1 = classify(p.r1, v.res, st.key_cu), w2 = classify(p.r2, v.res, st.key_cu);
  FixupArgs a{};
  a.rows = v.rows; a.cols_total = v.cols_total; a.in_col0 = v.in_col0; a.in_ncols = v.in_ncols; a.out_col0 = v.out_col0;
  a.map_cells = (unsigned)((size_t)v.rows * v.out_ncols);
  a.in_map_stride = (size_t)v.rows * v.in_ncols;
  for (int k = 0; k < 3; ++k) { a.wn[k] = wn.w[k]; a.w1[k] = w1.w[k]; a.w2[k] = w2.w[k]; }
  a.tip1 = w1.tips_on_circle; a.tip2 = w2.tips_on_circle;
  a.ncrit = p.ncrit;
  a.n_full = (double)wn.n;
  a.n_full_i = wn.n;
  a.res = v.res; a.slope_crit = p.slope_crit; a.step_crit = p.step_crit; a.rough_crit = p.rough_crit;
  a.inv_slope_crit = 1.0 / p.slope_crit; a.inv_rough_crit = 1.0 / p.rough_crit;
  // Tier 2 rounds n_z to float32 itself unless n_z lies so close to a rounding boundary that the REFERENCE's own rounding errors
  // could put its double result on the other side.  The reference forms the window offsets from absolute coordinates
  // (X[a] - mean): relative error eps_off <= 4 * 2^-53 * |X|max / res; the small-angle term s = 1 - n_z <= 2e-4 inherits ~4 eps_off,
  // i.e. 2e-4 * 16 * 2^-53 * (|X|max / res) / 2^-24 = 6e-12 * |X|max / res float32 ulps (6e-9 for the 8192^2 map at 0.02 m, with
  // tier 2's own error on centred coordinates an order below).  The band is 100 times that, at least 1e-6 ulp.  It applies to
  // n_z > 0.9998, or down to the band tier 1 certifies when that is wider (small slope_critical, nz_check_limit); past s = 2e-4
  // tier 2 scales it by the cell's own s / 2e-4, as the error grows in proportion to s.
  const double s_check = nz_check_limit(p.slope_crit);
  a.nz_check = s_check > 2e-4 ? 1.0 - s_check : 0.9998;
  a.nz_guard = std::max(1e-6, 100.0 * 6e-12 * v.coord_max / v.res);
  a.fuse_w = p.fuse_w;
  a.rowmask = mm ? mm->rowmask : (const unsigned char*)st.rowmask.p;
  a.colmask = mm ? mm->colmask : (const unsigned char*)st.colmask.p;
  a.rowmask_stride = mm ? mm->row_stride : 0u;
  a.colmask_stride = mm ? mm->col_stride : 0u;
  *out = a;
}

const char* fused_launch_obstacle(const SlabView& v, int nmaps, const float* elev, const ChainOut& o) {
  if ((reinterpret_cast<uintptr_t>(elev) & 15u) != 0) return "elevation pointer is not 16-byte aligned (TMA)";
  if ((size_t)v.rows * v.out_ncols * (size_t)nmaps >= ((size_t)1 << 30)) return "launch covers 2^30 or more cells";
  const float* outs[7] = {o.slope, o.step, o.rough, o.trav, o.nx, o.ny, o.nz};
  for (const float* q : outs)
    if (q && (reinterpret_cast<uintptr_t>(q) & 7u) != 0) return "an output layer is not 8-byte aligned";
  const int have_n = (o.nx != nullptr) + (o.ny != nullptr) + (o.nz != nullptr);
  if (have_n != 0 && have_n != 3) return "surface normal outputs must be given all three or none";
  return nullptr;
}

int launch_chain_fused(FusedState& st, const SlabView& v, const ChainDev& p, int nmaps, const float* elev, const ChainOut& o,
                       unsigned* list, unsigned* count, unsigned cap, int sms, cudaStream_t s, const MapMasks* mm) {
  if (st.shape_id < 0) { st.why = "fused stencil not eligible"; return 1; }
  if (const char* why = fused_launch_obstacle(v, nmaps, elev, o)) { st.why = why; return 1; }
  PFN_encodeTiled enc = get_encode();
  if (!enc) { st.why = "cuTensorMapEncodeTiled entry point unavailable"; return 1; }
  CUtensorMap map;
  const cuuint64_t dims[3] = {(cuuint64_t)v.rows, (cuuint64_t)v.in_ncols, (cuuint64_t)nmaps};
  const cuuint64_t strides[2] = {(cuuint64_t)v.rows * sizeof(float), (cuuint64_t)v.rows * v.in_ncols * sizeof(float)};
  const cuuint32_t box[3] = {(cuuint32_t)EROWS, (cuuint32_t)CH, 1};
  const cuuint32_t estr[3] = {1, 1, 1};
  const CUresult cr = enc(&map, CU_TENSOR_MAP_DATA_TYPE_FLOAT32, 3, const_cast<float*>(elev), dims, strides, box, estr,
                          CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_NONE, CU_TENSOR_MAP_L2_PROMOTION_L2_128B,
                          CU_TENSOR_MAP_FLOAT_OOB_FILL_NAN_REQUEST_ZERO_FMA);
  if (cr != CUDA_SUCCESS) { st.why = "cuTensorMapEncodeTiled failed (" + std::to_string((int)cr) + ")"; return 1; }

  const double res = v.res;
  const WindowClass wn = classify(p.rn, res, st.key_cu);
  FusedArgs a{};
  a.rows = v.rows; a.cols_total = v.cols_total;
  a.in_col0 = v.in_col0; a.in_ncols = v.in_ncols; a.out_col0 = v.out_col0; a.out_ncols = v.out_ncols;
  a.nstrips = (v.rows + OROWS - 1) / OROWS;
  a.nmaps = nmaps;
  a.map_cells = (unsigned)((size_t)v.rows * v.out_ncols);
  plan_levels(a, v.out_ncols, nmaps, sms * WARPS_PER_CTA);
  a.queue = count + 96;  // its own 128-byte line of the 512-byte counter block (words 8..49 hold tier-2 diagnostics)
  const double N = wn.n, K2 = wn.k2;
  a.a_cov = (float)(res * res * K2 / N);
  a.half_a = 0.5f * a.a_cov;
  // certification constants (DESIGN.md "certification")
  double rough_k = 0.06, cond_k = 0.25;
#ifdef TE_CALIBRATION  // calibration builds only (tools/dev_calib.py): the shipped library does not take its certification from the environment
  if (const char* e = std::getenv("TE_FUSED_ROUGH_K")) rough_k = std::atof(e);
  if (const char* e = std::getenv("TE_FUSED_COND_K")) cond_k = std::atof(e);
#endif
  a.cond_k = (float)cond_k;
  // Below the YAML's roughness_critical (0.05 m) rough_k is 1.5.  A cell at r ~ crit has a layer tolerance of 1e-6 absolute, and the
  // fp32 error of lambda0 moves the layer by about that error over 2 crit^2: in windows of nearly isotropic noise (cmag ~ lambda0)
  // fp32 lambda0 is off by up to ~2.5e-6 relative, and with 0.06 such cells at 0.02 ... 0.005 m on rough terrain left the
  // tolerance (1-5 per 1024^2 map; the flag lambda0 < rough_thr cmag^2 needs rough_k > crit r / cmag ~ 1.03 for the worst of
  // them).  With 1.5 every cell from r = 0.82 crit up is flagged (cmag >= lambda0), and below it the tolerance is 2.8e-6 or more.
  // At 0.05 m and above rough_k is the calibrated 0.06, so the YAML outputs keep every bit.
  if (p.rough_crit < ROUGH_CRIT_YAML) rough_k = std::max(rough_k, 1.5);
  a.rough_thr =(float)((rough_k / p.rough_crit) * (rough_k / p.rough_crit) * (N - 1.0) / N);
  a.kp = (float)(-res / N);
  a.invN = (float)(1.0 / N);
  a.n_over_nm1 = (float)(N / (N - 1.0));
  a.slope_crit = (float)p.slope_crit; a.inv_slope_crit = (float)(1.0 / p.slope_crit); a.minv_slope_crit = (float)(-1.0 / p.slope_crit);
  a.minv_step_crit = -step_layer_scale(p.step_crit, p.ncrit); a.minv_rough_crit = (float)(-1.0 / p.rough_crit);
  a.step_crit = (float)p.step_crit; a.inv_step_crit = (float)(1.0 / p.step_crit);
  a.step_cmp = (float)p.step_crit;
  if ((double)a.step_cmp > p.step_crit) a.step_cmp = std::nextafterf(a.step_cmp, -INFINITY);
  a.inv_ncrit = (float)(1.0 / (double)p.ncrit);
  a.rough_crit = (float)p.rough_crit; a.inv_rough_crit = (float)(1.0 / p.rough_crit);
  a.fuse_w = p.fuse_w;
  auto B2 = [](double v) { return (float)v; };  // a kernel constant: the double value rounded to float32 once, here
  a.k_invN = B2(1.0 / N); a.k_kp = B2(-res / N); a.k_half_a = B2(0.5 * (double)a.a_cov);
  a.k_nnm1 = B2(N / (N - 1.0)); a.k_rough_thr = B2((double)a.rough_thr);
  a.k_inv_ncrit = B2((double)a.inv_ncrit); a.k_fuse_w = B2((double)a.fuse_w);
  a.k_m0 = B2(wn.w[2] >= 0 ? 2 * wn.w[2] + 1 : 0); a.k_m1 = B2(wn.w[1] >= 0 ? 2 * wn.w[1] + 1 : 0);
  a.k_1em5 = B2(1e-5); a.k_1em10a = B2(1e-10 * (double)a.a_cov); a.k_mcond = B2(-cond_k);
  a.k_2p24 = B2(16777216.0); a.k_7p1em6 = B2(7.1e-6);
  a.k_2em6 = B2(2.5e-6);  // relative error budget of s = 1 - n_z besides the moments' (2e-6, plus two more MUFU results in s)
  // Absolute term of the rounding-boundary bound (qv * eps + k_bmargin, in float32 spacings of n_z).  It was meant to be 1e-3,
  // but that assignment was lost by accident (it ended up inside a trailing comment) and the kernel has run with 0 since.  It
  // stays 0 here so that the outputs stay bit-identical; restoring the 1e-3 floor is an open certification question (it would
  // send more cells near a rounding boundary to the fp64 fix-up and can change their float32 rounding).
  a.k_bmargin = B2(0.0);
  a.k_nz_check = B2(nz_check_limit(p.slope_crit));
  a.k_one = B2(1.0); a.k_two = B2(2.0); a.k_half = B2(0.5);
  a.k_p0 = B2(1.570796251296997); a.k_p1 = B2(-0.21459604799747467); a.k_p2 = B2(0.08894557505846024);
  a.k_p3 = B2(-0.05000271648168564); a.k_p4 = B2(0.03044925443828106); a.k_p5 = B2(-0.016484638676047325);
  a.k_p6 = B2(0.006254698149859905); a.k_p7 = B2(-0.0011488182935863733);
  a.rowmask = mm ? mm->rowmask : (const unsigned char*)st.rowmask.p;
  a.colmask = mm ? mm->colmask : (const unsigned char*)st.colmask.p;
  a.rowmask_stride = mm ? mm->row_stride : 0u;
  a.colmask_stride = mm ? mm->col_stride : 0u;
  a.slope = o.slope; a.step = o.step; a.rough = o.rough; a.trav = o.trav;
  a.nx = (o.nx && o.ny && o.nz) ? o.nx : nullptr; a.ny = o.ny; a.nz = o.nz;
  a.list = list; a.count = count; a.cap = cap;
  switch (st.shape_id) {
    case 0: return a.nx ? launch_shape<ShapeA, true>(st, map, a, sms, s) : launch_shape<ShapeA, false>(st, map, a, sms, s);
    case 1: return a.nx ? launch_shape<ShapeB, true>(st, map, a, sms, s) : launch_shape<ShapeB, false>(st, map, a, sms, s);
  }
  st.why = "unknown shape id";
  return 1;
}

}  // namespace te
