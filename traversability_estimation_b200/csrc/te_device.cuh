// te_device.cuh — device-side descriptors shared by all kernels of libte_b200.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

namespace te {

// Device view of one column slab of a column-major float32 layer set.
// Input layers hold global columns [in_col0, in_col0 + in_ncols); output layers hold
// [out_col0, out_col0 + out_ncols).  X/Y are the cell-centre coordinates of the GLOBAL map in
// double, computed on the host with grid_map's getPositionFromIndex operand order, so window
// membership is decided on exactly the numbers the reference's CircleIterator sees.
struct SlabView {
  int rows;
  int cols_total;
  int in_col0, in_ncols;
  int out_col0, out_ncols;
  const double* X;  // [rows]
  const double* Y;  // [cols_total]
  double res;
  double coord_max;  // largest |cell-centre coordinate| of the global map (host-side use: error bounds of the reference's
                     // absolute-coordinate arithmetic); of every map of a batch at per-map positions
  // A batch whose maps sit at their own positions (a te_map given positions): map m's tables start m * xs entries into X and
  // m * ys into Y, and its position is pos[2m], pos[2m + 1].  xs = ys = 0 and pos = nullptr: every map at the one position.
  int xs, ys;
  const double* pos;
};

// Chain parameters in the form the kernels want them.
struct ChainDev {
  double rn, rn2;  // normals radius, squared
  int Rn;          // max |index offset| that can be inside the normals circle
  int alg, axis;
  double slope_crit;
  double step_crit, r1, r1sq, r2, r2sq;
  int R1, R2, ncrit;
  double rough_crit, rr, rr2;
  int Rr;
  float fuse_w;
};

__device__ __forceinline__ bool finitef(float v) { return fabsf(v) < __int_as_float(0x7f800000); }
__device__ __forceinline__ float nanf_() { return __int_as_float(0x7fc00000); }

}  // namespace te
