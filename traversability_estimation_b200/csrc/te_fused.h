// te_fused.h — host interface of the fused chain stencil (te_fused.cu).
#pragma once
#include <cuda_runtime.h>
#include <string>
#include <vector>
#include "../../include/te_b200.h"
#include "te_kernels.h"

namespace te {

struct FusedState {
  std::string why;        // why the last eligibility check / launch failed
  bool valid = false;     // tables below match (geometry, params) of `key_*`
  te_geometry key_geo{};
  te_chain_params key_par{};
  int shape_id = -1;
  std::vector<unsigned char> h_rowmask, h_colmask;  // host copies of the tables below
  DevBuf rowmask, colmask;  // per-row / per-column on-circle membership bits
  bool smem_attr[4] = {false, false, false, false};  // dynamic shared memory limit raised for instantiation [shape*2 + normals]
                                                     // (a per-device function attribute; a context lives on one device)
  void invalidate() { valid = false; }
  void release();
};

// True when the fused stencil has an instantiation for these window shapes (fills the tables).
bool fused_eligible(FusedState& st, const std::vector<double>& X, const std::vector<double>& Y, const te_geometry* g,
                    const te_chain_params* p, cudaStream_t stream);
// Why this particular launch cannot use the fused stencil although the window shapes are eligible (pointer alignment, size,
// partial normal outputs), or nullptr.  TE_KERNEL_AUTO runs the generic kernel instead.
const char* fused_launch_obstacle(const SlabView& v, int nmaps, const float* elev, const ChainOut& o);

// Arguments of the tier-2 fix-up kernel (te_fixup.cu): integer window description + parameters.
struct FixupArgs {
  int rows, cols_total, in_col0, in_ncols, out_col0;
  unsigned map_cells;       // output cells per map (batched launches index cells across maps)
  size_t in_map_stride;     // elevation elements per map
  int wn[3], w1[3], w2[3];  // half-width per |column offset| (-1: column not in the window)
  int tip1, tip2;           // (+-2,0),(0,+-2) decided by the mask tables
  int ncrit;
  double n_full;            // cells of the full normals window
  int n_full_i;
  double res, slope_crit, step_crit, rough_crit;
  double inv_slope_crit, inv_rough_crit;
  double nz_guard;          // half-width, in float32 ulps, of the band around a rounding boundary of n_z that tier 2 leaves to tier 3
  float fuse_w;
  const unsigned char* rowmask;
  const unsigned char* colmask;
};

// Fills the tier-2 arguments for the shape the fused stencil was found eligible for.
void make_fixup_args(const FusedState& st, const SlabView& v, const ChainDev& p, FixupArgs* out);
// pdl: launch as a programmatic dependent of the preceding kernel of the stream (the kernel waits on griddepcontrol.wait)
void launch_fixup_t2(const FixupArgs& a, const float* elev, const ChainOut& o, const unsigned* list, const unsigned* count,
                     unsigned cap, unsigned* list3, unsigned* count3, unsigned cap3, int sms, cudaStream_t s, bool pdl);

// Work lists.  The fused kernel appends in warp-private chunks: entries equal to LIST_INVALID are padding and are skipped by the
// consumers; count[0] = list entries reserved (chunks), count[1] = cells flagged, count[2] = overflow flag (never set when the
// list holds fused_list_capacity() entries), count[4] = tier-3 entries, count[5] = tier-3 overflow flag.
constexpr unsigned LIST_INVALID = 0xffffffffu;
size_t fused_list_capacity(size_t cells, int sms);

// Returns 0 on success.  Cells whose result could not be certified in fp32 are appended to `list`.
// Work decomposition of the fused launch (see te_fused_plan in include/te_b200.h); host arithmetic only.
void fused_plan(int rows, int out_ncols, int nmaps, int sms, int out[19]);

int launch_chain_fused(FusedState& st, const SlabView& v, const ChainDev& p, int nmaps, const float* elev, const ChainOut& o,
                       unsigned* list, unsigned* count, unsigned cap, int sms, cudaStream_t s);

}  // namespace te
