// te_kernels.h — host-callable launchers of the device code (internal to libte_b200).
#pragma once
#include <cuda_runtime.h>
#include "te_device.cuh"

namespace te {

// A grow-only device allocation: reserve() reallocates (without keeping the contents) only when `bytes` exceeds the capacity.
struct DevBuf {
  void* p = nullptr;
  size_t cap = 0;
  cudaError_t reserve(size_t bytes) {
    if (bytes <= cap) return cudaSuccess;
    release();
    cudaError_t e = cudaMalloc(&p, bytes);
    if (e == cudaSuccess) cap = bytes;
    else p = nullptr;
    return e;
  }
  void release() {
    if (p) cudaFree(p);
    p = nullptr;
    cap = 0;
  }
};

struct ChainOut {
  float* slope;
  float* step;
  float* rough;
  float* trav;
  float* nx;  // may be null
  float* ny;
  float* nz;
};

// te_generic.cu — literal double-precision kernels (any radius / resolution).
void launch_chain_generic(const SlabView& v, const ChainDev& p, const float* elev, const ChainOut& o, int sms, cudaStream_t s);
// zero_next: 128 counter words the kernel zeroes for the next chain call (may be null); pdl: programmatic dependent launch
void launch_fixup(const SlabView& v, const ChainDev& p, const float* elev, const ChainOut& o, const unsigned int* list,
                  const unsigned int* count, unsigned int cap, unsigned int* zero_next, int sms, cudaStream_t s, bool pdl);
void launch_normals(const SlabView& v, const ChainDev& p, const float* elev, float* nx, float* ny, float* nz, int sms, cudaStream_t s);
void launch_slope(long long total, double crit, const float* nz, float* out, int sms, cudaStream_t s);
void launch_step(const SlabView& v, const ChainDev& p, const float* elev, float* out, int sms, cudaStream_t s);
void launch_roughness(const SlabView& v, const ChainDev& p, const float* elev, const float* nx, const float* ny, const float* nz,
                      float* out, int sms, cudaStream_t s);

// te_submap.cu — the read side of a te_map.  A window of te_map_get_submaps that has cells: its block of the map and where its
// layers go.  Columns are numbered flat over (window, layer, column), window by window.
struct SubmapWindow {
  long long col0;  // the window's first column in that numbering
  long long src;   // cell offset of its top-left cell in a source layer: top_col * map rows + top_row
  long long dst;   // float offset of its first layer in `out`
  int rows, cols;
};
struct SubmapGather {
  const float* const* layers;  // device table of the source layers (column-major, default order), in output order
  const SubmapWindow* win;     // device, in column order
  int nwin, map_rows;
  long long ncolumns;          // windows x layers x columns
  float* out;
};
// One k_map_gather_submaps launch for every column of every window (none when there is no column).
void launch_gather_submaps(const SubmapGather& a, int sms, cudaStream_t s);
// out[c] = upper[c] - lower[c] for n cells (device pointers), IEEE float32: publishTraversabilityMap's uncertainty_range.  One
// k_uncertainty_range launch (none for n = 0).
void launch_uncertainty_range(const float* upper, const float* lower, float* out, size_t n, int sms, cudaStream_t s);
// te_map_get_occupancy: GridMapRosConverter::toOccupancyGrid of nlayers layers of nmaps maps (device pointers).  Block q = l * nmaps
// + k of `out` (cells bytes at out + q * cells) is layer l of map slot[k] (slot null: map k) in grid order: out[q * cells + p] is
// the cell of source index cells - 1 - p of that map's column-major, default-order block, with layer l's data_min / data_max.
constexpr int kOccupancyMaxLayers = 17;  // te_layer bits 0 .. 17 but the unassigned 7
struct MapOccupancy {
  const float* layer[kOccupancyMaxLayers];  // resident layers in output order, every map of the te_map back to back
  const float* lower;                       // lower_bound: layer[range_l] (upper_bound) - lower is uncertainty_range
  float data_min[kOccupancyMaxLayers], data_max[kOccupancyMaxLayers];
  int nlayers, range_l;                     // range_l: output index of uncertainty_range, or -1
  int nmaps;                                // maps of the call
  const int* slot;                          // device, nmaps map indices, or null
  long long cells;                          // rows * cols
  unsigned char* out;
};
// One k_map_occupancy launch for every layer and map (none when there is no cell).
void launch_map_occupancy(const MapOccupancy& a, int sms, cudaStream_t s);
// te_map_get_point_cloud: GridMapRosConverter::toPointCloud of nmaps maps (device pointers), an ordered stream compaction.  Map k of
// the call is cut into `tiles` tiles of kCloudTile consecutive cells of its buffer order (linear index b: buffer cell (b % rows,
// b / rows), which is default-order cell ((b % rows - sr) mod rows, (b / rows - sc) mod cols)).  A cell is a point where the point
// layer and every basic layer are finite; its record is nfields entries of 4 bytes, entry point_e (if any) as x, y, z.  A layer
// source whose bit is set in its *_range mask is uncertainty_range: that pointer is upper_bound, and `lower` is subtracted.
constexpr int kCloudMaxFields = 32;
constexpr int kCloudMaxBasic = 17;  // te_layer bits 0 .. 17 but the unassigned 7
constexpr int kCloudTile = 1024;    // cells per tile: 4 chunks of one 256-thread block
struct CloudMap {                   // one map of a call: its slot in the te_map, start index and position
  int slot, sr, sc, pad;
  double px, py;
};
struct MapCloud {
  const float* field[kCloudMaxFields];  // entry e's resident layer, every map back to back; null: the NaN 0x7fc00000
  unsigned field_range;
  int nfields, point_e;                 // point_e: the entry that expands to x, y, z, or -1
  const float* point;
  const float* basic[kCloudMaxBasic];
  unsigned basic_range;                 // bit b: basic[b]; bit 31: point
  int nbasic;
  const float* lower;
  int rows, cols, nmaps, tiles;         // tiles per map
  long long cells;                      // rows * cols
  const CloudMap* maps;                 // device, nmaps; null: map k in slot k at (sr, sc) and (px, py)
  int sr, sc;
  double px, py, lenx, leny, res;
  unsigned long long* count;            // nmaps * tiles + 1 entries (the last 0)
  unsigned long long* first;            // their exclusive prefix sum: a tile's first point; first[k * tiles] is map k's offset
  long long* offsets;                   // device memory: gets first[k * tiles] for k = 0 .. nmaps; null in host memory
  int point_step;                       // bytes: 4 * (nfields + 2 when point_e >= 0)
  long long capacity;                   // points at or past it are not written
  unsigned char* out;
};
// Bytes of the device scratch the scan of launch_map_cloud_count needs for n tile counts.
size_t map_cloud_scan_bytes(long long n);
// k_map_cloud_count, then the exclusive sum of the counts into a.first (cub, in tmp of tmp_bytes): two launches.
cudaError_t launch_map_cloud_count(const MapCloud& a, void* tmp, size_t tmp_bytes, int sms, cudaStream_t s);
// k_map_cloud_scatter: every point below a.capacity to its record at a.out + point index * point_step, and a.offsets.  One launch.
void launch_map_cloud_scatter(const MapCloud& a, int sms, cudaStream_t s);
struct GridGeo;
// valid[q] = getIndex(xy[2q], xy[2q+1]) succeeds and traversability is finite there (device pointers; none launched for n = 0).
// A batch of nmaps maps of geometry g back to back in `trav`: position q is on map pos_map[q] (null: map 0), and a map outside
// 0 .. nmaps-1 gives 0.  map_pos (device, 2 * nmaps doubles, or null: every map at g's position): map m sits at map_pos[2m],
// map_pos[2m + 1] (needs pos_map).
void launch_valid_at(const GridGeo& g, const float* trav, int n, const double* xy, const int* pos_map, int nmaps, const double* map_pos,
                     unsigned char* valid, cudaStream_t s);
// te_map_at_poses: layers of a batch at npoints robot-frame points around each of nposes poses (device pointers).  Point t of
// pose k lands at pose_point_d (te_pose.cuh) on map pose_map[k] (null: map 0) and is read at the cell grid_get_index finds there,
// on that map's position (map_pos as in launch_valid_at); a map outside 0 .. nmaps-1, a non-finite position or one outside the
// map gives NaN (0x7fc00000) and valid 0.  Layer l of sample s = k * npoints + t goes to out[l * nposes * npoints + s].
constexpr int kAtPosesMaxLayers = 17;  // te_layer bits 0 .. 17 but the unassigned 7
struct MapAtPoses {
  const float* layer[kAtPosesMaxLayers];  // resident layers in output order, each nmaps maps back to back, column-major
  const float* lower;                     // lower_bound: layer[range_l] (upper_bound) - lower is uncertainty_range
  int nlayers, range_l;                   // range_l: output index of uncertainty_range, or -1
  int rows, cols, nmaps, nposes, npoints; // nposes * npoints < 2^31
  double res, lenx, leny, posx, posy;     // geometry, at the position of every map when map_pos is null
  const double* map_pos;
  const int* pose_map;
  const double* poses;                    // 7 per pose: x y z qx qy qz qw
  const float* points;                    // 3 per point: x y z
  float* out;
  unsigned char* valid;                   // may be null
};
// One k_map_at_poses launch (none for nposes = 0).
void launch_map_at_poses(const MapAtPoses& a, int sms, cudaStream_t s);

// nmaps windows of rows x cols cells, each read out of a source of src_rows x src_cols cells through that source's circular-buffer
// start index (device pointers).  Window k is win[k] = (top_row, top_col, start_row, start_col): it starts at source cell (top_row,
// top_col), which may lie outside the source, and layer l of it goes column-major to dst[k * nlayers + l].  Source cell (I, J) of
// window k's layer l is stored at src[k * nlayers + l][col_of(Jb) * src_rows + Ib], (Ib, Jb) = (I + start_row, J + start_col)
// modulo the source size and col_of the identity, or the table col_of when only some source columns were staged; a cell outside
// the source is NaN 0x7fc00000.  One kernel serves three moves:
//   - te_map_chain_submap / te_map_chain_windows: every window on the one larger map, at its top-left, with that map's start index;
//   - unwrapping a map that came in its own buffer order: top-left (0, 0), the map's block as source, its start index (sr, sc);
//   - re-wrapping a resident default-order map to that order: top-left (0, 0), start index ((rows - sr) % rows, (cols - sc) % cols).
// Cells move as 4-byte words, unchanged (NaN payloads and int32 layers included).
constexpr int kCutMaxLayers = 8;  // a cut's source layers: elevation and the seven carried layers
struct WindowCut {
  const int4* win;          // device, nmaps
  const float* const* src;  // device, nmaps * nlayers
  float* const* dst;        // device, nmaps * nlayers
  const int* col_of;        // device, src_cols entries, or null
  int nlayers, nmaps, rows, cols;
  int src_rows, src_cols;
  long long ncolumns;       // nmaps * nlayers * cols
};
// One k_map_cut_windows launch for every column of every window and layer (none when there is no column).
void launch_cut_windows(const WindowCut& a, int sms, cudaStream_t s);

// te_image.cu — addLayerFromImage for mono images: nmaps row-major images of rows x cols pixels (image m at px + m * image_stride
// bytes, its row i at + i * row_stride bytes; device memory, 2-byte pixels at even addresses and strides) into nmaps column-major
// float32 layers back to back at out: out[m*rows*cols + j*rows + i] = lower + diff * (pixel(m, i, j) / max pixel value).
struct ImageToLayer {
  const void* px;
  long long row_stride, image_stride;
  int rows, cols, nmaps;  // nmaps 1..65535
  int bpp;                // 1: mono8, 2: mono16 (host byte order)
  float lower, diff;      // lowerValue and mapValueDifference = upperValue - lowerValue
  float* out;
};
// One k_image_to_layer launch for every map.
void launch_image_to_layer(const ImageToLayer& a, cudaStream_t s);

}  // namespace te
