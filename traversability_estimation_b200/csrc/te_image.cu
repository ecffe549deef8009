// te_image.cu — GridMapCvConverter::addLayerFromImage for mono8 / mono16 images (k_image_to_layer): nmaps row-major images in,
// nmaps column-major float32 elevation layers out, in one launch.  Image row i is map row i, so each layer is its image
// transposed; a block stages a kTile x kTile tile in shared memory so that loads run along image rows and stores along layer
// columns.  Compiled with --fmad=false; the arithmetic is written with round-to-nearest intrinsics in the reference's operand
// order anyway, so its bits do not depend on compiler flags.
#include "te_kernels.h"

namespace te {
namespace {

constexpr int kTile = 64;      // pixels per tile side
constexpr int kThreads = 256;  // load: 16 threads x 4 pixels per image row; store: 64 threads per layer column

template <class T> struct Pixel;
template <> struct Pixel<unsigned char> { using V = uchar4; static constexpr float kMax = 255.0f; };     // CV_8UC1
template <> struct Pixel<unsigned short> { using V = ushort4; static constexpr float kMax = 65535.0f; };  // CV_16UC1

// elevation = lowerValue + mapValueDifference * ((float)pixel / maxImageValue), every operation float32 and IEEE-rounded.
template <class T>
__device__ __forceinline__ float pixel_to_height(T px, float lower, float diff) {
  return __fadd_rn(lower, __fmul_rn(diff, __fdiv_rn((float)px, Pixel<T>::kMax)));
}

// blockIdx.x: the tile (tile rows fastest), blockIdx.y: the map.  kVec: the images' base, row stride and image stride are
// multiples of 4 pixels (checked on the host), so a quad of pixels starting at a multiple-of-4 column is one aligned load.
template <class T, bool kVec>
__global__ void __launch_bounds__(kThreads) k_image_to_layer(ImageToLayer a) {
  using V = typename Pixel<T>::V;
  __shared__ float tile[kTile][kTile + 1];  // [image column][image row]
  const unsigned tiles_i = (unsigned)(a.rows + kTile - 1) / kTile;
  const int i0 = (int)(blockIdx.x % tiles_i) * kTile, j0 = (int)(blockIdx.x / tiles_i) * kTile;
  const unsigned char* img = (const unsigned char*)a.px + (long long)blockIdx.y * a.image_stride;

  const int q = threadIdx.x & 15, r = threadIdx.x >> 4, j = j0 + 4 * q;
  T px[4][4];
#pragma unroll
  for (int p = 0; p < 4; ++p) {
    const int i = i0 + r + 16 * p;
    if (i >= a.rows) continue;
    const T* row = (const T*)(img + (long long)i * a.row_stride);
    if (kVec && j + 3 < a.cols) {
      const V v = __ldg((const V*)(row + j));
      px[p][0] = v.x; px[p][1] = v.y; px[p][2] = v.z; px[p][3] = v.w;
    } else {
#pragma unroll
      for (int k = 0; k < 4; ++k)
        if (j + k < a.cols) px[p][k] = __ldg(row + j + k);
    }
  }
#pragma unroll
  for (int p = 0; p < 4; ++p) {
    const int il = r + 16 * p;
    if (i0 + il >= a.rows) continue;
#pragma unroll
    for (int k = 0; k < 4; ++k)
      if (j + k < a.cols) tile[4 * q + k][il] = pixel_to_height(px[p][k], a.lower, a.diff);
  }
  __syncthreads();

  const int il = threadIdx.x & 63, i = i0 + il;
  if (i >= a.rows) return;
  float* out = a.out + (size_t)blockIdx.y * a.rows * a.cols + i;
#pragma unroll
  for (int p = 0; p < kTile / 4; ++p) {
    const int jl = (threadIdx.x >> 6) + 4 * p;
    if (j0 + jl < a.cols) out[(size_t)(j0 + jl) * a.rows] = tile[jl][il];
  }
}

template <class T>
void launch_typed(const ImageToLayer& a, cudaStream_t s) {
  const unsigned tiles = (unsigned)((a.rows + kTile - 1) / kTile) * (unsigned)((a.cols + kTile - 1) / kTile);
  const dim3 grid(tiles, (unsigned)a.nmaps);
  const long long quad = 4 * (long long)sizeof(T);
  const bool vec = (uintptr_t)a.px % quad == 0 && a.row_stride % quad == 0 && (a.nmaps == 1 || a.image_stride % quad == 0);
  if (vec) k_image_to_layer<T, true><<<grid, kThreads, 0, s>>>(a);
  else k_image_to_layer<T, false><<<grid, kThreads, 0, s>>>(a);
}

}  // namespace

void launch_image_to_layer(const ImageToLayer& a, cudaStream_t s) {
  if (a.bpp == 1) launch_typed<unsigned char>(a, s);
  else launch_typed<unsigned short>(a, s);
}

}  // namespace te
