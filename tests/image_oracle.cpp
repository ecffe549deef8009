/*
 * image_oracle.cpp — CPU ORACLE of the reference node's image path (test infrastructure, NOT product code): te_image_geometry and
 * the elevation layer of te_map_chain_image(_maps) are checked against it.
 *
 * TraversabilityEstimation::imageCallback (TraversabilityEstimation.cpp:154-168) calls, on the first image,
 * GridMapRosConverter::initializeFromImage(image, imageResolution_, map, imagePosition_) and, on every image,
 * GridMapRosConverter::addLayerFromImage(image, "elevation", map, imageMinHeight_, imageMaxHeight_).
 *
 * RECALLED from grid_map 1.6.x (grid_map is not part of the reference checkout; like SURVEY.md Appendix A.1):
 *   initializeFromImage: map.setGeometry(Length(resolution * image.height, resolution * image.width), resolution, position)
 *   GridMap::setGeometry: size(k) = static_cast<int>(round(length(k) / resolution)); length_ = size.cast<double>() * resolution;
 *     position_ = position; startIndex_ = 0
 *   addLayerFromImage(image, layer, map, const float lowerValue, const float upperValue): the node's double heights are rounded
 *     to float at the call; CV_8UC1 and CV_16UC1 go to GridMapCvConverter::addLayerFromImage<uchar|ushort, 1>, which for every
 *     map index (imageIndex = the unwrapped index = the index, start index 0) sets
 *       mapValueDifference = upperValue - lowerValue                                    (float)
 *       data(i, j) = lowerValue + mapValueDifference * ((float)image.at(i, j) / maxImageValue)
 *     with maxImageValue = 255.0f (uchar) or 65535.0f (ushort).
 * Every operation is float32 and IEEE-rounded: the reference's host build targets x86-64 without FMA, and this file is compiled
 * with -ffp-contract=off.  Image row i is map row i, so the column-major layer is the image transposed.
 */
#include <cmath>
#include <cstdint>

template <class T>
static void layer(const unsigned char* image, int64_t rows, int64_t cols, int64_t row_stride, float lowerValue, float upperValue,
                  float maxImageValue, float* out) {
  const float mapValueDifference = upperValue - lowerValue;
  for (int64_t i = 0; i < rows; ++i) {
    const T* row = reinterpret_cast<const T*>(image + i * row_stride);
    for (int64_t j = 0; j < cols; ++j) out[j * rows + i] = lowerValue + mapValueDifference * ((float)row[j] / maxImageValue);
  }
}

extern "C" {

/* 6 doubles: rows, cols, length_x, length_y, position_x, position_y. */
void teo_image_geometry(int32_t height, int32_t width, double resolution, double position_x, double position_y, double* out) {
  const double length_x = resolution * height, length_y = resolution * width;
  const int rows = static_cast<int>(std::round(length_x / resolution));
  const int cols = static_cast<int>(std::round(length_y / resolution));
  out[0] = rows;
  out[1] = cols;
  out[2] = static_cast<double>(rows) * resolution;
  out[3] = static_cast<double>(cols) * resolution;
  out[4] = position_x;
  out[5] = position_y;
}

/* One image (bytes_per_pixel 1: mono8, 2: mono16, host byte order) into a column-major float32 layer of rows x cols. */
void teo_image_layer(int bytes_per_pixel, const void* image, int64_t rows, int64_t cols, int64_t row_stride, double min_height,
                     double max_height, float* out) {
  const float lower = (float)min_height, upper = (float)max_height;
  if (bytes_per_pixel == 1) layer<uint8_t>((const unsigned char*)image, rows, cols, row_stride, lower, upper, 255.0f, out);
  else layer<uint16_t>((const unsigned char*)image, rows, cols, row_stride, lower, upper, 65535.0f, out);
}

}  // extern "C"
