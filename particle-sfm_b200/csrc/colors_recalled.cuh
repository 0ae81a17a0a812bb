// colors_recalled.cuh — the image sampling of the colour extraction that restates a library the reference links but
// does not vendor: COLMAP 3.8's Bitmap::InterpolateBilinear on the 24-bit RGB bitmap Bitmap::Read(as_rgb = true)
// leaves, which Reconstruction::ExtractColorsForAllImages (reference base/reconstruction.cc:1250-1300) calls.  It is
// recalled, not pinned to a source line; oracle/colors_oracle.py restates the same function (RECALLED).  A correction
// is a change on each side.
#pragma once

namespace psfm {
namespace colors {

// ExtractColorsForAllImages samples at (X - 0.5, Y - 0.5): COLMAP puts the centre of the upper-left pixel at (0.5, 0.5)
constexpr double kPixelCentre = 0.5;

#ifdef __CUDACC__
// Bitmap::InterpolateBilinear(x, y, &color) on a top-down RGB8 image px [h][w][3].  FreeImage stores scanlines bottom
// up, so the function works on inv_y = h - 1 - y and scanline s is top-down row h - 1 - s:
//   x0 = floor(x), x1 = x0 + 1, y0 = floor(inv_y), y1 = y0 + 1; false if x0 < 0 || x1 >= w || y0 < 0 || y1 >= h
//   c  = dx_1 dy_1 p00 + dx dy_1 p01 + dx_1 dy p10 + dx dy p11 in double, left to right, stored as float
// p00 / p01 are columns x0 / x1 of scanline y0, p10 / p11 the same columns of scanline y1.  The bounds are tested on
// the floors in double, before the cast to int, so a NaN or a coordinate beyond int's range is no sample (the
// reference's cast is undefined there).  The unit is compiled with -fmad=false: no product is contracted.
__device__ __forceinline__ bool interpolate_bilinear(const unsigned char* px, int w, int h, double x, double y,
                                                     float* rgb) {
  const double inv_y = (double)(h - 1) - y;
  const double fx = floor(x), fy = floor(inv_y);
  if (!(fx >= 0.0 && fx <= (double)(w - 2) && fy >= 0.0 && fy <= (double)(h - 2))) return false;
  const int x0 = (int)fx, y0 = (int)fy;
  const double dx = x - x0, dy = inv_y - y0, dx_1 = 1 - dx, dy_1 = 1 - dy;
  const unsigned char* line0 = px + (size_t)(h - 1 - y0) * 3 * w;
  const unsigned char* line1 = px + (size_t)(h - 2 - y0) * 3 * w;
  const unsigned char *p00 = line0 + 3 * x0, *p01 = p00 + 3, *p10 = line1 + 3 * x0, *p11 = p10 + 3;
#pragma unroll
  for (int c = 0; c < 3; ++c)
    rgb[c] = (float)(dx_1 * dy_1 * p00[c] + dx * dy_1 * p01[c] + dx_1 * dy * p10[c] + dx * dy * p11[c]);
  return true;
}
#endif

}  // namespace colors
}  // namespace psfm
