/* oracle/preprocess_raw_oracle.c -- TEST INFRASTRUCTURE ONLY.
 *
 * CPU restatement of the host stages BadSlam::PreprocessFrame runs before it uploads a frame (bad_slam.cc:649-689): the median
 * densify filter, the median downscaling of the depth and the colour image pyramid -- what bba_preprocess_raw_frame runs as
 * stage 0 of the fused kernel.  Dense row-major images, one function per reference function.  Built on demand by
 * oracle/preprocess_raw_oracle.py (plain C, no OpenMP).
 *
 * PARITY STATUS: **parity unpinned**.  The reference's versions are host code on libvis::Image, which needs Eigen, so they
 * cannot be built into oracle/_ref.  The restatements are anchored on an independent numpy restatement, hand-built cases and
 * libvis's own DownscaleToHalfSize test (tests/test_oracle_preprocess_raw.py).
 */
#include <math.h>
#include <stdint.h>
#include <stdlib.h>

static int orc_cmp_u16(const void* a, const void* b) {
  const uint16_t x = *(const uint16_t*)a, y = *(const uint16_t*)b;
  return (x > y) - (x < y);
}

/* std::sort of `values`, then the middle element (preprocessing.cc:66-79, image.h:1036-1047); an even count takes the lower
 * middle value if |low - mean| < |high - mean| (strict, fp32 mean of the sorted values), else the upper one. */
static uint16_t orc_sorted_median(uint16_t* values, int count) {
  qsort(values, (size_t)count, sizeof(uint16_t), orc_cmp_u16);
  if (count % 2 == 1) return values[count / 2];
  float sum = 0;
  for (int i = 0; i < count; ++i) sum += values[i];
  const float average = sum / count;
  const float prev_diff = fabsf(values[count / 2 - 1] - average);
  const float next_diff = fabsf(values[count / 2] - average);
  return (prev_diff < next_diff) ? values[count / 2 - 1] : values[count / 2];
}

/* MedianFilterAndDensifyDepthMap (preprocessing.cc:40-85): one pass, 3x3 window clamped to the image, zeros excluded, at least
 * 2 values (else the pixel keeps its input value). */
void orc_median_filter_and_densify(int w, int h, const uint16_t* in, uint16_t* out) {
  for (int y = 0; y < h; ++y) {
    for (int x = 0; x < w; ++x) {
      uint16_t values[9];
      int count = 0;
      for (int dy = (y - 1 > 0 ? y - 1 : 0); dy <= (y + 1 < h - 1 ? y + 1 : h - 1); ++dy)
        for (int dx = (x - 1 > 0 ? x - 1 : 0); dx <= (x + 1 < w - 1 ? x + 1 : w - 1); ++dx)
          if (in[(size_t)dy * w + dx] != 0) values[count++] = in[(size_t)dy * w + dx];
      out[(size_t)y * w + x] = (count >= 2) ? orc_sorted_median(values, count) : in[(size_t)y * w + x];
    }
  }
}

/* Image::DownscaleUsingMedianWhileExcluding(0, out_w, out_h) (libvis image.h:1003-1053): box [W x / w, W (x + 1) / w) x
 * [H y / h, H (y + 1) / h) in u32 arithmetic, median of its non-zero pixels, 0 for a box without one. */
void orc_downscale_using_median_excluding_zero(int in_w, int in_h, const uint16_t* in, int out_w, int out_h, uint16_t* out) {
  uint16_t* values = (uint16_t*)malloc(sizeof(uint16_t) * (size_t)in_w * in_h);
  for (uint32_t y = 0; y < (uint32_t)out_h; ++y) {
    for (uint32_t x = 0; x < (uint32_t)out_w; ++x) {
      const uint32_t start_x = ((uint32_t)in_w * x) / (uint32_t)out_w, end_x = ((uint32_t)in_w * (x + 1)) / (uint32_t)out_w;
      const uint32_t start_y = ((uint32_t)in_h * y) / (uint32_t)out_h, end_y = ((uint32_t)in_h * (y + 1)) / (uint32_t)out_h;
      int count = 0;
      for (uint32_t oy = start_y; oy < end_y; ++oy)
        for (uint32_t ox = start_x; ox < end_x; ++ox)
          if (in[(size_t)oy * in_w + ox] != 0) values[count++] = in[(size_t)oy * in_w + ox];
      out[(size_t)y * out_w + x] = count ? orc_sorted_median(values, count) : 0;
    }
  }
  free(values);
}

/* Image<Vec3u8>::DownscaleToHalfSize (libvis image.h:929-948), one level of ImagePyramid (image_cache.h:205-231): in_w and in_h
 * even (the reference CHECKs it; returns -1 otherwise), a/4 + b/4 + c/4 + d/4 per channel with truncation. */
int orc_downscale_rgb_to_half_size(int in_w, int in_h, const uint8_t* in, uint8_t* out) {
  if (in_w % 2 != 0 || in_h % 2 != 0) return -1;
  const int w = in_w / 2, h = in_h / 2;
  for (int y = 0; y < h; ++y) {
    const uint8_t* upper = in + (size_t)(2 * y) * in_w * 3;
    const uint8_t* lower = upper + (size_t)in_w * 3;
    for (int x = 0; x < w; ++x)
      for (int c = 0; c < 3; ++c)
        out[((size_t)y * w + x) * 3 + c] = (uint8_t)(upper[6 * x + c] / 4 + upper[6 * x + 3 + c] / 4 + lower[6 * x + c] / 4 +
                                                     lower[6 * x + 3 + c] / 4);
  }
  return 0;
}
