// TEST HARNESS (CPU suite only): drives harness_preprocess_raw_frame (tests/harness/preprocess_raw_host.cpp) over ragged image
// sizes, every median iteration count and pyramid level, under -fsanitize=address,undefined with exactly-sized buffers, so that
// an out-of-bounds access of stage 0 (grown halo, box reads of the full-resolution depth, colour blocks) is caught.
#include <cstdint>
#include <cstdio>
#include <cstdlib>
#include <vector>
extern "C" int harness_preprocess_raw_frame(int w, int h, const float depth_K[4], float raw_to_float, float a, int cell, int cf_w,
                                            const float* cfactor, float sigma_xy, float sigma_inv_depth, float radius_factor,
                                            float max_depth_m, int median_iterations, int depth_level, int color_level, int raw_w,
                                            int raw_h, const uint16_t* raw_depth, uint16_t* out_depth, uint16_t* out_normals,
                                            uint16_t* out_radius, int cw, int ch, const uint8_t* rgb, uint8_t* rgba, float* min_max);
int main() {
  // raw sizes; the depth camera is int(W / 2^L + 0.5) (kept when it is at most W <= w 2^L, as the library requires)
  int sizes[][2] = {{70, 45}, {33, 31}, {8, 5}, {3, 3}, {1, 1}, {65, 33}, {139, 97}};
  // (median iterations, depth level, colour level, sigma_xy)
  int modes[][3] = {{1, 0, 0}, {2, 0, 1}, {8, 0, 0}, {0, 1, 1}, {0, 2, 2}, {0, 3, 3}, {0, 0, 2}};
  float sig[] = {1.5f, 0.2f, 8.0f};
  int runs = 0;
  for (auto& s : sizes) for (auto& m : modes) for (float sg : sig) {
    const int W = s[0], H = s[1], n = m[0], ld = m[1], lc = m[2];
    const int w = static_cast<int>(W / static_cast<double>(1 << ld) + 0.5), h = static_cast<int>(H / static_cast<double>(1 << ld) + 0.5);
    if (w < 1 || h < 1 || W > (w << ld) || H > (h << ld)) continue;
    const int cw = w, ch = h, cell = 4, cf_w = (w - 1) / cell + 1, cf_h = (h - 1) / cell + 1;
    std::vector<float> cf(cf_w * cf_h, 1e-3f);
    std::vector<uint16_t> raw(W * H), d(w * h), nn(w * h), r(w * h);
    std::vector<uint8_t> rgb(3 * (cw << lc) * (ch << lc)), rgba(4 * cw * ch);
    for (int i = 0; i < W * H; ++i) raw[i] = (rand() % 3 == 0) ? 0 : 1500 + (i % W) + rand() % 4;
    for (auto& v : rgb) v = rand() & 255;
    float K[4] = {0.5f * h + 7, 0.5f * h + 7, 0.5f * w - 0.5f, 0.5f * h - 0.5f}, mm[2];
    const int t = harness_preprocess_raw_frame(w, h, K, 1e-3f, 0.02f, cell, cf_w, cf.data(), sg, 0.005f, 2.0f, 3.0f, n, ld, lc, W, H,
                                               raw.data(), d.data(), nn.data(), r.data(), cw, ch, rgb.data(), rgba.data(), mm);
    printf("%dx%d -> %dx%d n %d depth level %d colour level %d sigma %.1f: %d tiles\n", W, H, w, h, n, ld, lc, sg, t);
    ++runs;
  }
  printf("%d runs\n", runs);
  return 0;
}
