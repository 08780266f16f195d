// A single-thread restatement of io::DrawProbabilityGrid (io/probability_grid_points_processor.cc)
// for the tests of csm_rt_grid2d_draw: the cropped limits of a grid's known-cells box, and per
// cell the grey level the reference computes, each float step in float, evaluated per cell (no
// table).  Built with -ffp-contract=off, so no step is fused.
#include <cmath>
#include <cstdint>

namespace {

constexpr float kMinProbability = 0.1f;                       // probability_values.h
constexpr float kMaxProbability = 1.f - kMinProbability;
constexpr float kMinCorrespondenceCost = 1.f - kMaxProbability;
constexpr float kMaxCorrespondenceCost = 1.f - kMinProbability;
constexpr uint8_t kUnknownValue = 128;

// The correspondence cost of a known cell value: values 1..32767 spread linearly over
// [kMinCorrespondenceCost, kMaxCorrespondenceCost].
float CorrespondenceCost(int value) {
  const float step = (kMaxCorrespondenceCost - kMinCorrespondenceCost) / 32766.f;
  return value * step + (kMinCorrespondenceCost - step);
}

// 255 * the probability of "free" (1 - GetProbability) rescaled to [0, 1], before rounding.
float Scaled(int value) {
  const float probability_of_hit = 1.f - CorrespondenceCost(value);   // GetProbability
  const float probability = 1.f - probability_of_hit;
  return 255 * ((probability - kMinProbability) / (kMaxProbability - kMinProbability));
}

uint8_t Grey(int value) {
  if (value == 0) return kUnknownValue;
  return static_cast<uint8_t>(std::lround(Scaled(value)));
}

}  // namespace

extern "C" {

int pgd_grey(int value) { return Grey(value); }

float pgd_scaled(int value) { return Scaled(value); }

// The image of a grid of cells[y * nx + x] with known-cells box {min x, min y, max x, max y}
// (box == nullptr: empty).  out = {width, height, offset x, offset y}; with pixels != nullptr
// pixel (x, y) goes to pixels[y * width + x] as a cairo ARGB32 word.
void pgd_draw(const uint16_t* cells, int nx, int ny, const int* box, int* out, uint32_t* pixels) {
  int ox = 0, oy = 0, width = 1, height = 1;
  if (box != nullptr) {
    ox = box[0];
    oy = box[1];
    width = box[2] - box[0] + 1;
    height = box[3] - box[1] + 1;
  }
  out[0] = width;
  out[1] = height;
  out[2] = ox;
  out[3] = oy;
  if (pixels == nullptr) return;
  for (int y = 0; y < height; ++y) {
    for (int x = 0; x < width; ++x) {
      const int cx = ox + x, cy = oy + y;
      const bool inside = cx >= 0 && cy >= 0 && cx < nx && cy < ny;
      const int value = inside ? cells[static_cast<long long>(cy) * nx + cx] : 0;
      const uint32_t v = Grey(value);
      pixels[static_cast<long long>(y) * width + x] = 0xFF000000u | v << 16 | v << 8 | v;
    }
  }
}

}  // extern "C"
