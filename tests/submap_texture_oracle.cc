// CPU restatement of the submap textures — TEST INFRASTRUCTURE ONLY.
//
// Written from the reference's behaviour, sequentially and per element as the reference does it:
//   * 3D (mapping/3d/submap_3d.cc:51-176): ExtractVoxelData over a voxel list in HybridGrid's
//     iteration order (tests/hybrid_grid_walk.cc gives that order), AccumulatePixelData into a
//     width x height vector of PixelData, ComputePixelValues, and the slice pose.
//   * 2D (probability_grid.cc:109-147, internal/2d/tsdf_2d.cc:137-181, grid_2d.cc:110-120):
//     DrawToSubmapTexture over the cropped limits, ProbabilityToLogOddsInteger evaluated directly
//     with the host's logf and the TSDF power with the host's powf.
// Float arithmetic is compiled with -ffp-contract=off.  The Rigid3f transform is csrc/rigid3f.h
// (the Eigen restatement the 3D matchers are checked with); the step table, the gzip member and
// the double slice pose are the library's own host code (csrc/submap_texture.h), exported here so
// that they can be checked on a machine without a GPU.
#include <climits>
#include <cmath>
#include <cstdint>
#include <cstring>
#include <string>
#include <vector>

#include "../cartographer_b200/csrc/rigid3f.h"
#include "../cartographer_b200/csrc/submap_texture.h"

namespace {

constexpr float kMinP = 0.1f;
constexpr float kMaxP = 1.f - kMinP;

float Logit(float p) { return std::log(p / (1.f - p)); }

// mapping/submaps.h:37-53
int ProbabilityToLogOddsInteger(float probability) {
  const float kMaxLogOdds = Logit(kMaxP);
  const float kMinLogOdds = Logit(kMinP);
  return static_cast<int>(std::lround((Logit(probability) - kMinLogOdds) * 254.f /
                                      (kMaxLogOdds - kMinLogOdds))) +
         1;
}

// probability_values.h / value_conversion_tables.cc: value -> float over [lo, hi]
float ValueToFloat(int value, float lo, float hi) {
  const float scale = (hi - lo) / 32766.f;
  return value * scale + (lo - scale);
}

void PushDelta(int delta, std::vector<uint8_t>* cells) {
  const uint8_t alpha = delta > 0 ? 0 : -delta;
  const uint8_t value = delta > 0 ? delta : 0;
  cells->push_back(value);
  cells->push_back((value || alpha) ? alpha : 1);
}

struct PixelData {
  int min_z = INT_MAX;
  int max_z = INT_MIN;
  int count = 0;
  float probability_sum = 0.f;
  float max_probability = 0.5f;
};

void PutSlice(const csm::Pose3d& s, double* out) {
  const double v[7] = {s.t.x, s.t.y, s.t.z, s.q.w, s.q.x, s.q.y, s.q.z};
  std::memcpy(out, v, sizeof(v));
}

csm::Pose3d PoseOf(const double* p) {
  return csm::Pose3d{csm::Vec3d{p[0], p[1], p[2]}, csm::Quat4d{p[3], p[4], p[5], p[6]}};
}

}  // namespace

extern "C" {

int sto_log_odds_integer(float p) { return ProbabilityToLogOddsInteger(p); }

// The step table's value for p (the device's lookup, on the host).
int sto_log_odds_from_steps(float p) {
  static const csm::LogOddsSteps steps = csm::MakeLogOddsSteps();
  return csm::LogOddsIntegerFromSteps(p, steps.t);
}

void sto_steps(float* out) {
  const csm::LogOddsSteps steps = csm::MakeLogOddsSteps();
  std::memcpy(out, steps.t, sizeof(steps.t));
}

// Every float in [kMinProbability, kMaxProbability] through the table against the direct
// function: the number of floats checked in *checked and of mismatches returned (the first one
// in *first).
int64_t sto_log_odds_exhaustive(int64_t* checked, float* first) {
  const csm::LogOddsSteps steps = csm::MakeLogOddsSteps();
  uint32_t lo, hi;
  std::memcpy(&lo, &kMinP, 4);
  std::memcpy(&hi, &kMaxP, 4);
  int64_t bad = 0;
  *checked = 0;
  for (uint32_t b = lo; b <= hi; ++b) {
    float p;
    std::memcpy(&p, &b, 4);
    ++*checked;
    if (csm::LogOddsIntegerFromSteps(p, steps.t) != ProbabilityToLogOddsInteger(p)) {
      if (bad == 0) *first = p;
      ++bad;
    }
  }
  return bad;
}

// AddToTextureProto's data for n voxels (idx n x 3, values) in iteration order: the raw cells
// (2 * width * height bytes, at most `capacity`), width, height and the slice pose
// {tx, ty, tz, qw, qx, qy, qz}.  Returns the number of cell bytes (-1 if over capacity).
int64_t sto_texture3d(const int32_t* idx, const uint16_t* values, int64_t n, float resolution,
                      const double* pose, uint8_t* cells_out, int64_t capacity, int32_t* width_out,
                      int32_t* height_out, double* slice_out) {
  const csm::Rigid3f transform{
      csm::Vec3f{static_cast<float>(pose[0]), static_cast<float>(pose[1]),
                 static_cast<float>(pose[2])},
      csm::Quatf{static_cast<float>(pose[3]), static_cast<float>(pose[4]),
                 static_cast<float>(pose[5]), static_cast<float>(pose[6])}};
  // ExtractVoxelData
  int min_index[2] = {INT_MAX, INT_MAX};
  int max_index[2] = {INT_MIN, INT_MIN};
  std::vector<int> voxels;   // x, y, z, value
  const float resolution_inverse = 1.f / resolution;
  for (int64_t i = 0; i < n; ++i) {
    const float probability = ValueToFloat(values[i], kMinP, kMaxP);
    if (probability < 0.501f) continue;
    const csm::Vec3f center{idx[3 * i] * resolution, idx[3 * i + 1] * resolution,
                            idx[3 * i + 2] * resolution};
    const csm::Vec3f g = csm::Rigid3Apply(transform, center);
    const int v[4] = {static_cast<int>(std::lround(g.x * resolution_inverse)),
                      static_cast<int>(std::lround(g.y * resolution_inverse)),
                      static_cast<int>(std::lround(g.z * resolution_inverse)), values[i]};
    voxels.insert(voxels.end(), v, v + 4);
    for (int a = 0; a < 2; ++a) {
      min_index[a] = std::min(min_index[a], v[a]);
      max_index[a] = std::max(max_index[a], v[a]);
    }
  }
  // int arithmetic with x86-64's wrap-around (the reference's signed overflow when no voxel
  // passed), spelled in unsigned
  const int width = static_cast<int>(static_cast<unsigned>(max_index[1]) -
                                     static_cast<unsigned>(min_index[1]) + 1u);
  const int height = static_cast<int>(static_cast<unsigned>(max_index[0]) -
                                      static_cast<unsigned>(min_index[0]) + 1u);
  *width_out = width;
  *height_out = height;
  // AccumulatePixelData
  std::vector<PixelData> pixels(static_cast<size_t>(width) * height);
  for (size_t k = 0; k < voxels.size(); k += 4) {
    const int* v = &voxels[k];
    if (v[0] < min_index[0] || v[1] < min_index[1] || v[0] > max_index[0] || v[1] > max_index[1])
      continue;
    PixelData& pixel = pixels[(max_index[0] - v[0]) * width + (max_index[1] - v[1])];
    ++pixel.count;
    pixel.min_z = std::min(pixel.min_z, v[2]);
    pixel.max_z = std::max(pixel.max_z, v[2]);
    const float probability = ValueToFloat(v[3], kMinP, kMaxP);
    pixel.probability_sum += probability;
    pixel.max_probability = std::max(pixel.max_probability, probability);
  }
  // ComputePixelValues
  std::vector<uint8_t> cells;
  for (const PixelData& pixel : pixels) {
    const float z_difference = pixel.count > 0 ? pixel.max_z - pixel.min_z : 0;
    if (z_difference < 3.f) {
      cells.push_back(0);
      cells.push_back(0);
      continue;
    }
    const float free_space = std::max(z_difference - pixel.count, 0.f);
    const float free_space_weight = 0.15f * free_space;
    const float total_weight = pixel.count + free_space_weight;
    const float free_space_probability = 1.f - pixel.max_probability;
    float average = (pixel.probability_sum + free_space_probability * free_space_weight) /
                    total_weight;
    average = average > kMaxP ? kMaxP : (average < kMinP ? kMinP : average);
    PushDelta(128 - ProbabilityToLogOddsInteger(average), &cells);
  }
  const csm::Pose3d global = PoseOf(pose);
  PutSlice(csm::InverseTimesTranslation(
               global, csm::Vec3d{max_index[0] * resolution, max_index[1] * resolution,
                                  global.t.z}),
           slice_out);
  if (static_cast<int64_t>(cells.size()) > capacity) return -1;
  std::memcpy(cells_out, cells.data(), cells.size());
  return static_cast<int64_t>(cells.size());
}

// DrawToSubmapTexture of a grid of nx x ny cells (row-major, x fastest; wcells != NULL for a
// TSDF2D with the converter (truncation, max_weight)) whose known-cells box is
// box = {min x, min y, max x, max y} (empty when min x > max x).
int64_t sto_texture2d(const uint16_t* cells, const uint16_t* wcells, int32_t nx, int32_t ny,
                      const int32_t* box, double resolution, double max_x, double max_y,
                      float truncation, float max_weight, const double* pose, uint8_t* cells_out,
                      int64_t capacity, int32_t* width_out, int32_t* height_out,
                      double* slice_out) {
  int offset[2] = {0, 0};
  int limits[2] = {1, 1};
  if (box[0] <= box[2]) {
    offset[0] = box[0];
    offset[1] = box[1];
    limits[0] = box[2] - box[0] + 1;
    limits[1] = box[3] - box[1] + 1;
  }
  std::vector<uint8_t> out;
  for (int y = 0; y < limits[1]; ++y)
    for (int x = 0; x < limits[0]; ++x) {
      const size_t at = static_cast<size_t>(y + offset[1]) * nx + (x + offset[0]);
      const uint16_t v = cells[at];
      if (v == 0) {
        out.push_back(0);
        out.push_back(0);
        continue;
      }
      int delta;
      if (wcells == nullptr) {
        const float probability =
            1.f - ValueToFloat(v, 1.f - kMaxP, 1.f - kMinP);   // 1 - correspondence cost
        delta = 128 - ProbabilityToLogOddsInteger(probability);
      } else {
        const float tsd = ValueToFloat(v, -truncation, truncation);
        const float weight = wcells[at] == 0 ? 0.f : ValueToFloat(wcells[at], 0.f, max_weight);
        float normalized_tsdf = std::abs(tsd);
        normalized_tsdf = std::pow(normalized_tsdf / truncation, 0.5f);
        const float normalized_weight = weight / max_weight;
        delta = static_cast<int>(std::round(normalized_weight * (normalized_tsdf * 255. - 128.)));
      }
      PushDelta(delta, &out);
    }
  *width_out = limits[0];
  *height_out = limits[1];
  const double mx = max_x - resolution * offset[1];
  const double my = max_y - resolution * offset[0];
  PutSlice(csm::InverseTimesTranslation(PoseOf(pose), csm::Vec3d{mx, my, 0.}), slice_out);
  (void)ny;
  if (static_cast<int64_t>(out.size()) > capacity) return -1;
  std::memcpy(cells_out, out.data(), out.size());
  return static_cast<int64_t>(out.size());
}

const char* sto_zlib_version() { return zlibVersion(); }

// The library's gzip member of data[0 .. n) into out (at most capacity bytes): its length, or
// -1.
int64_t sto_gzip(const uint8_t* data, int64_t n, uint8_t* out, int64_t capacity) {
  std::string z;
  if (!csm::GzipMember(data, static_cast<size_t>(n), &z)) return -1;
  if (static_cast<int64_t>(z.size()) > capacity) return -1;
  std::memcpy(out, z.data(), z.size());
  return static_cast<int64_t>(z.size());
}

}  // extern "C"
