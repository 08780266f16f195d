// CPU restatement of io::XRayPointsProcessor's Insert, WriteVoxels and IntoImage
// (io/xray_points_processor.cc:65-104, 170-239), written from their semantics: the parity
// reference of the device processor (cartographer_b200/csrc/xray.cu) and the host column of
// benchmarks/bench_xray.py.  One thread, ordered std::maps of voxels and columns, every float and
// double step as the reference's C++ types make it; build with -ffp-contract=off.  The transform
// is rigid3f.h's restatement of Eigen's Rigid3f * point.  Loaded by tests/xray_oracle.py.
#include <algorithm>
#include <array>
#include <cmath>
#include <cstdint>
#include <limits>
#include <map>
#include <set>
#include <utility>
#include <vector>

#include "../cartographer_b200/csrc/rigid3f.h"

namespace {

struct ColumnData {
  float sum_r = 0.f, sum_g = 0.f, sum_b = 0.f;
  uint32_t count = 0;
};

struct Aggregation {
  std::set<std::array<int, 3>> voxels;                    // (x, y, z)
  std::map<std::pair<int, int>, ColumnData> column_data;  // (y, z)
};

struct Processor {
  float resolution;
  double saturation_factor;
  csm::Rigid3f transform;
  std::vector<Aggregation> aggregations;
  bool empty = true;
  std::array<int, 3> lo{}, hi{};
};

// common::RoundToInt: std::lround narrowed to int.
int RoundToInt(float v) { return static_cast<int>(std::lround(v)); }

std::array<int, 3> CellIndex(const Processor& p, const float* point) {
  const csm::Vec3f q = csm::Rigid3Apply(p.transform, csm::Vec3f{point[0], point[1], point[2]});
  return {RoundToInt(q.x / p.resolution), RoundToInt(q.y / p.resolution),
          RoundToInt(q.z / p.resolution)};
}

bool InGrowableCube(const std::array<int, 3>& index) {
  for (int v : index)
    if (v < -8192 || v >= 8192) return false;
  return true;
}

// Mix (xray_points_processor.cc:65-67): a * (1. - t) is a double, t * b a float.
float Mix(const float a, const float b, const float t) { return a * (1. - t) + t * b; }

// io/color.h FloatComponentToUint8.
uint8_t ToUint8(float c) {
  const float clamped = c > 1.f ? 1.f : (c < 0.f ? 0.f : c);
  return static_cast<uint8_t>(RoundToInt(clamped * 255));
}

uint32_t Cairo(uint8_t r, uint8_t g, uint8_t b) {
  return static_cast<uint32_t>(255) << 24 | static_cast<uint32_t>(r) << 16 |
         static_cast<uint32_t>(g) << 8 | b;
}

}  // namespace

extern "C" {

// transform = {t x, y, z, q w, x, y, z}.
void* xo_create(double voxel_size, double saturation_factor, const float* transform,
                int num_aggregations) {
  Processor* p = new Processor;
  p->resolution = static_cast<float>(voxel_size);
  p->saturation_factor = saturation_factor;
  p->transform = csm::Rigid3f{csm::Vec3f{transform[0], transform[1], transform[2]},
                              csm::Quatf{transform[3], transform[4], transform[5], transform[6]}};
  p->aggregations.resize(num_aggregations);
  return p;
}

void xo_destroy(void* h) { delete static_cast<Processor*>(h); }

// Insert of one batch (rgb == NULL: black).  Returns -1, changing nothing, when a cell lies
// outside the cells the reference's grid can grow to (its CHECK would abort); else 0.
int xo_insert(void* h, int aggregation, const float* xyz, const float* rgb, int n) {
  Processor& p = *static_cast<Processor*>(h);
  for (int i = 0; i < n; ++i)
    if (!InGrowableCube(CellIndex(p, xyz + 3 * i))) return -1;
  Aggregation& a = p.aggregations[aggregation];
  const float black[3] = {0.f, 0.f, 0.f};
  for (int i = 0; i < n; ++i) {
    const std::array<int, 3> index = CellIndex(p, xyz + 3 * i);
    a.voxels.insert(index);
    for (int k = 0; k < 3; ++k) {
      p.lo[k] = p.empty ? index[k] : std::min(p.lo[k], index[k]);
      p.hi[k] = p.empty ? index[k] : std::max(p.hi[k], index[k]);
    }
    p.empty = false;
    ColumnData& column = a.column_data[std::make_pair(index[1], index[2])];
    const float* color = rgb ? rgb + 3 * i : black;
    column.sum_r += color[0];
    column.sum_g += color[1];
    column.sum_b += color[2];
    ++column.count;
  }
  return 0;
}

// The shared box; returns 1 while it is empty.
int xo_box(void* h, int* lo, int* hi) {
  const Processor& p = *static_cast<Processor*>(h);
  for (int k = 0; k < 3; ++k) {
    lo[k] = p.lo[k];
    hi[k] = p.hi[k];
  }
  return p.empty;
}

// One channel of IntoImage: Mix(1.f, mean, saturation) as a byte.
int xo_channel(float mean, float saturation) { return ToUint8(Mix(1.f, mean, saturation)); }

// WriteVoxels + IntoImage of one aggregation into pixels (cairo words, row-major); with
// pixels == NULL only the size.  Returns -1 (and 0 x 0) when the box is empty.
int xo_draw(void* h, int aggregation, uint32_t* pixels, int* width, int* height) {
  const Processor& p = *static_cast<Processor*>(h);
  *width = *height = 0;
  if (p.empty) return -1;
  const int w = p.hi[1] - p.lo[1] + 1, ht = p.hi[2] - p.lo[2] + 1;
  *width = w;
  *height = ht;
  if (!pixels) return 0;
  const Aggregation& a = p.aggregations[aggregation];
  struct PixelData {
    size_t n = 0;
    float mean_r = 0.f, mean_g = 0.f, mean_b = 0.f;
  };
  std::vector<PixelData> data(static_cast<size_t>(w) * ht);
  for (const auto& v : a.voxels) {
    PixelData& d = data[(p.hi[1] - v[1]) + static_cast<size_t>(p.hi[2] - v[2]) * w];
    const ColumnData& c = a.column_data.at(std::make_pair(v[1], v[2]));
    d.mean_r = c.sum_r / c.count;
    d.mean_g = c.sum_g / c.count;
    d.mean_b = c.sum_b / c.count;
    ++d.n;
  }
  float max = std::numeric_limits<float>::min();
  for (const PixelData& d : data)
    if (d.n != 0) max = std::max<float>(max, std::log(d.n));
  for (size_t i = 0; i < data.size(); ++i) {
    const PixelData& d = data[i];
    if (d.n == 0) {
      pixels[i] = Cairo(255, 255, 255);
      continue;
    }
    const float saturation = std::min<float>(1.0, std::log(d.n) / max * p.saturation_factor);
    pixels[i] = Cairo(ToUint8(Mix(1.f, d.mean_r, saturation)),
                      ToUint8(Mix(1.f, d.mean_g, saturation)),
                      ToUint8(Mix(1.f, d.mean_b, saturation)));
  }
  return 0;
}

// The aggregation's voxels in the set's (x, y, z) order; with indices == NULL only the count.
long long xo_voxels(void* h, int aggregation, int* indices) {
  const Aggregation& a = static_cast<Processor*>(h)->aggregations[aggregation];
  if (indices) {
    long long j = 0;
    for (const auto& v : a.voxels) {
      for (int k = 0; k < 3; ++k) indices[3 * j + k] = v[k];
      ++j;
    }
  }
  return static_cast<long long>(a.voxels.size());
}

// The aggregation's columns in ascending (y, z); with yz == NULL only the count.
long long xo_columns(void* h, int aggregation, int* yz, float* sums, uint32_t* counts) {
  const Aggregation& a = static_cast<Processor*>(h)->aggregations[aggregation];
  if (yz) {
    long long j = 0;
    for (const auto& c : a.column_data) {
      yz[2 * j] = c.first.first;
      yz[2 * j + 1] = c.first.second;
      sums[3 * j] = c.second.sum_r;
      sums[3 * j + 1] = c.second.sum_g;
      sums[3 * j + 2] = c.second.sum_b;
      counts[j] = c.second.count;
      ++j;
    }
  }
  return static_cast<long long>(a.column_data.size());
}

}  // extern "C"
