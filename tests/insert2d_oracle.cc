// CPU restatement of ProbabilityGridRangeDataInserter2D::Insert and the ProbabilityGrid pieces
// it touches (cartographer/mapping/2d/{probability_grid_range_data_inserter_2d,grid_2d,
// probability_grid}.cc, mapping/internal/2d/ray_to_pixel_mask.cc, mapping/probability_values.*).
// Sequential, as the reference runs: the parity reference of the device inserter
// (tests/test_gpu_insert2d.py) and the CPU column of benchmarks/bench_insert2d.py.  Test
// infrastructure, loaded through tests/insert2d_oracle.py; the product library never uses it.
// Build with -ffp-contract=off: float where the reference is float, double where it is double.
#include <algorithm>
#include <climits>
#include <cmath>
#include <cstdint>
#include <cstring>
#include <vector>

namespace {

constexpr int kValueCount = 32768;
constexpr uint16_t kUpdateMarker = 1u << 15;
constexpr int kSubpixelScale = 1000;
constexpr float kMinProbability = 0.1f;
constexpr float kMaxProbability = 1.f - kMinProbability;
constexpr float kMinCorrespondenceCost = 1.f - kMaxProbability;
constexpr float kMaxCorrespondenceCost = 1.f - kMinProbability;

template <typename T>
T Clamp(T v, T lo, T hi) {
  if (v > hi) return hi;
  if (v < lo) return lo;
  return v;
}
uint16_t BoundedFloatToValue(float f, float lo, float hi) {
  return static_cast<uint16_t>(
      static_cast<int>(std::lround((Clamp(f, lo, hi) - lo) * (32766.f / (hi - lo)))) + 1);
}
float Odds(float p) { return p / (1.f - p); }
float ProbabilityFromOdds(float o) { return o / (o + 1.f); }
float ProbabilityToCorrespondenceCost(float p) { return 1.f - p; }
float CorrespondenceCostToProbability(float c) { return 1.f - c; }
uint16_t CorrespondenceCostToValue(float c) {
  return BoundedFloatToValue(c, kMinCorrespondenceCost, kMaxCorrespondenceCost);
}
// kValueToCorrespondenceCost: SlowValueToBoundedFloat repeated for values with the marker
float ValueToCorrespondenceCost(uint16_t value) {
  const uint16_t v = value & static_cast<uint16_t>(kValueCount - 1);
  if (v == 0) return kMaxCorrespondenceCost;
  const float kScale = (kMaxCorrespondenceCost - kMinCorrespondenceCost) / (kValueCount - 2.f);
  return v * kScale + (kMinCorrespondenceCost - kScale);
}
std::vector<uint16_t> ComputeLookupTableToApplyCorrespondenceCostOdds(float odds) {
  std::vector<uint16_t> result;
  result.reserve(kValueCount);
  result.push_back(CorrespondenceCostToValue(ProbabilityToCorrespondenceCost(
                       ProbabilityFromOdds(odds))) + kUpdateMarker);
  for (int cell = 1; cell != kValueCount; ++cell)
    result.push_back(CorrespondenceCostToValue(ProbabilityToCorrespondenceCost(ProbabilityFromOdds(
                         odds * Odds(CorrespondenceCostToProbability(
                                    ValueToCorrespondenceCost(static_cast<uint16_t>(cell))))))) +
                     kUpdateMarker);
  return result;
}

struct XY { int x, y; };

struct Limits {
  double resolution, max_x, max_y;
  int nx, ny;
  XY GetCellIndex(float px, float py) const {
    return XY{static_cast<int>(std::lround((max_y - py) / resolution - 0.5)),
              static_cast<int>(std::lround((max_x - px) / resolution - 0.5))};
  }
  bool Contains(XY c) const { return c.x >= 0 && c.y >= 0 && c.x < nx && c.y < ny; }
};

struct Grid {
  Limits limits;
  std::vector<uint16_t> cells;
  std::vector<int> update_indices;
  bool box_empty = true;
  int box_min[2] = {0, 0}, box_max[2] = {0, 0};

  void Extend(XY c) {
    if (box_empty) {
      box_min[0] = box_max[0] = c.x;
      box_min[1] = box_max[1] = c.y;
      box_empty = false;
      return;
    }
    box_min[0] = std::min(box_min[0], c.x);
    box_min[1] = std::min(box_min[1], c.y);
    box_max[0] = std::max(box_max[0], c.x);
    box_max[1] = std::max(box_max[1], c.y);
  }
  int Flat(XY c) const { return limits.nx * c.y + c.x; }
  // ProbabilityGrid::ApplyLookupTable (probability_grid.cc:58-71)
  bool ApplyLookupTable(XY c, const std::vector<uint16_t>& table) {
    const int flat = Flat(c);
    uint16_t* cell = &cells[flat];
    if (*cell >= kUpdateMarker) return false;
    update_indices.push_back(flat);
    *cell = table[*cell];
    Extend(c);
    return true;
  }
  // Grid2D::FinishUpdate (grid_2d.cc:99-106)
  void FinishUpdate() {
    while (!update_indices.empty()) {
      cells[update_indices.back()] -= kUpdateMarker;
      update_indices.pop_back();
    }
  }
  // Grid2D::GrowLimits (grid_2d.cc:130-164)
  void GrowLimits(float px, float py) {
    while (!limits.Contains(limits.GetCellIndex(px, py))) {
      const int x_offset = limits.nx / 2, y_offset = limits.ny / 2;
      Limits nl{limits.resolution, limits.max_x + limits.resolution * y_offset,
                limits.max_y + limits.resolution * x_offset, 2 * limits.nx, 2 * limits.ny};
      const int stride = nl.nx;
      const int offset = x_offset + stride * y_offset;
      std::vector<uint16_t> nc(static_cast<size_t>(nl.nx) * nl.ny, 0);
      for (int i = 0; i < limits.ny; ++i)
        for (int j = 0; j < limits.nx; ++j)
          nc[offset + j + i * stride] = cells[j + i * limits.nx];
      cells.swap(nc);
      limits = nl;
      if (!box_empty) {
        box_min[0] += x_offset;
        box_max[0] += x_offset;
        box_min[1] += y_offset;
        box_max[1] += y_offset;
      }
    }
  }
  float GetProbability(XY c) const {
    if (!limits.Contains(c)) return kMinProbability;
    return CorrespondenceCostToProbability(ValueToCorrespondenceCost(cells[Flat(c)]));
  }
  // ProbabilityGrid::SetProbability (probability_grid.cc:41-49); false where the reference
  // CHECK-fails (the cell was known)
  bool SetProbability(XY c, float p) {
    uint16_t& cell = cells[Flat(c)];
    if (cell != 0) return false;
    cell = CorrespondenceCostToValue(ProbabilityToCorrespondenceCost(p));
    Extend(c);
    return true;
  }
};

// RayToPixelMask (internal/2d/ray_to_pixel_mask.cc:34-156)
void RayToPixelMask(XY b, XY e, int s, std::vector<XY>* mask) {
  if (b.x > e.x) std::swap(b, e);
  mask->clear();
  auto push = [&](XY c) {
    if (mask->empty() || mask->back().x != c.x || mask->back().y != c.y) mask->push_back(c);
  };
  if (b.x / s == e.x / s) {
    XY cur{b.x / s, std::min(b.y, e.y) / s};
    mask->push_back(cur);
    const int end_y = std::max(b.y, e.y) / s;
    for (; cur.y <= end_y; ++cur.y) push(cur);
    return;
  }
  const int64_t dx = e.x - b.x;
  const int64_t dy = e.y - b.y;
  const int64_t denominator = 2 * s * dx;
  XY cur{b.x / s, b.y / s};
  mask->push_back(cur);
  int64_t sub_y = (2 * (b.y % s) + 1) * dx;
  const int first_pixel = 2 * s - 2 * (b.x % s) - 1;
  const int last_pixel = 2 * (e.x % s) + 1;
  const int end_x = std::max(b.x, e.x) / s;
  sub_y += dy * first_pixel;
  if (dy > 0) {
    while (true) {
      push(cur);
      while (sub_y > denominator) {
        sub_y -= denominator;
        ++cur.y;
        push(cur);
      }
      ++cur.x;
      if (sub_y == denominator) {
        sub_y -= denominator;
        ++cur.y;
      }
      if (cur.x == end_x) break;
      sub_y += dy * 2 * s;
    }
    sub_y += dy * last_pixel;
    push(cur);
    while (sub_y > denominator) {
      sub_y -= denominator;
      ++cur.y;
      push(cur);
    }
    return;
  }
  while (true) {
    push(cur);
    while (sub_y < 0) {
      sub_y += denominator;
      --cur.y;
      push(cur);
    }
    ++cur.x;
    if (sub_y == 0) {
      sub_y += denominator;
      --cur.y;
    }
    if (cur.x == end_x) break;
    sub_y += dy * 2 * s;
  }
  sub_y += dy * last_pixel;
  push(cur);
  while (sub_y < 0) {
    sub_y += denominator;
    --cur.y;
    push(cur);
  }
}

struct Inserter {
  std::vector<uint16_t> hit_table, miss_table;
  bool insert_free_space;
};

}  // namespace

extern "C" {

void* i2d_grid_new(double resolution, double max_x, double max_y, int nx, int ny,
                   const uint16_t* cells) {
  Grid* g = new Grid;
  g->limits = Limits{resolution, max_x, max_y, nx, ny};
  g->cells.assign(static_cast<size_t>(nx) * ny, 0);
  if (cells) {   // a grid made from cells: its known-cells box is that of its known cells
    for (int y = 0; y < ny; ++y)
      for (int x = 0; x < nx; ++x) {
        g->cells[static_cast<size_t>(y) * nx + x] = cells[static_cast<size_t>(y) * nx + x];
        if (cells[static_cast<size_t>(y) * nx + x] != 0) g->Extend(XY{x, y});
      }
  }
  return g;
}
void i2d_grid_free(void* g) { delete static_cast<Grid*>(g); }
// limits3 = {resolution, max_x, max_y}; ints = {nx, ny, box_empty, min_x, min_y, max_x, max_y}
void i2d_grid_info(const void* gp, double* limits3, int* ints) {
  const Grid* g = static_cast<const Grid*>(gp);
  limits3[0] = g->limits.resolution;
  limits3[1] = g->limits.max_x;
  limits3[2] = g->limits.max_y;
  ints[0] = g->limits.nx;
  ints[1] = g->limits.ny;
  ints[2] = g->box_empty ? 1 : 0;
  ints[3] = g->box_min[0];
  ints[4] = g->box_min[1];
  ints[5] = g->box_max[0];
  ints[6] = g->box_max[1];
}
void i2d_grid_cells(const void* gp, uint16_t* out) {
  const Grid* g = static_cast<const Grid*>(gp);
  std::memcpy(out, g->cells.data(), g->cells.size() * sizeof(uint16_t));
}
float i2d_grid_get_probability(const void* g, int x, int y) {
  return static_cast<const Grid*>(g)->GetProbability(XY{x, y});
}
int i2d_grid_set_probability(void* g, int x, int y, float p) {
  return static_cast<Grid*>(g)->SetProbability(XY{x, y}, p) ? 1 : 0;
}
int i2d_grid_apply_odds(void* g, int x, int y, float odds) {
  return static_cast<Grid*>(g)->ApplyLookupTable(
             XY{x, y}, ComputeLookupTableToApplyCorrespondenceCostOdds(odds)) ? 1 : 0;
}
void i2d_grid_finish_update(void* g) { static_cast<Grid*>(g)->FinishUpdate(); }
void i2d_grid_cell_index(const void* g, float px, float py, int* out) {
  const XY c = static_cast<const Grid*>(g)->limits.GetCellIndex(px, py);
  out[0] = c.x;
  out[1] = c.y;
}

// ProbabilityGrid::ComputeCroppedGrid (probability_grid.cc:91-107, grid_2d.cc:110-120)
void* i2d_grid_crop(const void* gp) {
  const Grid* g = static_cast<const Grid*>(gp);
  XY offset{0, 0};
  int nx = 1, ny = 1;
  if (!g->box_empty) {
    offset = XY{g->box_min[0], g->box_min[1]};
    nx = g->box_max[0] - g->box_min[0] + 1;
    ny = g->box_max[1] - g->box_min[1] + 1;
  }
  const double resolution = g->limits.resolution;
  Grid* c = static_cast<Grid*>(i2d_grid_new(resolution, g->limits.max_x - resolution * offset.y,
                                            g->limits.max_y - resolution * offset.x, nx, ny,
                                            nullptr));
  for (int y = 0; y < ny; ++y)
    for (int x = 0; x < nx; ++x) {
      const XY src{x + offset.x, y + offset.y};
      if (!(g->limits.Contains(src) && g->cells[g->Flat(src)] != 0)) continue;   // IsKnown
      c->SetProbability(XY{x, y}, g->GetProbability(src));
    }
  return c;
}

void* i2d_inserter_new(double hit_probability, double miss_probability, int insert_free_space) {
  Inserter* ins = new Inserter;
  ins->hit_table = ComputeLookupTableToApplyCorrespondenceCostOdds(
      Odds(static_cast<float>(hit_probability)));
  ins->miss_table = ComputeLookupTableToApplyCorrespondenceCostOdds(
      Odds(static_cast<float>(miss_probability)));
  ins->insert_free_space = insert_free_space != 0;
  return ins;
}
void i2d_inserter_free(void* ins) { delete static_cast<Inserter*>(ins); }
void i2d_inserter_tables(const void* ip, uint16_t* hit, uint16_t* miss) {
  const Inserter* ins = static_cast<const Inserter*>(ip);
  std::memcpy(hit, ins->hit_table.data(), kValueCount * sizeof(uint16_t));
  std::memcpy(miss, ins->miss_table.data(), kValueCount * sizeof(uint16_t));
}

// ProbabilityGridRangeDataInserter2D::Insert (probability_grid_range_data_inserter_2d.cc:35-133)
void i2d_insert(const void* ip, void* gp, const float* origin, const float* returns, int n,
                const float* misses, int m) {
  const Inserter* ins = static_cast<const Inserter*>(ip);
  Grid* g = static_cast<Grid*>(gp);
  // GrowAsNeeded
  float lo[2] = {origin[0], origin[1]}, hi[2] = {origin[0], origin[1]};
  auto extend = [&](const float* p) {
    for (int a = 0; a < 2; ++a) {
      lo[a] = std::min(lo[a], p[a]);
      hi[a] = std::max(hi[a], p[a]);
    }
  };
  for (int i = 0; i < n; ++i) extend(returns + 3 * i);
  for (int i = 0; i < m; ++i) extend(misses + 3 * i);
  constexpr float kPadding = 1e-6f;
  g->GrowLimits(lo[0] - kPadding, lo[1] - kPadding);
  g->GrowLimits(hi[0] + kPadding, hi[1] + kPadding);
  // CastRays
  const Limits& L = g->limits;
  const Limits S{L.resolution / kSubpixelScale, L.max_x, L.max_y, L.nx * kSubpixelScale,
                 L.ny * kSubpixelScale};
  const XY begin = S.GetCellIndex(origin[0], origin[1]);
  std::vector<XY> ends;
  ends.reserve(n);
  for (int i = 0; i < n; ++i) {
    ends.push_back(S.GetCellIndex(returns[3 * i], returns[3 * i + 1]));
    g->ApplyLookupTable(XY{ends.back().x / kSubpixelScale, ends.back().y / kSubpixelScale},
                        ins->hit_table);
  }
  if (ins->insert_free_space) {
    std::vector<XY> ray;
    for (const XY& end : ends) {
      RayToPixelMask(begin, end, kSubpixelScale, &ray);
      for (const XY& c : ray) g->ApplyLookupTable(c, ins->miss_table);
    }
    for (int i = 0; i < m; ++i) {
      RayToPixelMask(begin, S.GetCellIndex(misses[3 * i], misses[3 * i + 1]), kSubpixelScale, &ray);
      for (const XY& c : ray) g->ApplyLookupTable(c, ins->miss_table);
    }
  }
  g->FinishUpdate();
}

// RayToPixelMask into out (x, y pairs, capacity cap pixels); returns the pixel count.
int i2d_ray_to_pixel_mask(int bx, int by, int ex, int ey, int subpixel_scale, int* out, int cap) {
  std::vector<XY> mask;
  RayToPixelMask(XY{bx, by}, XY{ex, ey}, subpixel_scale, &mask);
  for (size_t i = 0; i < mask.size() && static_cast<int>(i) < cap; ++i) {
    out[2 * i] = mask[i].x;
    out[2 * i + 1] = mask[i].y;
  }
  return static_cast<int>(mask.size());
}

// The crop's SetProbability(GetProbability(v)) round trip for every value (0: unknown).
void i2d_crop_table(uint16_t* out) {
  out[0] = 0;
  for (int v = 1; v < kValueCount; ++v)
    out[v] = CorrespondenceCostToValue(ProbabilityToCorrespondenceCost(
        CorrespondenceCostToProbability(ValueToCorrespondenceCost(static_cast<uint16_t>(v)))));
}

}  // extern "C"
