// CPU restatement of TSDFRangeDataInserter2D::Insert (mapping/internal/2d/
// tsdf_range_data_inserter_2d.cc), TSDF2D (tsdf_2d.cc, tsd_value_converter.{h,cc},
// value_conversion_tables.cc) and NormalEstimation2D (normal_estimation_2d.cc).  Sequential, in
// the reference's operation order: the parity reference of the device inserter
// (tests/test_gpu_insert_tsdf2d.py) and the CPU column of benchmarks/bench_insert_tsdf2d.py.
// Test infrastructure, loaded through tests/insert_tsdf2d_oracle.py; the product library never
// uses it.  It reuses the ProbabilityGrid restatement's MapLimits, Grid2D (cells, known-cells
// box, GrowLimits, FinishUpdate) and RayToPixelMask by including it.
// Build with -ffp-contract=off: float where the reference is float, double where it is double.
#include "insert2d_oracle.cc"

#include <limits>

namespace {

struct P3 { float x, y, z; };

// Eigen's norm() of float vectors: the squares summed in index order, one sqrt
float Norm2(float x, float y) { return std::sqrt(x * x + y * y); }
float Norm3(float x, float y, float z) { return std::sqrt(x * x + y * y + z * z); }

// TSDValueConverter with ValueConversionTables' value -> float map (value_conversion_tables.cc)
struct TSDValueConverter {
  float max_tsd, min_tsd, max_weight, tsd_resolution, weight_resolution;
  TSDValueConverter(float truncation, float maximum_weight)
      : max_tsd(truncation), min_tsd(-truncation), max_weight(maximum_weight),
        tsd_resolution(32766.f / (max_tsd - min_tsd)),
        weight_resolution(32766.f / (max_weight - 0.f)) {}
  static float ValueToBoundedFloat(uint16_t value, float unknown, float lo, float hi) {
    const uint16_t v = value & static_cast<uint16_t>(~kUpdateMarker);
    if (v == 0) return unknown;
    const float kScale = (hi - lo) / 32766.f;
    return v * kScale + (lo - kScale);
  }
  float ValueToTSD(uint16_t v) const { return ValueToBoundedFloat(v, min_tsd, min_tsd, max_tsd); }
  float ValueToWeight(uint16_t v) const { return ValueToBoundedFloat(v, 0.f, 0.f, max_weight); }
  uint16_t TSDToValue(float tsd) const {
    return static_cast<uint16_t>(
        static_cast<int>(std::lround((Clamp(tsd, min_tsd, max_tsd) - min_tsd) * tsd_resolution)) + 1);
  }
  uint16_t WeightToValue(float w) const {
    return static_cast<uint16_t>(
        static_cast<int>(std::lround((Clamp(w, 0.f, max_weight) - 0.f) * weight_resolution)) + 1);
  }
};

// TSDF2D: Grid's cells are its tsd cells (Grid2D's correspondence_cost_cells)
struct Tsdf : Grid {
  std::vector<uint16_t> weights;
  TSDValueConverter conv;
  Tsdf(float truncation, float max_weight) : conv(truncation, max_weight) {}
  // TSDF2D::GrowLimits: Grid2D::GrowLimits of the tsd cells and the box, and the same doublings
  // of the weight cells (unknown value 0 in both)
  void GrowLimits(float px, float py) {
    const Limits old = limits;
    Grid::GrowLimits(px, py);
    if (limits.nx == old.nx) return;
    int ox = 0, oy = 0;
    for (int nx = old.nx, ny = old.ny; nx < limits.nx; nx *= 2, ny *= 2) {
      ox += nx / 2;
      oy += ny / 2;
    }
    std::vector<uint16_t> nw(static_cast<size_t>(limits.nx) * limits.ny, 0);
    for (int i = 0; i < old.ny; ++i)
      for (int j = 0; j < old.nx; ++j)
        nw[(oy + i) * static_cast<size_t>(limits.nx) + ox + j] =
            weights[i * static_cast<size_t>(old.nx) + j];
    weights.swap(nw);
  }
  bool CellIsUpdated(XY c) const { return cells[Flat(c)] >= kUpdateMarker; }
  void SetCell(XY c, float tsd, float weight) {
    const int flat = Flat(c);
    if (cells[flat] >= kUpdateMarker) return;
    update_indices.push_back(flat);
    Extend(c);
    cells[flat] = conv.TSDToValue(tsd) + kUpdateMarker;
    weights[flat] = conv.WeightToValue(weight);
  }
  float GetTSD(XY c) const {
    return limits.Contains(c) ? conv.ValueToTSD(cells[Flat(c)]) : conv.min_tsd;
  }
  float GetWeight(XY c) const {
    return limits.Contains(c) ? conv.ValueToWeight(weights[Flat(c)]) : 0.f;
  }
};

struct TsdfOptions {
  float truncation_distance;   // static_cast<float> of the double options, as the reference uses them
  float maximum_weight;
  bool update_free_space;
  int num_normal_samples;
  float sample_radius;
  bool project;
  int range_exponent;
  double angle_bandwidth, distance_bandwidth;
};

const float kSqrtTwoPi = std::sqrt(2.0 * M_PI);

float GaussianKernel(const float x, const float sigma) {
  return 1.0 / (kSqrtTwoPi * sigma) * std::exp(-0.5 * x * x / (sigma * sigma));
}

template <typename T>
T NormalizeAngleDifference(T difference) {
  const T kPi = T(M_PI);
  while (difference > kPi) difference -= 2. * kPi;
  while (difference < -kPi) difference += 2. * kPi;
  return difference;
}

// RangeDataSorter: normalized() divides by the norm unless it is zero
struct RangeDataSorter {
  float ox, oy;
  bool operator()(const P3& lhs, const P3& rhs) const {
    float l[2] = {lhs.x - ox, lhs.y - oy}, r[2] = {rhs.x - ox, rhs.y - oy};
    for (float* v : {l, r}) {
      const float z = v[0] * v[0] + v[1] * v[1];
      if (z > 0.f) {
        const float n = std::sqrt(z);
        v[0] /= n;
        v[1] /= n;
      }
    }
    if ((l[1] < 0.f) != (r[1] < 0.f)) return l[1] < 0.f;
    if (l[1] < 0.f) return l[0] < r[0];
    return l[0] > r[0];
  }
};

float EstimateNormal(const std::vector<P3>& returns, size_t index, size_t begin, size_t end,
                     const P3& origin) {
  const P3& p = returns[index];
  if (end - begin < 2) return std::atan2(origin.y - p.y, origin.x - p.x);
  float mean[3] = {0.f, 0.f, 0.f};
  const float to_obs[3] = {origin.x - p.x, origin.y - p.y, origin.z - p.z};
  for (size_t k = begin; k < end; ++k) {
    if (k == index) continue;
    const float tangent[3] = {p.x - returns[k].x, p.y - returns[k].y, p.z - returns[k].z};
    float n[3] = {-tangent[1], tangent[0], 0.f};
    if (Norm3(n[0], n[1], n[2]) < 1e-6f) continue;
    if (n[0] * to_obs[0] + n[1] * to_obs[1] + n[2] * to_obs[2] < 0)
      for (float& v : n) v = -v;
    const float z = n[0] * n[0] + n[1] * n[1] + n[2] * n[2];   // normalize()
    if (z > 0.f) {
      const float s = std::sqrt(z);
      for (float& v : n) v /= s;
    }
    for (int a = 0; a < 3; ++a) mean[a] += n[a];
  }
  return std::atan2(mean[1], mean[0]);
}

std::vector<float> EstimateNormals(const std::vector<P3>& returns, const P3& origin,
                                   int num_normal_samples, float sample_radius) {
  std::vector<float> normals;
  const size_t max_num_samples = num_normal_samples;
  for (size_t cur = 0; cur < returns.size(); ++cur) {
    const P3& hit = returns[cur];
    auto dist = [&](size_t k) {
      return Norm3(hit.x - returns[k].x, hit.y - returns[k].y, hit.z - returns[k].z);
    };
    size_t begin = cur;
    for (; begin > 0 && cur - begin < max_num_samples / 2 && dist(begin - 1) < sample_radius;
         --begin) {
    }
    size_t end = cur;
    for (; end < returns.size() && end - cur < std::ceil(max_num_samples / 2.0) + 1 &&
           dist(end) < sample_radius;
         ++end) {
    }
    normals.push_back(EstimateNormal(returns, cur, begin, end, origin));
  }
  return normals;
}

struct HitRay {
  float hx, hy, normal, range;
  std::vector<XY> mask;
};

// TSDFRangeDataInserter2D::Insert + FinishUpdate.  false (and the grid unchanged) where the
// reference would index past its arrays (a mask pixel outside the grown grid) or where the grid
// would grow to 30000 cells per axis, or a mask cell still carries the update marker.
bool TsdfInsert(const TsdfOptions& opt, Tsdf* g, const P3& origin, std::vector<P3> returns) {
  const float truncation = opt.truncation_distance;
  // GrowAsNeeded, on a copy of the limits first
  float lo[2] = {origin.x, origin.y}, hi[2] = {origin.x, origin.y};
  for (const P3& p : returns) {
    float d[3] = {p.x - origin.x, p.y - origin.y, p.z - origin.z};
    const float z = d[0] * d[0] + d[1] * d[1] + d[2] * d[2];
    if (z > 0.f) {
      const float s = std::sqrt(z);
      for (float& v : d) v /= s;
    }
    const float e[2] = {p.x + truncation * d[0], p.y + truncation * d[1]};
    for (int a = 0; a < 2; ++a) {
      lo[a] = std::min(lo[a], e[a]);
      hi[a] = std::max(hi[a], e[a]);
    }
  }
  constexpr float kPadding = 1e-6f;
  const float corners[2][2] = {{lo[0] - kPadding, lo[1] - kPadding},
                               {hi[0] + kPadding, hi[1] + kPadding}};
  Limits L = g->limits;
  int ox = 0, oy = 0;
  for (const auto& c : corners)
    while (!L.Contains(L.GetCellIndex(c[0], c[1]))) {
      if (2 * L.nx >= 30000 || 2 * L.ny >= 30000) return false;
      ox += L.nx / 2;
      oy += L.ny / 2;
      L = Limits{L.resolution, L.max_x + L.resolution * (L.ny / 2),
                 L.max_y + L.resolution * (L.nx / 2), 2 * L.nx, 2 * L.ny};
    }
  // sort, normals
  std::vector<float> normals;
  const bool angle_weight = opt.angle_bandwidth != 0.f;
  if (opt.project || angle_weight) {
    std::sort(returns.begin(), returns.end(), RangeDataSorter{origin.x, origin.y});
    normals = EstimateNormals(returns, origin, opt.num_normal_samples, opt.sample_radius);
  }
  // every ray's mask against the grown limits, checked before anything changes
  const Limits S{L.resolution / kSubpixelScale, L.max_x, L.max_y, L.nx * kSubpixelScale,
                 L.ny * kSubpixelScale};
  // GetCellIndex; false where the pixel (C division) of the index lies outside the grid, which
  // RayToPixelMask then contains (and where the reference's int could overflow)
  auto superscaled = [&](float px, float py, XY* out) {
    const long ix = std::lround((S.max_y - py) / S.resolution - 0.5);
    const long iy = std::lround((S.max_x - px) / S.resolution - 0.5);
    if (ix <= -kSubpixelScale || iy <= -kSubpixelScale || ix >= S.nx || iy >= S.ny) return false;
    *out = XY{static_cast<int>(ix), static_cast<int>(iy)};
    return true;
  };
  std::vector<HitRay> rays;
  for (size_t k = 0; k < returns.size(); ++k) {
    HitRay h;
    h.hx = returns[k].x;
    h.hy = returns[k].y;
    h.normal = normals.empty() ? std::numeric_limits<float>::quiet_NaN() : normals[k];
    const float ray[2] = {h.hx - origin.x, h.hy - origin.y};
    h.range = Norm2(ray[0], ray[1]);
    if (h.range < truncation) continue;
    const float ratio = truncation / h.range;
    const float b[2] = {opt.update_free_space ? origin.x : origin.x + (1.0f - ratio) * ray[0],
                        opt.update_free_space ? origin.y : origin.y + (1.0f - ratio) * ray[1]};
    const float e[2] = {origin.x + (1.0f + ratio) * ray[0], origin.y + (1.0f + ratio) * ray[1]};
    XY sb, se;
    if (!superscaled(b[0], b[1], &sb) || !superscaled(e[0], e[1], &se)) return false;
    RayToPixelMask(sb, se, kSubpixelScale, &h.mask);
    for (const XY& c : h.mask) {
      if (!L.Contains(c)) return false;
      const XY old{c.x - ox, c.y - oy};
      if (g->limits.Contains(old) && g->cells[g->Flat(old)] >= kUpdateMarker) return false;
    }
    rays.push_back(std::move(h));
  }
  g->GrowLimits(corners[0][0], corners[0][1]);
  g->GrowLimits(corners[1][0], corners[1][1]);
  // InsertHit for every ray in order
  for (const HitRay& h : rays) {
    const float ray[2] = {h.hx - origin.x, h.hy - origin.y};
    float w_angle = 1.f;
    if (angle_weight) {
      const float angle = NormalizeAngleDifference(h.normal - std::atan2(-ray[1], -ray[0]));
      w_angle = GaussianKernel(angle, opt.angle_bandwidth);
    }
    float w_range = 1.f;
    if (opt.range_exponent != 0) {
      w_range = 0.f;
      if (std::abs(h.range) > 1e-6f) w_range = 1.f / (std::pow(h.range, opt.range_exponent));
    }
    for (const XY& c : h.mask) {
      if (g->CellIsUpdated(c)) continue;
      // MapLimits::GetCellCenter
      const float cx = g->limits.max_x - g->limits.resolution * (c.y + 0.5);
      const float cy = g->limits.max_y - g->limits.resolution * (c.x + 0.5);
      float update_tsd = h.range - Norm2(cx - origin.x, cy - origin.y);
      if (opt.project)
        update_tsd = (cx - h.hx) * std::cos(h.normal) + (cy - h.hy) * std::sin(h.normal);
      update_tsd = Clamp(update_tsd, -truncation, truncation);
      float update_weight = w_range * w_angle;
      if (opt.distance_bandwidth != 0.f)
        update_weight *= GaussianKernel(update_tsd, opt.distance_bandwidth);
      // UpdateCell
      if (update_weight == 0.f) continue;
      const float tsd = g->GetTSD(c), weight = g->GetWeight(c);
      float updated_weight = weight + update_weight;
      const float updated_sdf = (tsd * weight + update_tsd * update_weight) / updated_weight;
      updated_weight = std::min(updated_weight, opt.maximum_weight);
      g->SetCell(c, updated_sdf, updated_weight);
    }
  }
  g->FinishUpdate();
  return true;
}

}  // namespace

extern "C" {

// A TSDF2D of the given limits and converter; tsd / weight cells may be NULL (all unknown).  A grid
// made from cells takes the box of its non-zero tsd cells as its known-cells box.
void* i2t_grid_new(double resolution, double max_x, double max_y, int nx, int ny,
                   float truncation, float max_weight, const uint16_t* tsd, const uint16_t* weight) {
  Tsdf* g = new Tsdf(truncation, max_weight);
  g->limits = Limits{resolution, max_x, max_y, nx, ny};
  const size_t n = static_cast<size_t>(nx) * ny;
  g->cells.assign(n, 0);
  g->weights.assign(n, 0);
  for (int y = 0; tsd && y < ny; ++y)
    for (int x = 0; x < nx; ++x) {
      const size_t i = static_cast<size_t>(y) * nx + x;
      g->cells[i] = tsd[i];
      if (weight) g->weights[i] = weight[i];
      if (tsd[i] != 0) g->Extend(XY{x, y});
    }
  return g;
}
void i2t_grid_free(void* g) { delete static_cast<Tsdf*>(g); }
// as i2d_grid_info
void i2t_grid_info(const void* gp, double* limits3, int* ints) {
  i2d_grid_info(static_cast<const Grid*>(static_cast<const Tsdf*>(gp)), limits3, ints);
}
void i2t_grid_cells(const void* gp, uint16_t* tsd, uint16_t* weight) {
  const Tsdf* g = static_cast<const Tsdf*>(gp);
  std::memcpy(tsd, g->cells.data(), g->cells.size() * sizeof(uint16_t));
  std::memcpy(weight, g->weights.data(), g->weights.size() * sizeof(uint16_t));
}
// out = {is_known, GetTSD, GetWeight} of cell (x, y)
void i2t_grid_get(const void* gp, int x, int y, float* out) {
  const Tsdf* g = static_cast<const Tsdf*>(gp);
  const XY c{x, y};
  out[0] = g->limits.Contains(c) && g->cells[g->Flat(c)] != 0 ? 1.f : 0.f;   // Grid2D::IsKnown
  out[1] = g->GetTSD(c);
  out[2] = g->GetWeight(c);
}
void i2t_grid_cell_index(const void* g, float px, float py, int* out) {
  const XY c = static_cast<const Tsdf*>(g)->limits.GetCellIndex(px, py);
  out[0] = c.x;
  out[1] = c.y;
}

// options: the double fields of csm_tsdf_inserter_options2d in declaration order
// {truncation_distance, maximum_weight, update_free_space, num_normal_samples, sample_radius,
//  project_sdf_distance_to_scan_normal, update_weight_range_exponent, angle bandwidth,
//  distance bandwidth}
void* i2t_inserter_new(const double* o) {
  TsdfOptions* opt = new TsdfOptions;
  opt->truncation_distance = static_cast<float>(o[0]);
  opt->maximum_weight = static_cast<float>(o[1]);
  opt->update_free_space = o[2] != 0.;
  opt->num_normal_samples = static_cast<int>(o[3]);
  opt->sample_radius = static_cast<float>(o[4]);
  opt->project = o[5] != 0.;
  opt->range_exponent = static_cast<int>(o[6]);
  opt->angle_bandwidth = o[7];
  opt->distance_bandwidth = o[8];
  return opt;
}
void i2t_inserter_free(void* o) { delete static_cast<TsdfOptions*>(o); }
// 1 if inserted, 0 if refused (grid unchanged)
int i2t_insert(const void* op, void* gp, const float* origin, const float* returns, int n) {
  std::vector<P3> r(n);
  for (int i = 0; i < n; ++i) r[i] = P3{returns[3 * i], returns[3 * i + 1], returns[3 * i + 2]};
  return TsdfInsert(*static_cast<const TsdfOptions*>(op), static_cast<Tsdf*>(gp),
                    P3{origin[0], origin[1], origin[2]}, std::move(r)) ? 1 : 0;
}
// EstimateNormals of n returns (in the given order) into out
void i2t_estimate_normals(const float* returns, int n, const float* origin, int num_normal_samples,
                          float sample_radius, float* out) {
  std::vector<P3> r(n);
  for (int i = 0; i < n; ++i) r[i] = P3{returns[3 * i], returns[3 * i + 1], returns[3 * i + 2]};
  const std::vector<float> normals =
      EstimateNormals(r, P3{origin[0], origin[1], origin[2]}, num_normal_samples, sample_radius);
  std::memcpy(out, normals.data(), sizeof(float) * normals.size());
}

}  // extern "C"
