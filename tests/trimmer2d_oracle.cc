// CPU restatement of OverlappingSubmapsTrimmer2D's coverage pass
// (mapping/internal/2d/overlapping_submaps_trimmer_2d.cc:27-102, 145-182), restated from its
// structure for the tests and for the CPU column of benchmarks/bench_trimmer2d.py: a std::map of
// global cells to (submap, time) lists filled submap by submap and cell by cell, a per-cell
// std::sort by descending time with the reference's comparator, and a std::map<int, uint16_t>
// of covered cells per submap.  Compiled with -ffp-contract=off, as the reference is built.
#include <algorithm>
#include <cmath>
#include <cstdint>
#include <map>
#include <utility>
#include <vector>

namespace {

// Eigen's Quaternion * Vector3 (_transformVector) followed by + t.
void Transform(const double* t, const double* q, const double c[3], double p[3]) {
  const double w = q[0], v[3] = {q[1], q[2], q[3]};
  double uv[3] = {v[1] * c[2] - v[2] * c[1], v[2] * c[0] - v[0] * c[2], v[0] * c[1] - v[1] * c[0]};
  for (int k = 0; k < 3; ++k) uv[k] += uv[k];
  const double x[3] = {v[1] * uv[2] - v[2] * uv[1], v[2] * uv[0] - v[0] * uv[2],
                       v[0] * uv[1] - v[1] * uv[0]};
  for (int k = 0; k < 3; ++k) p[k] = c[k] + w * uv[k] + x[k] + t[k];
}

}  // namespace

extern "C" {

// n submaps: cells[i] (num_y x num_x[i], row-major), box[4 i ..] = cropped limits
// {offset x, offset y, num_x_cells, num_y_cells}, limits[3 i ..] = {max x, max y, resolution},
// poses[7 i ..] = global_frame_from_local_frame {tx, ty, tz, qw, qx, qy, qz}, freshness[i].
// Writes trim[i], counts[i] (covered entries before the uint16 wrap) and
// stats = {entries, coverage cells, cells whose cut was a std::sort of more than 16 entries}.
void tro_trim(int32_t n, const uint16_t* const* cells, const int32_t* num_x, const int32_t* box,
              const double* limits, const double* poses, const int64_t* freshness,
              double first_max_x, double first_max_y, double first_resolution,
              uint16_t fresh_submaps_count, uint16_t min_covered_cells_count, uint8_t* trim,
              uint32_t* counts, int64_t* stats) {
  using Entry = std::pair<int, int64_t>;
  std::map<std::pair<int64_t, int64_t>, std::vector<Entry>> coverage;
  int64_t entries = 0;
  for (int i = 0; i < n; ++i) {
    const int ox = box[4 * i], oy = box[4 * i + 1], w = box[4 * i + 2], h = box[4 * i + 3];
    const double max_x = limits[3 * i], max_y = limits[3 * i + 1], res = limits[3 * i + 2];
    for (int y = 0; y < h; ++y) {
      for (int x = 0; x < w; ++x) {
        const int ix = x + ox, iy = y + oy;
        if (cells[i][static_cast<size_t>(iy) * num_x[i] + ix] == 0) continue;   // !IsKnown
        const double c[3] = {max_x - res * (iy + 0.5), max_y - res * (ix + 0.5), 0.};
        double p[3];
        Transform(poses + 7 * i, poses + 7 * i + 3, c, p);
        const std::pair<int64_t, int64_t> key{std::lround((first_max_x - p[0]) / first_resolution),
                                              std::lround((first_max_y - p[1]) / first_resolution)};
        coverage[key].emplace_back(i, freshness[i]);
        ++entries;
      }
    }
  }
  std::map<int, uint16_t> covered;
  std::vector<uint32_t> total(n, 0u);
  int64_t sorted_large = 0;
  for (const auto& cell : coverage) {
    std::vector<Entry> kept(cell.second);
    if (kept.size() > fresh_submaps_count) {
      if (kept.size() > 16) ++sorted_large;
      std::sort(kept.begin(), kept.end(), [](const Entry& left, const Entry& right) {
        return left.second > right.second;
      });
      kept.erase(kept.begin() + fresh_submaps_count, kept.end());
    }
    for (const Entry& e : kept) {
      ++covered[e.first];
      ++total[e.first];
    }
  }
  for (int i = 0; i < n; ++i) {
    const auto it = covered.find(i);
    trim[i] = it == covered.end() || it->second < min_covered_cells_count;
    counts[i] = total[i];
  }
  stats[0] = entries;
  stats[1] = static_cast<int64_t>(coverage.size());
  stats[2] = sorted_large;
}

}  // extern "C"
