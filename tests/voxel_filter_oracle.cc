// CPU restatement of sensor::VoxelFilter and sensor::AdaptiveVoxelFilter
// (sensor/internal/voxel_filter.cc), written from their semantics: the parity reference of the
// device filter (cartographer_b200/csrc/voxel_filter.cu) and the host column of
// benchmarks/bench_voxel_filter.py.  The generator is wrapped in an engine that counts the raw
// draws and the draws the distribution rejects.  Loaded by tests/voxel_filter_oracle.py.
#include <cmath>
#include <cstdint>
#include <random>
#include <unordered_map>
#include <vector>

namespace {

// std::minstd_rand0 with counters.  The distribution asks for min() / max() and draws through
// operator(); a draw is rejected when the next operator() comes within the same call.
struct CountingEngine {
  using result_type = std::minstd_rand0::result_type;
  static constexpr result_type min() { return std::minstd_rand0::min(); }
  static constexpr result_type max() { return std::minstd_rand0::max(); }
  std::minstd_rand0 engine;
  long long draws = 0;
  result_type operator()() {
    ++draws;
    return engine();
  }
};

// Replays a fixed sequence of raw outputs (for the distribution check).
struct ReplayEngine {
  using result_type = std::minstd_rand0::result_type;
  static constexpr result_type min() { return std::minstd_rand0::min(); }
  static constexpr result_type max() { return std::minstd_rand0::max(); }
  const uint32_t* raw;
  int at = 0;
  result_type operator()() { return raw[at++]; }
};

uint64_t Key(const float* p, float resolution) {
  const float ix = p[0] / resolution, iy = p[1] / resolution, iz = p[2] / resolution;
  const uint64_t x = static_cast<int>(std::lround(ix));
  const uint64_t y = static_cast<int>(std::lround(iy));
  const uint64_t z = static_cast<int>(std::lround(iz));
  return (x << 42) + (y << 21) + z;
}

// The kept flags of VoxelFilter(points, resolution); calls / draws count the distribution
// calls and the raw draws.
std::vector<bool> Filter(const std::vector<const float*>& pts, float resolution,
                         long long* calls, long long* draws) {
  CountingEngine generator;
  std::unordered_map<uint64_t, std::pair<int, int>> voxels;
  long long n_calls = 0;
  for (size_t i = 0; i < pts.size(); ++i) {
    auto& voxel = voxels[Key(pts[i], resolution)];
    voxel.first++;
    if (voxel.first == 1) {
      voxel.second = static_cast<int>(i);
    } else {
      ++n_calls;
      std::uniform_int_distribution<> distribution(1, voxel.first);
      if (distribution(generator) == voxel.first) voxel.second = static_cast<int>(i);
    }
  }
  std::vector<bool> used(pts.size(), false);
  for (const auto& v : voxels) used[v.second.second] = true;
  if (calls) *calls += n_calls;
  if (draws) *draws += generator.draws;
  return used;
}

std::vector<int> Kept(const std::vector<bool>& used, const std::vector<int>& index) {
  std::vector<int> out;
  for (size_t i = 0; i < used.size(); ++i)
    if (used[i]) out.push_back(index[i]);
  return out;
}

}  // namespace

extern "C" {

uint64_t vfo_key(float x, float y, float z, float resolution) {
  const float p[3] = {x, y, z};
  return Key(p, resolution);
}

// The first `count` outputs of a default-seeded std::minstd_rand0.
void vfo_generator(int count, uint32_t* out) {
  std::minstd_rand0 g;
  for (int i = 0; i < count; ++i) out[i] = static_cast<uint32_t>(g());
}

// uniform_int_distribution<int>(1, k) fed the raw outputs raw[0 ..]; *used is how many it took.
int vfo_uniform(int k, const uint32_t* raw, int* used) {
  ReplayEngine e{raw};
  std::uniform_int_distribution<> d(1, k);
  const int r = d(e);
  *used = e.at;
  return r;
}

// VoxelFilter: kept input indices in input order; returns their count.  calls / draws (may be
// null) get the distribution calls and raw draws, so draws - calls are the rejections.
int vfo_voxel_filter(const float* xyz, int n, float resolution, int* kept, long long* calls,
                     long long* draws) {
  std::vector<const float*> pts(n);
  std::vector<int> index(n);
  for (int i = 0; i < n; ++i) {
    pts[i] = xyz + 3 * i;
    index[i] = i;
  }
  const std::vector<int> out = Kept(Filter(pts, resolution, calls, draws), index);
  for (size_t i = 0; i < out.size(); ++i) kept[i] = out[i];
  return static_cast<int>(out.size());
}

// AdaptiveVoxelFilter: kept input indices (into the unfiltered cloud); returns their count.
// *final_length gets the length of the returned VoxelFilter (0 when the range-filtered cloud
// is returned), *trials the number of VoxelFilter calls.
int vfo_adaptive_voxel_filter(const float* xyz, int n, float max_length, float min_num_points,
                              float max_range, int* kept, float* final_length, int* trials) {
  std::vector<const float*> pts;
  std::vector<int> index;
  for (int i = 0; i < n; ++i) {
    const float* p = xyz + 3 * i;
    const float norm = std::sqrt((p[0] * p[0] + p[1] * p[1]) + p[2] * p[2]);
    if (norm <= max_range) {
      pts.push_back(p);
      index.push_back(i);
    }
  }
  int n_trials = 0;
  auto filter = [&](float length) {
    ++n_trials;
    return Kept(Filter(pts, length, nullptr, nullptr), index);
  };
  auto finish = [&](const std::vector<int>& out, float length) {
    for (size_t i = 0; i < out.size(); ++i) kept[i] = out[i];
    *final_length = length;
    *trials = n_trials;
    return static_cast<int>(out.size());
  };
  if (static_cast<float>(pts.size()) <= min_num_points) return finish(index, 0.f);
  std::vector<int> result = filter(max_length);
  if (static_cast<float>(result.size()) >= min_num_points) return finish(result, max_length);
  float low_length = 0.f;
  for (float high_length = max_length; high_length > 1e-2f * max_length; high_length /= 2.f) {
    low_length = high_length / 2.f;
    result = filter(low_length);
    if (static_cast<float>(result.size()) >= min_num_points) {
      while ((high_length - low_length) / low_length > 1e-1f) {
        const float mid_length = (low_length + high_length) / 2.f;
        std::vector<int> candidate = filter(mid_length);
        if (static_cast<float>(candidate.size()) >= min_num_points) {
          low_length = mid_length;
          result = std::move(candidate);
        } else {
          high_length = mid_length;
        }
      }
      return finish(result, low_length);
    }
  }
  return finish(result, low_length);
}

}  // extern "C"
