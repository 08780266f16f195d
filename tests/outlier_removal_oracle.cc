// CPU restatement of io::OutlierRemovingPointsProcessor's three phases
// (io/outlier_removing_points_processor.cc:53-129), written from their semantics: the parity
// reference of the device processor (cartographer_b200/csrc/outlier3d.cu) and the host column
// of benchmarks/bench_outlier_removal.py.  One thread, a std::map of voxels, every float step as
// the reference writes it; build with -ffp-contract=off.  Loaded by
// tests/outlier_removal_oracle.py.
#include <array>
#include <cmath>
#include <cstdint>
#include <map>
#include <vector>

namespace {

struct VoxelData {
  int hits = 0;
  int rays = 0;
};

struct Processor {
  double voxel_size;
  double miss_per_hit_limit;
  float resolution;                                  // HybridGridBase(float resolution)
  std::map<std::array<int, 3>, VoxelData> voxels;
};

// common::RoundToInt: std::lround narrowed to int.
int RoundToInt(float v) { return static_cast<int>(std::lround(v)); }

// HybridGridBase::GetCellIndex.
std::array<int, 3> CellIndex(const Processor& p, float x, float y, float z) {
  return {RoundToInt(x / p.resolution), RoundToInt(y / p.resolution),
          RoundToInt(z / p.resolution)};
}

// value(): a voxel that was never hit reads {0, 0}.
VoxelData Value(const Processor& p, const std::array<int, 3>& index) {
  const auto it = p.voxels.find(index);
  return it == p.voxels.end() ? VoxelData() : it->second;
}

bool InGrowableCube(const std::array<int, 3>& index) {
  for (int v : index)
    if (v < -8192 || v >= 8192) return false;
  return true;
}

float Length(const float* point, const float* origin, float* delta) {
  for (int a = 0; a < 3; ++a) delta[a] = point[a] - origin[a];
  return std::sqrt((delta[0] * delta[0] + delta[1] * delta[1]) + delta[2] * delta[2]);
}

}  // namespace

extern "C" {

void* oro_create(double voxel_size, double miss_per_hit_limit) {
  return new Processor{voxel_size, miss_per_hit_limit, static_cast<float>(voxel_size), {}};
}

void oro_destroy(void* h) { delete static_cast<Processor*>(h); }

// ProcessInPhaseOne.  Returns -1, changing nothing, when a hit lies outside the voxels the
// reference's grid can grow to (its CHECK would abort); else 0.
int oro_add_hits(void* h, const float* xyz, int n) {
  Processor& p = *static_cast<Processor*>(h);
  for (int i = 0; i < n; ++i)
    if (!InGrowableCube(CellIndex(p, xyz[3 * i], xyz[3 * i + 1], xyz[3 * i + 2]))) return -1;
  for (int i = 0; i < n; ++i) ++p.voxels[CellIndex(p, xyz[3 * i], xyz[3 * i + 1], xyz[3 * i + 2])].hits;
  return 0;
}

// The x the loop `for (float x = 0; x < length; x += voxel_size)` visits, into out (capacity
// cap); returns their number, or -1 when x stops growing below length (an endless loop).
long long oro_ray_samples(double voxel_size, float length, float* out, long long cap) {
  long long k = 0;
  for (float x = 0; x < length; x += voxel_size) {
    if (k < cap) out[k] = x;
    ++k;
    const float before = x;
    if (static_cast<float>(x + voxel_size) == before) return -1;
  }
  return k;
}

// ProcessInPhaseTwo for one batch.  Returns -1, changing nothing, when a ray would never end;
// else the number of samples taken.
long long oro_count_rays(void* h, const float* origin, const float* xyz, int n) {
  Processor& p = *static_cast<Processor*>(h);
  float delta[3];
  float max_length = 0.f;
  for (int i = 0; i < n; ++i) max_length = std::fmax(max_length, Length(xyz + 3 * i, origin, delta));
  if (oro_ray_samples(p.voxel_size, max_length, nullptr, 0) < 0) return -1;
  long long samples = 0;
  for (int i = 0; i < n; ++i) {
    const float length = Length(xyz + 3 * i, origin, delta);
    for (float x = 0; x < length; x += p.voxel_size) {
      const float s = x / length;
      const std::array<int, 3> index =
          CellIndex(p, origin[0] + s * delta[0], origin[1] + s * delta[1], origin[2] + s * delta[2]);
      if (Value(p, index).hits > 0) ++p.voxels[index].rays;
      ++samples;
    }
  }
  return samples;
}

// ProcessInPhaseThree for one batch: the kept indices in input order; returns their number.
int oro_filter(void* h, const float* xyz, int n, int* kept) {
  const Processor& p = *static_cast<Processor*>(h);
  int num_kept = 0;
  for (int i = 0; i < n; ++i) {
    const VoxelData voxel = Value(p, CellIndex(p, xyz[3 * i], xyz[3 * i + 1], xyz[3 * i + 2]));
    if (voxel.rays < p.miss_per_hit_limit * voxel.hits) kept[num_kept++] = i;
  }
  return num_kept;
}

// Every voxel in the map's (x, y, z) order; with indices == NULL only the count.
long long oro_voxels(void* h, int* indices, int* hits, int* rays) {
  const Processor& p = *static_cast<Processor*>(h);
  if (indices) {
    long long j = 0;
    for (const auto& v : p.voxels) {
      for (int a = 0; a < 3; ++a) indices[3 * j + a] = v.first[a];
      hits[j] = v.second.hits;
      rays[j] = v.second.rays;
      ++j;
    }
  }
  return static_cast<long long>(p.voxels.size());
}

// GetCellIndex of one point at `resolution`.
void oro_cell_index(float x, float y, float z, float resolution, int* out) {
  out[0] = RoundToInt(x / resolution);
  out[1] = RoundToInt(y / resolution);
  out[2] = RoundToInt(z / resolution);
}

}  // extern "C"
