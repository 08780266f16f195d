// TEST INFRASTRUCTURE ONLY — never linked into libcsm_b200.so.
//
// A single-thread restatement of what Submap3D::InsertData (mapping/3d/submap_3d.cc:271-294)
// does to a scan before RangeDataInserter3D sees it, and of its histogram update:
//   * local_pose().inverse() in double (transform/rigid_transform.h:148-152, Eigen's
//     _transformVector), cast to float;
//   * TransformRangeData (sensor/range_data.cc:25-32) with rigid3f.h's Rigid3Apply;
//   * FilterRangeDataByMaxRange (submap_3d.cc:41-49): (p - origin).norm() <= max_range;
//   * GetCellIndex (hybrid_grid.h:428-433) with the 2^14 cube test;
//   * GetYaw(local_pose().inverse().rotation() * local_from_gravity_aligned) in double and
//     RotationalScanMatcher::RotateHistogram (rotational_scan_matcher.cc:141-162) in float.
// Built by the tests with -O2 -ffp-contract=off.
#include <cmath>
#include <vector>

#include "../cartographer_b200/csrc/rigid3f.h"

namespace {

struct Qd { double w, x, y, z; };

// Eigen 3.3 _transformVector in double: uv = q.vec x v; uv += uv; v + w uv + q.vec x uv.
void RotateD(const Qd& q, const double* v, double* out) {
  double uv[3] = {q.y * v[2] - q.z * v[1], q.z * v[0] - q.x * v[2], q.x * v[1] - q.y * v[0]};
  for (double& u : uv) u += u;
  const double c[3] = {q.y * uv[2] - q.z * uv[1], q.z * uv[0] - q.x * uv[2],
                       q.x * uv[1] - q.y * uv[0]};
  for (int a = 0; a < 3; ++a) out[a] = v[a] + q.w * uv[a] + c[a];
}

csm::Rigid3f InverseCast(const double* pose) {
  const Qd conj{pose[3], -pose[4], -pose[5], -pose[6]};
  double t[3];
  RotateD(conj, pose, t);
  return csm::Rigid3f{{static_cast<float>(-t[0]), static_cast<float>(-t[1]),
                       static_cast<float>(-t[2])},
                      {static_cast<float>(conj.w), static_cast<float>(conj.x),
                       static_cast<float>(conj.y), static_cast<float>(conj.z)}};
}

}  // namespace

extern "C" {

// inverse[7]: local_pose().inverse().cast<float>() as {t xyz, q wxyz}.
void submap_inverse(const double* pose, float* inverse) {
  const csm::Rigid3f r = InverseCast(pose);
  const float v[7] = {r.t.x, r.t.y, r.t.z, r.q.w, r.q.x, r.q.y, r.q.z};
  for (int k = 0; k < 7; ++k) inverse[k] = v[k];
}

// The origin and the n returns in the submap frame, and kept[i] = the range filter.
void submap_transform(const double* pose, const float* origin, const float* returns, int n,
                      float max_range, float* out_origin, float* out_returns,
                      unsigned char* kept) {
  const csm::Rigid3f inv = InverseCast(pose);
  const csm::Vec3f o = csm::Rigid3Apply(inv, csm::Vec3f{origin[0], origin[1], origin[2]});
  out_origin[0] = o.x;
  out_origin[1] = o.y;
  out_origin[2] = o.z;
  for (int i = 0; i < n; ++i) {
    const float* p = returns + 3 * i;
    const csm::Vec3f q = csm::Rigid3Apply(inv, csm::Vec3f{p[0], p[1], p[2]});
    out_returns[3 * i] = q.x;
    out_returns[3 * i + 1] = q.y;
    out_returns[3 * i + 2] = q.z;
    const float dx = q.x - o.x, dy = q.y - o.y, dz = q.z - o.z;
    kept[i] = std::sqrt((dx * dx + dy * dy) + dz * dz) <= max_range;
  }
}

// GetCellIndex of n points; ok[i] = 0 outside the 2^14 cube or for a non-finite point.
void submap_cells(const float* points, int n, float resolution, int* cells, unsigned char* ok) {
  for (int i = 0; i < n; ++i) {
    ok[i] = 1;
    for (int a = 0; a < 3; ++a) {
      const float q = points[3 * i + a] / resolution;
      if (!(q > -8192.5f && q < 8191.5f)) {
        ok[i] = 0;
        cells[3 * i + a] = 0;
        continue;
      }
      cells[3 * i + a] = static_cast<int>(std::lround(q));
    }
  }
}

float submap_yaw(const double* pose, const double* q) {
  const Qd p{pose[3], -pose[4], -pose[5], -pose[6]};
  const Qd r{p.w * q[0] - p.x * q[1] - p.y * q[2] - p.z * q[3],
             p.w * q[1] + p.x * q[0] + p.y * q[3] - p.z * q[2],
             p.w * q[2] + p.y * q[0] + p.z * q[1] - p.x * q[3],
             p.w * q[3] + p.z * q[0] + p.x * q[2] - p.y * q[1]};
  const double unit_x[3] = {1., 0., 0.};
  double d[3];
  RotateD(r, unit_x, d);
  return static_cast<float>(std::atan2(d[1], d[0]));
}

// histogram += RotateHistogram(scan, angle), size floats each.
void submap_accumulate_histogram(float* histogram, const float* scan, int size, float angle) {
  if (size == 0) return;
  const float rotate_by_buckets = -angle * size / M_PI;
  int full_buckets = static_cast<int>(std::lround(rotate_by_buckets - 0.5f));
  const float fraction = rotate_by_buckets - full_buckets;
  while (full_buckets < 0) full_buckets += size;
  for (int i = 0; i < size; ++i) {
    const float r0 = scan[(i + full_buckets) % size];
    const float r1 = scan[(i + 1 + full_buckets) % size];
    histogram[i] += fraction * r1 + (1.f - fraction) * r0;
  }
}

}  // extern "C"
