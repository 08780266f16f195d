// The host side of drawing submap textures (submap_texture.cu): ProbabilityToLogOddsInteger as a
// step table, the gzip member of common::FastGzipString, the slice pose in Rigid3d arithmetic and
// the proto::SubmapQuery::Response::SubmapTexture framing.  Plain C++ (zlib and libm), so that the
// CPU test harness (tests/submap_texture_oracle.cc) includes it too; LogOddsIntegerFromSteps is
// the one lookup the device kernels and the harness both run.
#ifndef CSM_SUBMAP_TEXTURE_H_
#define CSM_SUBMAP_TEXTURE_H_

#include <zlib.h>

#include <cmath>
#include <cstdint>
#include <cstring>
#include <string>

#include "proto_write.h"
#include "value_conversion.h"

#ifdef __CUDACC__
#define CSM_TEX_HD __host__ __device__ __forceinline__
#else
#define CSM_TEX_HD inline
#endif

namespace csm {

// ---- ProbabilityToLogOddsInteger (mapping/submaps.h:37-53) ------------------------------------
// ProbabilityToLogOddsInteger(p) = RoundToInt((Logit(p) - kMinLogOdds) * 254.f /
// (kMaxLogOdds - kMinLogOdds)) + 1 with Logit(p) = std::log(p / (1.f - p)), on the host's logf.
// The device's logf is not glibc's, so the device never evaluates it: the function is a step
// function of p onto 1..255, and steps[k] is the smallest float p in [kMinProbability,
// kMaxProbability] whose value is at least k + 2 (found by bisection over the float bit patterns
// with the expression itself).  Both callers (the 2D ProbabilityGrid cells and the 3D pixels'
// clamped averages) pass p in [kMinProbability, kMaxProbability]; that every such float gives
// the direct value back through the table is checked exhaustively on the CPU.
constexpr int kLogOddsSteps = 254;
struct LogOddsSteps {
  float t[kLogOddsSteps];
};

inline int ProbabilityToLogOddsIntegerHost(float probability) {
  auto logit = [](float p) { return std::log(p / (1.f - p)); };
  const float max_log_odds = logit(kMaxProbability);
  const float min_log_odds = logit(kMinProbability);
  return static_cast<int>(
             std::lround((logit(probability) - min_log_odds) * 254.f / (max_log_odds - min_log_odds))) +
         1;
}

inline float FloatFromBits(uint32_t b) {
  float f;
  std::memcpy(&f, &b, 4);
  return f;
}
inline uint32_t BitsFromFloat(float f) {
  uint32_t b;
  std::memcpy(&b, &f, 4);
  return b;
}

inline LogOddsSteps MakeLogOddsSteps() {
  LogOddsSteps s;
  const uint32_t lo = BitsFromFloat(kMinProbability), hi = BitsFromFloat(kMaxProbability);
  for (int k = 0; k < kLogOddsSteps; ++k) {
    const int want = k + 2;
    // the first bit pattern in [lo, hi + 1) whose value reaches `want` (positive floats order
    // like their bit patterns); hi + 1 (a float above kMaxProbability) if none does
    uint32_t a = lo, b = hi + 1;
    while (a < b) {
      const uint32_t m = a + (b - a) / 2;
      if (ProbabilityToLogOddsIntegerHost(FloatFromBits(m)) >= want)
        b = m;
      else
        a = m + 1;
    }
    s.t[k] = FloatFromBits(a);
  }
  return s;
}

// 1 + the number of steps at or below p.
CSM_TEX_HD int LogOddsIntegerFromSteps(float p, const float* steps) {
  int a = 0, b = kLogOddsSteps;
  while (a < b) {
    const int m = (a + b) >> 1;
    if (steps[m] <= p)
      a = m + 1;
    else
      b = m;
  }
  return a + 1;
}

// ---- common::FastGzipString (common/port.h:48-57) ----------------------------------------------
// boost::iostreams::gzip_compressor(zlib::best_speed): the 10-byte header boost writes (no name,
// comment or extra field, mtime 0, XFL 4 for best_speed, OS 255 "unknown"), a raw deflate stream
// at level 1, window 15, memLevel 8, default strategy, and the CRC-32 and ISIZE trailer.  zlib's
// deflate output does not depend on how the input is split between calls without a flush, so one
// Z_FINISH call gives the stream boost's chunked writes give.  Appends to *out; false if zlib
// fails.
inline bool GzipMember(const uint8_t* data, size_t n, std::string* out) {
  static const uint8_t kHeader[10] = {0x1f, 0x8b, 8, 0, 0, 0, 0, 0, 4, 0xff};
  z_stream z;
  std::memset(&z, 0, sizeof(z));
  if (deflateInit2(&z, Z_BEST_SPEED, Z_DEFLATED, -MAX_WBITS, 8, Z_DEFAULT_STRATEGY) != Z_OK)
    return false;
  const size_t start = out->size();
  const uLong bound = deflateBound(&z, static_cast<uLong>(n));
  out->resize(start + sizeof(kHeader) + bound + 8);
  uint8_t* o = reinterpret_cast<uint8_t*>(&(*out)[start]);
  std::memcpy(o, kHeader, sizeof(kHeader));
  z.next_in = const_cast<Bytef*>(data);
  z.avail_in = static_cast<uInt>(n);
  z.next_out = o + sizeof(kHeader);
  z.avail_out = static_cast<uInt>(bound);
  const int r = deflate(&z, Z_FINISH);
  const size_t body = bound - z.avail_out;
  deflateEnd(&z);
  if (r != Z_STREAM_END) return false;
  const uint32_t crc = static_cast<uint32_t>(crc32(crc32(0L, Z_NULL, 0), data, static_cast<uInt>(n)));
  const uint32_t isize = static_cast<uint32_t>(n);
  uint8_t* t = o + sizeof(kHeader) + body;
  for (int i = 0; i < 4; ++i) t[i] = static_cast<uint8_t>(crc >> (8 * i));
  for (int i = 0; i < 4; ++i) t[4 + i] = static_cast<uint8_t>(isize >> (8 * i));
  out->resize(start + sizeof(kHeader) + body + 8);
  return true;
}

// ---- the slice pose: transform::Rigid3d arithmetic in double (transform/rigid_transform.h) ----
struct Vec3d { double x, y, z; };
struct Quat4d { double w, x, y, z; };
struct Pose3d { Vec3d t; Quat4d q; };

inline Vec3d CrossD(const Vec3d& a, const Vec3d& b) {
  return Vec3d{a.y * b.z - a.z * b.y, a.z * b.x - a.x * b.z, a.x * b.y - a.y * b.x};
}

// Eigen 3.3 QuaternionBase::_transformVector: uv = 2 (q.vec x v); v + q.w uv + q.vec x uv.
inline Vec3d RotateD(const Quat4d& q, const Vec3d& v) {
  const Vec3d qv{q.x, q.y, q.z};
  Vec3d uv = CrossD(qv, v);
  uv = Vec3d{uv.x + uv.x, uv.y + uv.y, uv.z + uv.z};
  const Vec3d c = CrossD(qv, uv);
  return Vec3d{(v.x + q.w * uv.x) + c.x, (v.y + q.w * uv.y) + c.y, (v.z + q.w * uv.z) + c.z};
}

// Eigen 3.3 quat_product<Architecture::SSE, ..., double> (Geometry_SSE.h, the SSE2 path): the
// pairs (x, y) and (z, w) each from two packed products.
inline Quat4d QuatMulD(const Quat4d& a, const Quat4d& b) {
  Quat4d r;
  r.x = (a.w * b.x + a.y * b.z) - (a.z * b.y - a.x * b.w);
  r.y = (a.w * b.y + a.y * b.w) + (a.z * b.x - a.x * b.z);
  r.z = (a.w * b.z - a.y * b.x) + (a.x * b.y + a.z * b.w);
  r.w = (a.w * b.w - a.y * b.y) - (a.x * b.x + a.z * b.z);
  return r;
}

// coeffs().normalized(): the Packet2d reduction (x² + z²) + (y² + w²), then q / sqrt.
inline Quat4d QuatNormalizedD(const Quat4d& q) {
  const double n2 = (q.x * q.x + q.z * q.z) + (q.y * q.y + q.w * q.w);
  if (!(n2 > 0.)) return q;
  const double n = std::sqrt(n2);
  return Quat4d{q.w / n, q.x / n, q.y / n, q.z / n};
}

// pose.inverse() * Rigid3d::Translation(v) (rigid_transform.h:148-152, 181-189).
inline Pose3d InverseTimesTranslation(const Pose3d& pose, const Vec3d& v) {
  const Quat4d rot{pose.q.w, -pose.q.x, -pose.q.y, -pose.q.z};
  const Vec3d rt = RotateD(rot, pose.t);
  const Vec3d inv_t{-rt.x, -rt.y, -rt.z};
  const Vec3d a = RotateD(rot, v);
  return Pose3d{Vec3d{a.x + inv_t.x, a.y + inv_t.y, a.z + inv_t.z},
                QuatNormalizedD(QuatMulD(rot, Quat4d{1., 0., 0., 0.}))};
}

// ---- proto::SubmapQuery::Response::SubmapTexture (submap_visualization.proto:47-62) -----------
// cells = 1 (bytes), width = 2, height = 3 (int32), resolution = 4 (double), slice_pose = 5
// (transform.proto Rigid3d: translation = 1 {x, y, z = 1..3}, rotation = 2 {x, y, z, w = 1..4});
// transform::ToProto always sets both sub-messages.  The proto_write.h rules apply.
struct TextureMessage {
  int64_t vec_len, quat_len, pose_len, total;
};

inline TextureMessage SizeTexture(size_t cells_len, int32_t width, int32_t height,
                                  double resolution, const Pose3d& slice) {
  using namespace wire;
  TextureMessage m;
  m.vec_len = DoubleFieldSize(slice.t.x) + DoubleFieldSize(slice.t.y) + DoubleFieldSize(slice.t.z);
  m.quat_len = DoubleFieldSize(slice.q.x) + DoubleFieldSize(slice.q.y) +
               DoubleFieldSize(slice.q.z) + DoubleFieldSize(slice.q.w);
  m.pose_len = DelimitedSize(m.vec_len) + DelimitedSize(m.quat_len);
  m.total = (cells_len ? DelimitedSize(static_cast<int64_t>(cells_len)) : 0) +
            Int32FieldSize(width) + Int32FieldSize(height) + DoubleFieldSize(resolution) +
            DelimitedSize(m.pose_len);
  return m;
}

inline void WriteTexture(uint8_t* p, const TextureMessage& m, const std::string& cells,
                         int32_t width, int32_t height, double resolution, const Pose3d& slice) {
  using namespace wire;
  if (!cells.empty()) {
    p = PutDelimitedHeader(p, 1, static_cast<int64_t>(cells.size()));
    std::memcpy(p, cells.data(), cells.size());
    p += cells.size();
  }
  p = PutInt32Field(p, 2, width);
  p = PutInt32Field(p, 3, height);
  p = PutDoubleField(p, 4, resolution);
  p = PutDelimitedHeader(p, 5, m.pose_len);
  p = PutDelimitedHeader(p, 1, m.vec_len);
  p = PutDoubleField(p, 1, slice.t.x);
  p = PutDoubleField(p, 2, slice.t.y);
  p = PutDoubleField(p, 3, slice.t.z);
  p = PutDelimitedHeader(p, 2, m.quat_len);
  p = PutDoubleField(p, 1, slice.q.x);
  p = PutDoubleField(p, 2, slice.q.y);
  p = PutDoubleField(p, 3, slice.q.z);
  PutDoubleField(p, 4, slice.q.w);
}

}  // namespace csm

#undef CSM_TEX_HD

#endif  // CSM_SUBMAP_TEXTURE_H_
