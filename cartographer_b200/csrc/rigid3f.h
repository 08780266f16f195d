// Eigen's float quaternion and rigid-transform arithmetic (Quaternionf, transform::Rigid3f) as
// the reference evaluates it, for the host and the device alike.  The names are those of the
// oracle's restatement (oracle/oracle_common.h, oracle/oracle_3d.h).  Plain C++ without nvcc,
// so that g++ harnesses include it too.  Under nvcc every function is __host__ __device__ and
// the elementary float operations are round-to-nearest intrinsics on the device, which ptxas
// never contracts into an FMA; the host is built with -ffp-contract=off.
#ifndef CSM_RIGID3F_H_
#define CSM_RIGID3F_H_

#include <cmath>

#ifdef __CUDACC__
#define CSM_HD __host__ __device__ __forceinline__
#else
#define CSM_HD inline
#endif

namespace csm {

#ifdef __CUDA_ARCH__
CSM_HD float FAdd(float a, float b) { return __fadd_rn(a, b); }
CSM_HD float FSub(float a, float b) { return __fsub_rn(a, b); }
CSM_HD float FMul(float a, float b) { return __fmul_rn(a, b); }
CSM_HD float FDiv(float a, float b) { return __fdiv_rn(a, b); }
CSM_HD float FSqrt(float a) { return __fsqrt_rn(a); }
#else
CSM_HD float FAdd(float a, float b) { return a + b; }
CSM_HD float FSub(float a, float b) { return a - b; }
CSM_HD float FMul(float a, float b) { return a * b; }
CSM_HD float FDiv(float a, float b) { return a / b; }
CSM_HD float FSqrt(float a) { return std::sqrt(a); }
#endif

struct Vec3f { float x, y, z; };
struct Quatf { float w, x, y, z; };
struct Quatd { double w, x, y, z; };
struct Rigid3f { Vec3f t; Quatf q; };

// Eigen 3.3 MatrixBase::cross for 3-vectors (scalar path).
CSM_HD Vec3f Cross(const Vec3f& a, const Vec3f& b) {
  return Vec3f{FSub(FMul(a.y, b.z), FMul(a.z, b.y)), FSub(FMul(a.z, b.x), FMul(a.x, b.z)),
               FSub(FMul(a.x, b.y), FMul(a.y, b.x))};
}

// Eigen 3.3 QuaternionBase::_transformVector:
//   uv = q.vec x v; uv += uv; return v + q.w * uv + q.vec x uv.
// The two cross products, uv and q.vec x uv:
struct RotationTerms { Vec3f uv, c; };
CSM_HD RotationTerms MakeRotationTerms(const Quatf& q, const Vec3f& v) {
  const Vec3f qv{q.x, q.y, q.z};
  Vec3f uv = Cross(qv, v);
  uv = Vec3f{FAdd(uv.x, uv.x), FAdd(uv.y, uv.y), FAdd(uv.z, uv.z)};
  return RotationTerms{uv, Cross(qv, uv)};
}

CSM_HD Vec3f Rotate(const Quatf& q, const Vec3f& v) {
  const RotationTerms r = MakeRotationTerms(q, v);
  return Vec3f{FAdd(FAdd(v.x, FMul(q.w, r.uv.x)), r.c.x),
               FAdd(FAdd(v.y, FMul(q.w, r.uv.y)), r.c.y),
               FAdd(FAdd(v.z, FMul(q.w, r.uv.z)), r.c.z)};
}

// transform/rigid_transform.h:192-196 with translation == Zero (Rigid3f::Rotation), applied per
// point by sensor/point_cloud.cc:56-64.
CSM_HD Vec3f RotateAsRigid3f(const Quatf& q, const Vec3f& v) {
  const Vec3f r = Rotate(q, v);
  return Vec3f{FAdd(r.x, 0.f), FAdd(r.y, 0.f), FAdd(r.z, 0.f)};
}

// Rigid3f * point (transform/rigid_transform.h:192-196): Rotate, then + translation.  Each
// component is one expression rather than Rotate(q, p) + t: the values are the same, and this
// is the instruction order the 3D matcher's kernels were measured with.
CSM_HD Vec3f Rigid3Apply(const Rigid3f& r, const Vec3f& p) {
  const RotationTerms e = MakeRotationTerms(r.q, p);
  return Vec3f{FAdd(FAdd(FAdd(p.x, FMul(r.q.w, e.uv.x)), e.c.x), r.t.x),
               FAdd(FAdd(FAdd(p.y, FMul(r.q.w, e.uv.y)), e.c.y), r.t.y),
               FAdd(FAdd(FAdd(p.z, FMul(r.q.w, e.uv.z)), e.c.z), r.t.z)};
}

// Quaternionf(AngleAxisf(angle, UnitZ)) from c = cos(angle / 2), s = sin(angle / 2):
// w = c, vec = s * (0, 0, 1).
CSM_HD Quatf QuatFromCosSinZ(float c, float s) {
  return Quatf{c, FMul(s, 0.f), FMul(s, 0.f), FMul(s, 1.f)};
}

// Eigen 3.3 Geometry/arch/Geometry_SSE.h quat_product<SSE, float>.
CSM_HD Quatf QuatMul(const Quatf& a, const Quatf& b) {
  Quatf r;
  r.x = FAdd(FSub(FMul(a.x, b.w), FMul(a.z, b.y)), FAdd(FMul(a.y, b.z), FMul(a.w, b.x)));
  r.y = FAdd(FSub(FMul(a.y, b.w), FMul(a.x, b.z)), FAdd(FMul(a.z, b.x), FMul(a.w, b.y)));
  r.z = FAdd(FSub(FMul(a.z, b.w), FMul(a.y, b.x)), FAdd(FMul(a.x, b.y), FMul(a.w, b.z)));
  r.w = FAdd(FSub(FMul(a.w, b.w), FMul(a.x, b.x)), -FAdd(FMul(a.z, b.z), FMul(a.y, b.y)));
  return r;
}

// coeffs().squaredNorm() in the Packet4f reduction order (x² + z²) + (y² + w²).
CSM_HD float QuatSquaredNorm(const Quatf& q) {
  return FAdd(FAdd(FMul(q.x, q.x), FMul(q.z, q.z)), FAdd(FMul(q.y, q.y), FMul(q.w, q.w)));
}

// q / sqrt(squaredNorm) if that is > 0, else q unchanged.
CSM_HD Quatf QuatNormalized(const Quatf& q) {
  const float z = QuatSquaredNorm(q);
  if (z > 0.f) {
    const float n = FSqrt(z);
    return Quatf{FDiv(q.w, n), FDiv(q.x, n), FDiv(q.y, n), FDiv(q.z, n)};
  }
  return q;
}

CSM_HD Quatf QuatConjugate(const Quatf& q) { return Quatf{q.w, -q.x, -q.y, -q.z}; }

// conjugate / squaredNorm, the zero quaternion if that is not > 0.
CSM_HD Quatf QuatInverse(const Quatf& q) {
  const float n2 = QuatSquaredNorm(q);
  if (n2 > 0.f) return Quatf{FDiv(q.w, n2), FDiv(-q.x, n2), FDiv(-q.y, n2), FDiv(-q.z, n2)};
  return Quatf{0.f, 0.f, 0.f, 0.f};
}

// transform/rigid_transform.h:148-152
CSM_HD Rigid3f Rigid3Inverse(const Rigid3f& r) {
  const Quatf rot = QuatConjugate(r.q);
  const Vec3f v = Rotate(rot, r.t);
  return Rigid3f{Vec3f{-v.x, -v.y, -v.z}, rot};
}

// transform/rigid_transform.h:181-189
CSM_HD Rigid3f Rigid3Mul(const Rigid3f& a, const Rigid3f& b) {
  return Rigid3f{Rigid3Apply(a, b.t), QuatNormalized(QuatMul(a.q, b.q))};
}

// The rest is host only: double arithmetic, which the device could contract, and libm.

// q.inverse().cast<float>() of a double quaternion.
inline Quatf QuatCastInverseD(const Quatd& q) {
  const double n2 = (q.x * q.x + q.z * q.z) + (q.y * q.y + q.w * q.w);
  Quatd inv{0., 0., 0., 0.};
  if (n2 > 0.) inv = Quatd{q.w / n2, -q.x / n2, -q.y / n2, -q.z / n2};
  return Quatf{static_cast<float>(inv.w), static_cast<float>(inv.x), static_cast<float>(inv.y),
               static_cast<float>(inv.z)};
}

// transform::Rigid3d::inverse().cast<float>() (rigid_transform.h:148-152) of pose {t xyz,
// q wxyz}: the conjugate, and -(conjugate * t) by Eigen 3.3's _transformVector in double.
inline Rigid3f Rigid3dInverseCast(const double pose[7]) {
  const double w = pose[3], x = -pose[4], y = -pose[5], z = -pose[6];
  const double* t = pose;
  double uv[3] = {y * t[2] - z * t[1], z * t[0] - x * t[2], x * t[1] - y * t[0]};
  for (double& u : uv) u += u;
  const double c[3] = {y * uv[2] - z * uv[1], z * uv[0] - x * uv[2], x * uv[1] - y * uv[0]};
  return Rigid3f{Vec3f{static_cast<float>(-(t[0] + w * uv[0] + c[0])),
                       static_cast<float>(-(t[1] + w * uv[1] + c[1])),
                       static_cast<float>(-(t[2] + w * uv[2] + c[2]))},
                 Quatf{static_cast<float>(w), static_cast<float>(x), static_cast<float>(y),
                       static_cast<float>(z)}};
}

// Quaternionf(AngleAxisf(angle, UnitZ)): Eigen takes cos / sin of the float half angle.
inline Quatf QuatFromAngleAxisZ(float angle) {
  const float ha = 0.5f * angle;
  return QuatFromCosSinZ(std::cos(ha), std::sin(ha));
}

// transform/transform.h:42-47
inline float GetYaw(const Quatf& q) {
  const Vec3f d = Rotate(q, Vec3f{1.f, 0.f, 0.f});
  return std::atan2(d.y, d.x);
}

// transform/transform.h:34-37: 2 * atan2(rotation.vec().norm(), |rotation.w()|)
inline float GetAngle(const Rigid3f& transform) {
  const Quatf& q = transform.q;
  return 2.f * std::atan2(std::sqrt(q.x * q.x + q.y * q.y + q.z * q.z), std::abs(q.w));
}

// transform/transform.h:85-99
inline Quatf AngleAxisVectorToRotationQuaternion(const Vec3f& aa) {
  float scale = 0.5f;
  float w = 1.f;
  constexpr double kCutoffAngle = 1e-8;
  const float squared_norm = aa.x * aa.x + aa.y * aa.y + aa.z * aa.z;
  if (squared_norm > kCutoffAngle) {
    const float norm = std::sqrt(squared_norm);
    scale = static_cast<float>(std::sin(norm / 2.) / norm);
    w = static_cast<float>(std::cos(norm / 2.));
  }
  return Quatf{w, scale * aa.x, scale * aa.y, scale * aa.z};
}

}  // namespace csm

#undef CSM_HD

#endif  // CSM_RIGID3F_H_
