// TEST INFRASTRUCTURE ONLY — never linked into libcsm_b200.so.
//
// Evaluates every function of cartographer_b200/csrc/rigid3f.h on the host next to the oracle's
// function of the same name (oracle/oracle_common.h, oracle/oracle_3d.h) and compares the
// results bit for bit.  tests/test_rigid3f_cpu.py builds it together with oracle/oracle_3d.cc,
// with the oracle's flags (-O3 -ffp-contract=off).
#include <cstdio>
#include <cstring>

#include "../cartographer_b200/csrc/rigid3f.h"
#include "../oracle/oracle_3d.h"

namespace {

struct Mismatches {
  int count = 0;
  char* msg;
  int msg_len;

  template <typename A, typename B>
  void Check(const char* name, int record, const A& a, const B& b) {
    static_assert(sizeof(A) == sizeof(B), "layouts differ");
    if (std::memcmp(&a, &b, sizeof(A)) == 0) return;
    if (count++ == 0) std::snprintf(msg, msg_len, "%s differs on record %d", name, record);
  }
};

template <typename V>
V Vec(const float* p) { return V{p[0], p[1], p[2]}; }
template <typename Q>
Q Quat(const float* p) { return Q{p[0], p[1], p[2], p[3]}; }

}  // namespace

// `rec`: n records of 21 floats: quaternions a (w, x, y, z) and b, a point v, translations ta and
// tb, an angle about z and an angle-axis vector.  `qd`: nd double quaternions (w, x, y, z).
// Returns the number of mismatches and describes the first one in `msg`.
extern "C" int rigid3f_compare(const float* rec, int n, const double* qd, int nd, char* msg,
                               int msg_len) {
  Mismatches m{0, msg, msg_len};
  for (int i = 0; i < n; ++i) {
    const float* r = rec + 21 * static_cast<long>(i);
    const csm::Quatf qa = Quat<csm::Quatf>(r), qb = Quat<csm::Quatf>(r + 4);
    const oracle::Quatf oqa = Quat<oracle::Quatf>(r), oqb = Quat<oracle::Quatf>(r + 4);
    const csm::Vec3f v = Vec<csm::Vec3f>(r + 8), ta = Vec<csm::Vec3f>(r + 11),
                     tb = Vec<csm::Vec3f>(r + 14), aa = Vec<csm::Vec3f>(r + 18);
    const oracle::Vec3f ov = Vec<oracle::Vec3f>(r + 8), ota = Vec<oracle::Vec3f>(r + 11),
                        otb = Vec<oracle::Vec3f>(r + 14), oaa = Vec<oracle::Vec3f>(r + 18);
    const float angle = r[17];
    const csm::Rigid3f ra{ta, qa}, rb{tb, qb};
    const oracle::Rigid3f ora{ota, oqa}, orb{otb, oqb};

    m.Check("Cross", i, csm::Cross(v, ta), oracle::Cross(ov, ota));
    m.Check("Rotate", i, csm::Rotate(qa, v), oracle::Rotate(oqa, ov));
    m.Check("RotateAsRigid3f", i, csm::RotateAsRigid3f(qa, v), oracle::RotateAsRigid3f(oqa, ov));
    m.Check("Rigid3Apply", i, csm::Rigid3Apply(ra, v), oracle::Rigid3Apply(ora, ov));
    m.Check("QuatFromAngleAxisZ", i, csm::QuatFromAngleAxisZ(angle),
            oracle::QuatFromAngleAxisZ(angle));
    m.Check("QuatMul", i, csm::QuatMul(qa, qb), oracle::QuatMul(oqa, oqb));
    m.Check("QuatSquaredNorm", i, csm::QuatSquaredNorm(qa), oracle::QuatSquaredNorm(oqa));
    m.Check("QuatNormalized", i, csm::QuatNormalized(qa), oracle::QuatNormalized(oqa));
    m.Check("QuatConjugate", i, csm::QuatConjugate(qa), oracle::QuatConjugate(oqa));
    m.Check("QuatInverse", i, csm::QuatInverse(qa), oracle::QuatInverse(oqa));
    m.Check("Rigid3Inverse", i, csm::Rigid3Inverse(ra), oracle::Rigid3Inverse(ora));
    m.Check("Rigid3Mul", i, csm::Rigid3Mul(ra, rb), oracle::Rigid3Mul(ora, orb));
    m.Check("GetYaw", i, csm::GetYaw(qa), oracle::GetYaw(oqa));
    m.Check("GetAngle", i, csm::GetAngle(ra), oracle::GetAngle(ora));
    m.Check("AngleAxisVectorToRotationQuaternion", i,
            csm::AngleAxisVectorToRotationQuaternion(aa),
            oracle::AngleAxisVectorToRotationQuaternion(oaa));
  }
  for (int i = 0; i < nd; ++i) {
    const double* p = qd + 4 * static_cast<long>(i);
    m.Check("QuatCastInverseD", i, csm::QuatCastInverseD(csm::Quatd{p[0], p[1], p[2], p[3]}),
            oracle::QuatCastInverseD(oracle::Quatd{p[0], p[1], p[2], p[3]}));
  }
  return m.count;
}
