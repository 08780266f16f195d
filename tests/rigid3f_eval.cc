// TEST INFRASTRUCTURE ONLY — never linked into libcsm_b200.so.
//
// Evaluates the functions of cartographer_b200/csrc/rigid3f.h that local_slam.py restates in
// numpy float32 (rigid3f_apply, rigid3f_mul, rigid3f_inverse, embed3d_f's rotation), so that
// tests/test_local_slam2d_stages_cpu.py can compare the Python results with the header's bit
// for bit.  It is linked with tests/rigid3f_check.cc, which holds the header equal to the
// oracle on the same records.
#include "../cartographer_b200/csrc/rigid3f.h"

// `rec`: n records of 21 floats laid out as in rigid3f_check.cc.  `out`: 21 floats per record:
// Rigid3Apply(ra, v) (3), Rigid3Mul(ra, rb) (7: t, q), Rigid3Inverse(ra) (7) and
// QuatFromAngleAxisZ(angle) (4).
extern "C" void rigid3f_eval(const float* rec, int n, float* out) {
  for (int i = 0; i < n; ++i) {
    const float* r = rec + 21 * static_cast<long>(i);
    float* o = out + 21 * static_cast<long>(i);
    const csm::Rigid3f ra{csm::Vec3f{r[11], r[12], r[13]}, csm::Quatf{r[0], r[1], r[2], r[3]}};
    const csm::Rigid3f rb{csm::Vec3f{r[14], r[15], r[16]}, csm::Quatf{r[4], r[5], r[6], r[7]}};
    const csm::Vec3f p = csm::Rigid3Apply(ra, csm::Vec3f{r[8], r[9], r[10]});
    const csm::Rigid3f m = csm::Rigid3Mul(ra, rb);
    const csm::Rigid3f v = csm::Rigid3Inverse(ra);
    const csm::Quatf z = csm::QuatFromAngleAxisZ(r[17]);
    const float vals[21] = {p.x,     p.y,     p.z,     m.t.x,   m.t.y,   m.t.z,   m.q.w,
                            m.q.x,   m.q.y,   m.q.z,   v.t.x,   v.t.y,   v.t.z,   v.q.w,
                            v.q.x,   v.q.y,   v.q.z,   z.w,     z.x,     z.y,     z.z};
    for (int k = 0; k < 21; ++k) o[k] = vals[k];
  }
}
