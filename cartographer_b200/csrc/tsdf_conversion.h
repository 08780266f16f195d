// TSDValueConverter's value -> tsd / weight constants, shared by the real-time matcher
// (rt2d.cu), the refinement's host side (refine2d.cu) and the refinement's CPU emulation
// harness; plain C++, no CUDA.
#ifndef CSM_TSDF_CONVERSION_H_
#define CSM_TSDF_CONVERSION_H_

namespace csm {

// tsd_value_converter.cc:24-34, value_conversion_tables.cc:29-37 evaluated in float:
// value * scale + bias for value > 0.
struct TsdfConversion {
  float tsd_scale, tsd_bias, min_tsd, w_scale, w_bias;
};

inline TsdfConversion MakeTsdfConversion(float truncation, float max_weight) {
  TsdfConversion c;
  c.min_tsd = -truncation;
  c.tsd_scale = (truncation - c.min_tsd) / 32766.f;
  c.tsd_bias = c.min_tsd - c.tsd_scale;
  c.w_scale = (max_weight - 0.f) / 32766.f;
  c.w_bias = 0.f - c.w_scale;
  return c;
}

}  // namespace csm

#endif  // CSM_TSDF_CONVERSION_H_
