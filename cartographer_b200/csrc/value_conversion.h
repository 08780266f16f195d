// The 16-bit cell encoding of the grids (cartographer/mapping/probability_values.{h,cc},
// value_conversion_tables.cc, tsd_value_converter.{h,cc}) in float, as the reference evaluates
// it: value 0 is unknown, values 1..32767 map linearly onto [lo, hi], and bit 15 marks a cell
// already updated in the current insert.  Plain C++ on the host, so that the CPU emulation
// harnesses include it too; the two device helpers at the end are CUDA only.
#ifndef CSM_VALUE_CONVERSION_H_
#define CSM_VALUE_CONVERSION_H_

#include <cmath>
#include <cstdint>

namespace csm {

constexpr int kValueCount = 32768;             // probability_values.cc:25
constexpr uint16_t kUpdateMarker = 1u << 15;   // probability_values.h:82, tsd_value_converter.h:95

// probability_values.h:64-67
constexpr float kMinProbability = 0.1f;
constexpr float kMaxProbability = 1.f - kMinProbability;
constexpr float kMinCorrespondenceCost = 1.f - kMaxProbability;
constexpr float kMaxCorrespondenceCost = 1.f - kMinProbability;

// SlowValueToBoundedFloat (value_conversion_tables.cc:29-37) for value > 0:
// value * scale + bias, the float bounds [lo, hi] spread over values 1..32767.
struct ValueConversion {
  float scale, bias;
  float operator()(int value) const { return value * scale + bias; }
};

inline ValueConversion MakeValueConversion(float lo, float hi) {
  ValueConversion c;
  c.scale = (hi - lo) / (kValueCount - 2.f);
  c.bias = lo - c.scale;
  return c;
}

// Values per unit of [lo, hi]: the factor of BoundedFloatToValue and of TSDValueConverter's
// TSDToValue / WeightToValue (tsd_value_converter.cc:24-34).
inline float ValueResolution(float lo, float hi) { return (kValueCount - 2.f) / (hi - lo); }

// BoundedFloatToValue (probability_values.h:32-44)
inline uint16_t BoundedFloatToValue(float v, float lo, float hi) {
  const float c = v > hi ? hi : (v < lo ? lo : v);
  return static_cast<uint16_t>(std::lround((c - lo) * ValueResolution(lo, hi)) + 1);
}

inline float Odds(float p) { return p / (1.f - p); }
inline float ProbabilityFromOdds(float odds) { return odds / (odds + 1.f); }

// ComputeLookupTableToApplyOdds (probability_values.cc:76-87) into kValueCount entries.
inline void ComputeLookupTableToApplyOdds(float odds, uint16_t* table) {
  const ValueConversion probability = MakeValueConversion(kMinProbability, kMaxProbability);
  table[0] = BoundedFloatToValue(ProbabilityFromOdds(odds), kMinProbability, kMaxProbability) +
             kUpdateMarker;
  for (int cell = 1; cell != kValueCount; ++cell)
    table[cell] = BoundedFloatToValue(ProbabilityFromOdds(odds * Odds(probability(cell))),
                                      kMinProbability, kMaxProbability) +
                  kUpdateMarker;
}

// ComputeLookupTableToApplyCorrespondenceCostOdds (probability_values.cc:89-105) into
// kValueCount entries.
inline void ComputeLookupTableToApplyCorrespondenceCostOdds(float odds, uint16_t* table) {
  const ValueConversion cost = MakeValueConversion(kMinCorrespondenceCost, kMaxCorrespondenceCost);
  table[0] = BoundedFloatToValue(1.f - ProbabilityFromOdds(odds), kMinCorrespondenceCost,
                                 kMaxCorrespondenceCost) +
             kUpdateMarker;
  for (int cell = 1; cell != kValueCount; ++cell)
    table[cell] = BoundedFloatToValue(1.f - ProbabilityFromOdds(odds * Odds(1.f - cost(cell))),
                                      kMinCorrespondenceCost, kMaxCorrespondenceCost) +
                  kUpdateMarker;
}

// TSDValueConverter's value -> tsd / weight (tsd_value_converter.cc:24-34): tsd over
// [-truncation, truncation], weight over [0, max_weight].
struct TsdfConversion {
  float tsd_scale, tsd_bias, min_tsd, w_scale, w_bias;
};

inline TsdfConversion MakeTsdfConversion(float truncation, float max_weight) {
  const ValueConversion tsd = MakeValueConversion(-truncation, truncation);
  const ValueConversion weight = MakeValueConversion(0.f, max_weight);
  return TsdfConversion{tsd.scale, tsd.bias, -truncation, weight.scale, weight.bias};
}

#ifdef __CUDACC__
// ApplyLookupTable (probability_grid.cc:58-71, hybrid_grid.h:502-518) on one cell: applies
// `table` unless the cell carries the update marker; true if this call applied it.
__device__ __forceinline__ bool ApplyTable(uint16_t* cell, const uint16_t* __restrict__ table) {
  unsigned short* c = reinterpret_cast<unsigned short*>(cell);
  unsigned short old = *c;
  while (!(old & kUpdateMarker)) {
    const unsigned short prev = atomicCAS(c, old, table[old]);
    if (prev == old) return true;
    old = prev;
  }
  return false;
}

// FinishUpdate on cell `i` of `cells`: neighbouring 16-bit cells share a word, so the marker is
// cleared with a 32-bit atomic (the array holds whole words).
template <typename Index>
__device__ __forceinline__ void ClearUpdateMarker(uint16_t* cells, Index i) {
  unsigned* word = reinterpret_cast<unsigned*>(cells + (i & ~static_cast<Index>(1)));
  atomicAnd(word, ~(static_cast<unsigned>(kUpdateMarker) << (16 * (i & 1))));
}
#endif

}  // namespace csm

#endif  // CSM_VALUE_CONVERSION_H_
