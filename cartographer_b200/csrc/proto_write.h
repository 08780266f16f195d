// Protobuf wire-format writing for csm_grid3d_to_proto and csm_rt_grid2d_to_proto: the few
// proto3 encodings proto::HybridGrid and proto::Grid2D need, byte for byte as the protobuf C++
// serialiser writes them (fields in field-number order, implicit-presence scalars omitted when
// zero, repeated scalars packed, empty repeated fields omitted).  Every writer returns the
// advanced pointer; the *Size functions give the bytes the writer would emit, so that a message
// can be sized before anything is written.
#ifndef CSM_PROTO_WRITE_H_
#define CSM_PROTO_WRITE_H_

#include <cstdint>
#include <cstring>

namespace csm {
namespace wire {

enum { kVarint = 0, kFixed64 = 1, kLengthDelimited = 2, kFixed32 = 5 };

inline int64_t VarintSize(uint64_t v) {
  int64_t n = 1;
  while (v >= 0x80) {
    v >>= 7;
    ++n;
  }
  return n;
}

inline uint8_t* PutVarint(uint8_t* p, uint64_t v) {
  while (v >= 0x80) {
    *p++ = static_cast<uint8_t>(v | 0x80);
    v >>= 7;
  }
  *p++ = static_cast<uint8_t>(v);
  return p;
}

// Field keys of field numbers below 16 are one byte.
inline uint8_t* PutKey(uint8_t* p, int field, int wire_type) {
  *p++ = static_cast<uint8_t>((field << 3) | wire_type);
  return p;
}

// int32 as protobuf writes it: negative values sign-extended to ten bytes.
inline uint64_t Int32Bits(int32_t v) { return static_cast<uint64_t>(static_cast<int64_t>(v)); }
// sint32: zig-zag.
inline uint64_t ZigZag32(int32_t v) {
  return static_cast<uint32_t>((static_cast<uint32_t>(v) << 1) ^ static_cast<uint32_t>(v >> 31));
}

// A proto3 float / double is written unless its bit pattern is all zeros: +0.0 is omitted and
// -0.0 is written (the bit-pattern test protobuf C++'s generated serialisers make).
inline bool FloatPresent(float v) {
  uint32_t b;
  std::memcpy(&b, &v, 4);
  return b != 0;
}
inline bool DoublePresent(double v) {
  uint64_t b;
  std::memcpy(&b, &v, 8);
  return b != 0;
}

inline int64_t FloatFieldSize(float v) { return FloatPresent(v) ? 5 : 0; }
inline uint8_t* PutFloatField(uint8_t* p, int field, float v) {
  if (!FloatPresent(v)) return p;
  p = PutKey(p, field, kFixed32);
  std::memcpy(p, &v, 4);
  return p + 4;
}
inline int64_t DoubleFieldSize(double v) { return DoublePresent(v) ? 9 : 0; }
inline uint8_t* PutDoubleField(uint8_t* p, int field, double v) {
  if (!DoublePresent(v)) return p;
  p = PutKey(p, field, kFixed64);
  std::memcpy(p, &v, 8);
  return p + 8;
}
inline int64_t Int32FieldSize(int32_t v) { return v != 0 ? 1 + VarintSize(Int32Bits(v)) : 0; }
inline uint8_t* PutInt32Field(uint8_t* p, int field, int32_t v) {
  if (v == 0) return p;
  return PutVarint(PutKey(p, field, kVarint), Int32Bits(v));
}

// A length-delimited field (sub-message or packed repeated field) of `len` payload bytes.
inline int64_t DelimitedSize(int64_t len) { return 1 + VarintSize(len) + len; }
inline uint8_t* PutDelimitedHeader(uint8_t* p, int field, int64_t len) {
  return PutVarint(PutKey(p, field, kLengthDelimited), static_cast<uint64_t>(len));
}

}  // namespace wire
}  // namespace csm

#endif  // CSM_PROTO_WRITE_H_
