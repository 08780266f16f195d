// Grid ingest from Cartographer's serialized forms, straight into device stacks.
//   * proto::Grid2D      (mapping/proto/grid_2d.proto:23-42)   -> csm_stack2d
//   * proto::HybridGrid  (mapping/proto/hybrid_grid.proto:19-28) -> csm_matcher3d
//   * a .pbstream file   (io/proto_stream.cc:27-110 framing: 8-byte magic, then
//     [8-byte little-endian size, gzip blob]*; every blob after the header is a
//     proto::SerializedData, mapping/proto/serialization.proto) -> one stack per 2D submap
// The protobuf runtime is not needed: the wire format of these few messages is decoded by
// hand (varints, length-delimited fields, fixed32/64), following the field numbers in the
// .proto files cited above.  Mirrors Grid2D::Grid2D(const proto::Grid2D&) (mapping/2d/
// grid_2d.cc:75-96) and HybridGrid(const proto::HybridGrid&) (mapping/3d/hybrid_grid.h:473-484).
#include <zlib.h>

#include <cstdio>
#include <string>

#include "engine2d.cuh"
#include "value_conversion.h"

namespace {

using namespace csm;

struct Reader {
  const uint8_t* p;
  const uint8_t* end;
  bool ok = true;
  Reader(const uint8_t* b, size_t n) : p(b), end(b + n) {}
  bool done() const { return p >= end || !ok; }
  uint64_t Varint() {
    uint64_t v = 0;
    for (int shift = 0; shift < 64 && p < end; shift += 7) {
      const uint8_t b = *p++;
      v |= static_cast<uint64_t>(b & 0x7f) << shift;
      if (!(b & 0x80)) return v;
    }
    ok = false;
    return 0;
  }
  // returns the field number, sets wire type; for length-delimited fields sets [sub, sub+len)
  int Field(int* wire, Reader* sub, uint64_t* scalar) {
    const uint64_t key = Varint();
    if (!ok) return 0;
    *wire = static_cast<int>(key & 7);
    switch (*wire) {
      case 0: *scalar = Varint(); break;
      case 1:
        if (end - p < 8) { ok = false; return 0; }
        std::memcpy(scalar, p, 8); p += 8; break;
      case 5: {
        if (end - p < 4) { ok = false; return 0; }
        uint32_t v; std::memcpy(&v, p, 4); p += 4; *scalar = v; break;
      }
      case 2: {
        const uint64_t len = Varint();
        if (!ok || len > static_cast<uint64_t>(end - p)) { ok = false; return 0; }
        *sub = Reader(p, static_cast<size_t>(len));
        p += len;
        break;
      }
      default: ok = false; return 0;
    }
    return static_cast<int>(key >> 3);
  }
};

inline double AsDouble(uint64_t bits) { double d; std::memcpy(&d, &bits, 8); return d; }
inline float AsFloat(uint64_t bits) { const uint32_t b = static_cast<uint32_t>(bits); float f; std::memcpy(&f, &b, 4); return f; }
inline int32_t ZigZag(uint64_t v) { return static_cast<int32_t>((v >> 1) ^ (~(v & 1) + 1)); }

// repeated int32 / sint32, packed or not
template <typename F>
void Repeated(int wire, Reader& sub, uint64_t scalar, F push) {
  if (wire == 2) {
    while (!sub.done()) { const uint64_t v = sub.Varint(); if (sub.ok) push(v); }
  } else {
    push(scalar);
  }
}

struct Grid2DProto {
  double resolution = 0., max_x = 0., max_y = 0.;
  int nx = 0, ny = 0;
  float min_cost = 0.f, max_cost = 0.f;
  bool has_min = false, has_max = false, is_tsdf = false;
  std::vector<uint16_t> cells;
};

bool ParseGrid2D(Reader r, Grid2DProto* g, std::string* err) {
  int wire;
  uint64_t v;
  Reader sub(nullptr, 0);
  while (!r.done()) {
    const int f = r.Field(&wire, &sub, &v);
    if (!r.ok) break;
    if (f == 1 && wire == 2) {          // MapLimits limits
      Reader l = sub;
      Reader s2(nullptr, 0);
      while (!l.done()) {
        const int lf = l.Field(&wire, &s2, &v);
        if (!l.ok) break;
        if (lf == 1 && wire == 1) g->resolution = AsDouble(v);
        else if (lf == 2 && wire == 2) {  // Vector2d max
          Reader m = s2; Reader s3(nullptr, 0);
          while (!m.done()) {
            const int mf = m.Field(&wire, &s3, &v);
            if (!m.ok) break;
            if (mf == 1 && wire == 1) g->max_x = AsDouble(v);
            else if (mf == 2 && wire == 1) g->max_y = AsDouble(v);
          }
        } else if (lf == 3 && wire == 2) {  // CellLimits
          Reader c = s2; Reader s3(nullptr, 0);
          while (!c.done()) {
            const int cf = c.Field(&wire, &s3, &v);
            if (!c.ok) break;
            if (cf == 1 && wire == 0) g->nx = static_cast<int>(v);
            else if (cf == 2 && wire == 0) g->ny = static_cast<int>(v);
          }
        }
      }
      if (!l.ok) r.ok = false;
    } else if (f == 2) {                // repeated int32 cells
      bool range_ok = true;
      Repeated(wire, sub, v, [&](uint64_t c) {
        if (c > 65535u) range_ok = false;   // CHECK_LE(cell, uint16 max), grid_2d.cc:93
        g->cells.push_back(static_cast<uint16_t>(c));
      });
      if (!range_ok) { *err = "a cell value exceeds uint16"; return false; }
    } else if (f == 5 && wire == 2) {
      g->is_tsdf = true;
    } else if (f == 6 && wire == 5) {
      g->min_cost = AsFloat(v); g->has_min = true;
    } else if (f == 7 && wire == 5) {
      g->max_cost = AsFloat(v); g->has_max = true;
    }
  }
  if (!r.ok) { *err = "malformed proto::Grid2D"; return false; }
  // MinCorrespondenceCostFromProto / Max... (grid_2d.cc:27-52): legacy grids without the
  // two fields are probability grids with the default bounds
  if (g->min_cost == 0.f && g->max_cost == 0.f) {
    g->min_cost = kMinCorrespondenceCost;
    g->max_cost = kMaxCorrespondenceCost;
  }
  if (g->nx < 1 || g->ny < 1 || static_cast<size_t>(g->nx) * g->ny != g->cells.size()) {
    *err = "cell count does not match the cell limits";
    return false;
  }
  return true;
}

struct HybridProto {
  float resolution = 0.f;
  std::vector<int32_t> x, y, z;
  std::vector<uint16_t> values;
};

bool ParseHybrid(Reader r, HybridProto* g, std::string* err) {
  int wire;
  uint64_t v;
  Reader sub(nullptr, 0);
  bool range_ok = true;
  while (!r.done()) {
    const int f = r.Field(&wire, &sub, &v);
    if (!r.ok) break;
    if (f == 1 && wire == 5) g->resolution = AsFloat(v);
    else if (f == 3) Repeated(wire, sub, v, [&](uint64_t c) { g->x.push_back(ZigZag(c)); });
    else if (f == 4) Repeated(wire, sub, v, [&](uint64_t c) { g->y.push_back(ZigZag(c)); });
    else if (f == 5) Repeated(wire, sub, v, [&](uint64_t c) { g->z.push_back(ZigZag(c)); });
    else if (f == 6) Repeated(wire, sub, v, [&](uint64_t c) {
      if (c > 65535u) range_ok = false;
      g->values.push_back(static_cast<uint16_t>(c));
    });
  }
  if (!r.ok || !range_ok) { *err = "malformed proto::HybridGrid"; return false; }
  // CHECK_EQ(values_size, {x,y,z}_indices_size) (hybrid_grid.h:475-477)
  if (g->x.size() != g->values.size() || g->y.size() != g->values.size() ||
      g->z.size() != g->values.size()) {
    *err = "index / value counts differ";
    return false;
  }
  return true;
}

// HybridGrid(const proto&) stores SetProbability(ValueToProbability(v)) =
// ProbabilityToValue(ValueToProbability(v)): identity for 1..32767, 0 stays unknown... except
// that SetProbability of kMinProbability yields value 1; value 0 entries are not serialized.
void FlattenHybrid(const HybridProto& g, std::vector<int32_t>* idx, std::vector<uint16_t>* val) {
  idx->reserve(3 * g.values.size());
  val->reserve(g.values.size());
  for (size_t i = 0; i < g.values.size(); ++i) {
    idx->push_back(g.x[i]);
    idx->push_back(g.y[i]);
    idx->push_back(g.z[i]);
    uint16_t v = g.values[i] & 0x7fff;
    if (v == 0) v = 1;   // ValueToProbability(0) = kMinProbability -> ProbabilityToValue = 1
    val->push_back(v);
  }
}

bool Gunzip(const uint8_t* data, size_t n, std::string* out) {
  z_stream zs;
  std::memset(&zs, 0, sizeof(zs));
  if (inflateInit2(&zs, 16 + MAX_WBITS) != Z_OK) return false;
  zs.next_in = const_cast<Bytef*>(data);
  zs.avail_in = static_cast<uInt>(n);
  char buf[1 << 16];
  int rc;
  do {
    zs.next_out = reinterpret_cast<Bytef*>(buf);
    zs.avail_out = sizeof(buf);
    rc = inflate(&zs, Z_NO_FLUSH);
    if (rc != Z_OK && rc != Z_STREAM_END) { inflateEnd(&zs); return false; }
    out->append(buf, sizeof(buf) - zs.avail_out);
  } while (rc != Z_STREAM_END);
  inflateEnd(&zs);
  return true;
}

}  // namespace

extern "C" {

csm_status csm_grid2d_proto_decode(const uint8_t* grid2d, int64_t size, csm_grid2d_info* info,
                                   uint16_t* cells, int64_t cells_capacity) {
  CSM_REQUIRE(grid2d && size >= 0 && info, "null pointer");
  Grid2DProto g;
  std::string err;
  if (!ParseGrid2D(Reader(grid2d, static_cast<size_t>(size)), &g, &err)) {
    SetError("%s", err.c_str());
    return CSM_E_INVALID;
  }
  info->num_x_cells = g.nx;
  info->num_y_cells = g.ny;
  info->resolution = g.resolution;
  info->max_x = g.max_x;
  info->max_y = g.max_y;
  info->min_correspondence_cost = g.min_cost;
  info->max_correspondence_cost = g.max_cost;
  info->is_tsdf = g.is_tsdf ? 1 : 0;
  if (cells) {
    CSM_REQUIRE(cells_capacity >= static_cast<int64_t>(g.cells.size()), "cell buffer too small");
    std::memcpy(cells, g.cells.data(), g.cells.size() * 2);
  }
  return CSM_OK;
}

csm_status csm_stack2d_create_from_proto(const uint8_t* grid2d, int64_t size, int32_t depth,
                                         int32_t device, csm_stack2d** out) {
  CSM_REQUIRE(grid2d && size >= 0 && out, "null pointer");
  Grid2DProto g;
  std::string err;
  if (!ParseGrid2D(Reader(grid2d, static_cast<size_t>(size)), &g, &err)) {
    SetError("%s", err.c_str());
    return CSM_E_INVALID;
  }
  CSM_REQUIRE(!g.is_tsdf, "the fast matcher's stack is built from a ProbabilityGrid");
  return csm_stack2d_create(g.cells.data(), g.nx, g.ny, g.resolution, g.max_x, g.max_y,
                            g.min_cost, g.max_cost, depth, device, out);
}

csm_status csm_matcher3d_create_from_proto(const uint8_t* hi, int64_t hi_size, const uint8_t* lo,
                                           int64_t lo_size, const float* histogram,
                                           int32_t histogram_size, const csm_options3d* options,
                                           int32_t device, csm_matcher3d** out) {
  CSM_REQUIRE(hi && lo && hi_size >= 0 && lo_size >= 0 && out, "null pointer");
  HybridProto gh, gl;
  std::string err;
  if (!ParseHybrid(Reader(hi, static_cast<size_t>(hi_size)), &gh, &err) ||
      !ParseHybrid(Reader(lo, static_cast<size_t>(lo_size)), &gl, &err)) {
    SetError("%s", err.c_str());
    return CSM_E_INVALID;
  }
  std::vector<int32_t> hi_idx, lo_idx;
  std::vector<uint16_t> hi_val, lo_val;
  FlattenHybrid(gh, &hi_idx, &hi_val);
  FlattenHybrid(gl, &lo_idx, &lo_val);
  return csm_matcher3d_create(hi_idx.data(), hi_val.data(), static_cast<int64_t>(hi_val.size()),
                              gh.resolution, 0, lo_idx.data(), lo_val.data(),
                              static_cast<int64_t>(lo_val.size()), gl.resolution, histogram,
                              histogram_size, options, device, out);
}

csm_status csm_pbstream_load_stacks2d(const char* path, int32_t depth, int32_t device,
                                      int32_t max_stacks, csm_stack2d** stacks,
                                      int32_t* submap_ids, int32_t* num_loaded) {
  CSM_REQUIRE(path && num_loaded, "null pointer");
  CSM_REQUIRE(max_stacks >= 0 && (max_stacks == 0 || stacks), "stack array");
  *num_loaded = 0;
  FILE* f = std::fopen(path, "rb");
  if (!f) { SetError("cannot open %s", path); return CSM_E_INVALID; }
  struct Close { FILE* f; ~Close() { std::fclose(f); } } closer{f};
  auto read_u64 = [&](uint64_t* v) {
    uint8_t b[8];
    if (std::fread(b, 1, 8, f) != 8) return false;
    *v = 0;
    for (int i = 7; i >= 0; --i) *v = (*v << 8) | b[i];
    return true;
  };
  uint64_t magic = 0;
  if (!read_u64(&magic) || magic != 0x7b1d1f7b5bf501dbull) {   // io/proto_stream.cc:27
    SetError("%s is not a proto stream (bad magic)", path);
    return CSM_E_INVALID;
  }
  std::vector<uint8_t> blob;
  int count = 0;
  uint64_t size = 0;
  bool first = true;
  while (read_u64(&size)) {
    CSM_REQUIRE(size < (1ull << 32), "chunk too large");
    blob.resize(static_cast<size_t>(size));
    if (size && std::fread(blob.data(), 1, blob.size(), f) != blob.size()) {
      SetError("truncated proto stream");
      return CSM_E_INVALID;
    }
    std::string msg;
    if (!Gunzip(blob.data(), blob.size(), &msg)) {
      SetError("gzip inflate failed");
      return CSM_E_INVALID;
    }
    if (first) { first = false; continue; }   // SerializationHeader (io/internal/mapping_state_serialization)
    // SerializedData { Submap submap = 3 { SubmapId submap_id = 1; Submap2D submap_2d = 2 { Grid2D grid = 4 } } }
    Reader r(reinterpret_cast<const uint8_t*>(msg.data()), msg.size());
    int wire;
    uint64_t v;
    Reader sub(nullptr, 0);
    while (!r.done()) {
      const int fld = r.Field(&wire, &sub, &v);
      if (!r.ok) break;
      if (fld != 3 || wire != 2) continue;
      Reader sm = sub;
      Reader s2(nullptr, 0);
      int traj = 0, index = 0;
      Reader grid(nullptr, 0);
      bool has_grid = false;
      while (!sm.done()) {
        const int sf = sm.Field(&wire, &s2, &v);
        if (!sm.ok) break;
        if (sf == 1 && wire == 2) {        // SubmapId { trajectory_id = 1, submap_index = 2 }
          Reader id = s2; Reader s3(nullptr, 0);
          while (!id.done()) {
            const int idf = id.Field(&wire, &s3, &v);
            if (!id.ok) break;
            if (idf == 1 && wire == 0) traj = static_cast<int>(v);
            else if (idf == 2 && wire == 0) index = static_cast<int>(v);
          }
        } else if (sf == 2 && wire == 2) {  // Submap2D
          Reader s2d = s2; Reader s3(nullptr, 0);
          while (!s2d.done()) {
            const int f2 = s2d.Field(&wire, &s3, &v);
            if (!s2d.ok) break;
            if (f2 == 4 && wire == 2) { grid = s3; has_grid = true; }
          }
        }
      }
      if (!has_grid) continue;
      if (count < max_stacks) {
        CSM_TRY(csm_stack2d_create_from_proto(grid.p, grid.end - grid.p, depth, device,
                                              &stacks[count]));
        if (submap_ids) { submap_ids[2 * count] = traj; submap_ids[2 * count + 1] = index; }
      }
      ++count;
    }
  }
  *num_loaded = count;   // may exceed max_stacks: call again with a larger array
  return CSM_OK;
}

}  // extern "C"
