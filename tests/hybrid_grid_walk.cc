// CPU restatement of HybridGrid's storage and iterator — TEST INFRASTRUCTURE ONLY.
//
// mapping/3d/hybrid_grid.h: GridBase<uint16> = DynamicGrid<NestedGrid<FlatGrid<uint16, 3>, 3>>.
//   * FlatGrid (:59-128): 8^3 values at ToFlatIndex (:40-43, z outermost); its iterator walks them
//     in that order and skips default (0) values (:57, :106-115).
//   * NestedGrid (:130-238): 8^3 meta cells, each a FlatGrid allocated on first write; its
//     iterator walks the meta cells in ToFlatIndex order, skips null ones and runs each one's
//     FlatGrid iterator.
//   * DynamicGrid (:240-407): 2^bits_ meta cells per axis (bits_ starts at 1), each a NestedGrid,
//     indices shifted by grid_size() / 2; a write outside the cube first Grow()s it (:385-405:
//     bits_ + 1, old meta cells moved by 2^(bits_ - 1)); its iterator walks the meta cells in
//     ToFlatIndex order and un-shifts the index (:300-340).
// HybridGrid::ToProto (:528-540) writes the voxels in this iterator's order; csm_grid3d_voxels is
// checked against it.  The walk below follows the data structure, not a key formula.
#include <array>
#include <cstdint>
#include <memory>
#include <vector>

namespace {

int ToFlatIndex(int x, int y, int z, int bits) { return (((z << bits) + y) << bits) + x; }

struct Flat {
  std::array<uint16_t, 512> cells{};
};
struct Nested {
  std::array<std::unique_ptr<Flat>, 512> cells;
};

struct Dynamic {
  int bits = 1;
  std::vector<std::unique_ptr<Nested>> meta = std::vector<std::unique_ptr<Nested>>(8);
  int grid_size() const { return 64 << bits; }

  void Grow() {
    const int new_bits = bits + 1;
    std::vector<std::unique_ptr<Nested>> grown(8 * meta.size());
    for (int z = 0; z != (1 << bits); ++z)
      for (int y = 0; y != (1 << bits); ++y)
        for (int x = 0; x != (1 << bits); ++x) {
          const int o = 1 << (bits - 1);
          grown[ToFlatIndex(x + o, y + o, z + o, new_bits)] =
              std::move(meta[ToFlatIndex(x, y, z, bits)]);
        }
    meta = std::move(grown);
    bits = new_bits;
  }

  uint16_t* mutable_value(int x, int y, int z) {
    const int h = grid_size() >> 1;
    const int s[3] = {x + h, y + h, z + h};
    for (int a = 0; a < 3; ++a)
      if (static_cast<unsigned>(s[a]) >= static_cast<unsigned>(grid_size())) {
        Grow();
        return mutable_value(x, y, z);
      }
    std::unique_ptr<Nested>& n = meta[ToFlatIndex(s[0] / 64, s[1] / 64, s[2] / 64, bits)];
    if (!n) n.reset(new Nested);
    const int i[3] = {s[0] % 64, s[1] % 64, s[2] % 64};
    std::unique_ptr<Flat>& f = n->cells[ToFlatIndex(i[0] / 8, i[1] / 8, i[2] / 8, 3)];
    if (!f) f.reset(new Flat);
    return &f->cells[ToFlatIndex(i[0] % 8, i[1] % 8, i[2] % 8, 3)];
  }

  // The three nested iterators, flattened: every non-zero value in visiting order.
  template <typename Fn>
  void Walk(Fn fn) const {
    const int side = 1 << bits;
    for (int m = 0; m < side * side * side; ++m) {
      const Nested* n = meta[m].get();
      if (!n) continue;
      const int mx = m & (side - 1), my = (m >> bits) & (side - 1), mz = (m >> bits) >> bits;
      for (int k = 0; k < 512; ++k) {
        const Flat* f = n->cells[k].get();
        if (!f) continue;
        const int kx = k & 7, ky = (k >> 3) & 7, kz = k >> 6;
        for (int c = 0; c < 512; ++c) {
          if (f->cells[c] == 0) continue;
          const int cx = c & 7, cy = (c >> 3) & 7, cz = c >> 6;
          const int h = (1 << (bits - 1)) * 64;
          fn(mx * 64 + kx * 8 + cx - h, my * 64 + ky * 8 + cy - h, mz * 64 + kz * 8 + cz - h,
             f->cells[c]);
        }
      }
    }
  }
};

}  // namespace

extern "C" {

void* hgw_new() { return new Dynamic; }
void hgw_free(void* g) { delete static_cast<Dynamic*>(g); }
int hgw_bits(void* g) { return static_cast<Dynamic*>(g)->bits; }

// *mutable_value(index) = value for each entry in order (writes of 0 allocate, as they do in the
// reference, and leave nothing for the walk to visit).
void hgw_set(void* g, const int32_t* idx, const uint16_t* values, int64_t n) {
  Dynamic* d = static_cast<Dynamic*>(g);
  for (int64_t i = 0; i < n; ++i)
    *d->mutable_value(idx[3 * i], idx[3 * i + 1], idx[3 * i + 2]) = values[i];
}

// The walk into idx (n x 3) / values; returns the number of voxels, writing at most capacity.
int64_t hgw_walk(void* g, int32_t* idx, uint16_t* values, int64_t capacity) {
  int64_t n = 0;
  static_cast<Dynamic*>(g)->Walk([&](int x, int y, int z, uint16_t v) {
    if (n < capacity) {
      idx[3 * n] = x;
      idx[3 * n + 1] = y;
      idx[3 * n + 2] = z;
      values[n] = v;
    }
    ++n;
  });
  return n;
}

}  // extern "C"
