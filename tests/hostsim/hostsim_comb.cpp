// Host build of the comb key record and its ladder (key_comb_build, ecmult_comb) for GPU-less unit tests.
// TEST BUILD ONLY: never linked into the product library.
#include "../../rusty_kaspa_b200/csrc/kgv_verify.cuh"
#include <cstdint>
#include <cstring>
using namespace kgv;

struct HostTab {
  uint32_t d[8][16];
  void put(int e, int w, uint32_t v) { d[e][w] = v; }
  uint32_t get(int e, int w) const { return d[e][w]; }
};
// Generator-table entries are computed on demand from their offset in a table placed at address 0 (the device reads the prebuilt
// [8][65536][16] table); any other address is a record entry and is read as it is.
struct HostGLoad {
  void operator()(fe& x, fe& y, const uint32_t* entry) const {
    const uintptr_t idx = (uintptr_t)entry / 64;
    if (idx < (uintptr_t)8 * 65536) {
      fe bx, by;
      gtab_base(bx, by, (int)(idx >> 16));
      gtab_entry(x, y, (uint32_t)(idx & 0xFFFFu), bx, by);
      return;
    }
    for (int w = 0; w < 8; w++) { x.v[w] = entry[w]; y.v[w] = entry[8 + w]; }
  }
};
extern "C" {
// pkw: 8 big-endian words of x; rec: KGV_KC_WORDS words.  Returns the record's verdict.
int hs_comb_build(const uint32_t* pkw, uint32_t tag, uint32_t* rec) {
  key_comb_build(rec, tag, pkw);
  return (int)rec[KGV_KC_STATUS];
}
// R = kP * P + kG * G from P's comb record (kP, kG: 8 little-endian limbs, < n).  Returns 1 for the point at infinity, else 0 and the
// canonical affine x, y of R (8 limbs each) in xy.
int hs_ecmult_comb(const uint32_t* rec, const uint32_t* kP, const uint32_t* kG, uint32_t* xy) {
  HostTab tab;
  gej R;
  ecmult_comb(R, kP, kG, rec, tab, (const uint32_t*)nullptr, HostGLoad());
  if (R.inf) return 1;
  fe zi, zi2, x, y;
  fe_inv(zi, R.z);
  fe_sqr(zi2, zi);
  fe_mul(x, R.x, zi2);
  fe_mul(y, R.y, zi2);
  fe_mul(y, y, zi);
  fe_normalize(x);
  fe_normalize(y);
  memcpy(xy, x.v, 32);
  memcpy(xy + 8, y.v, 32);
  return 0;
}
void hs_gtab_base(int j, uint32_t* xy) {
  fe x, y;
  gtab_base(x, y, j);
  memcpy(xy, x.v, 32);
  memcpy(xy + 8, y.v, 32);
}
}
