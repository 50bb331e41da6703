// Host build of the comb-form key record (key_joint_record_build, KGV_JR_*) and the reference pair it is checked against
// (key_comb_build + key_joint_build, KGV_KJ_*), for GPU-less unit tests.
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
// as in hostsim_comb.cpp: generator-table entries computed on demand from their offset in a table placed at address 0, any other
// address read as it is
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
// the layout: words per record, then the offsets of P, the verdict and the joint table
void hs_jr_layout(uint32_t* out) {
  out[0] = KGV_JR_WORDS;
  out[1] = KGV_JR_P;
  out[2] = KGV_JR_STATUS;
  out[3] = KGV_JR_JOINT;
  out[4] = KGV_KJ_WORDS;
  out[5] = KGV_KJ_JOINT;
}
// pkw: 8 big-endian words of x; rec: KGV_JR_WORDS words, filled as k_key_prepare fills a comb-form record.  Returns the verdict.
int hs_jr_build(const uint32_t* pkw, uint32_t tag, uint32_t* rec) {
  key_joint_record_build(rec, tag, pkw);
  return (int)rec[KGV_JR_STATUS];
}
// the reference pair: rec: KGV_KJ_WORDS words.  Returns the verdict.
int hs_ref_build(const uint32_t* pkw, uint32_t tag, uint32_t* rec) {
  key_comb_build(rec, tag, pkw);
  if (rec[KGV_KC_STATUS] == KGV_ST_VALID) key_joint_build(rec);
  return (int)rec[KGV_KC_STATUS];
}
// R = kP * P + kG * G by ecmult_joint from a record of hs_jr_build, as ecmult_key calls it.  Returns 1 for the point at infinity,
// else 0 and the canonical affine x, y of R in xy.
int hs_jr_ecmult(const uint32_t* rec, const uint32_t* kP, const uint32_t* kG, uint32_t* xy) {
  HostTab tab;
  gej R;
  ecmult_joint(R, kP, kG, rec + KGV_JR_P, rec + KGV_JR_JOINT, tab, (const uint32_t*)nullptr, HostGLoad());
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
}
