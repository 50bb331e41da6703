// Host build of the joint table of a comb record and its ladder (key_joint_build, recode_joint, ecmult_joint) for GPU-less unit tests.
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
static int affine_out(const gej& R, uint32_t* xy) {
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
extern "C" {
// pkw: 8 big-endian words of x; rec: KGV_KJ_WORDS words, filled as k_key_prepare fills a comb-form record.  Returns the verdict.
int hs_joint_build(const uint32_t* pkw, uint32_t tag, uint32_t* rec) {
  key_comb_build(rec, tag, pkw);
  if (rec[KGV_KC_STATUS] == KGV_ST_VALID) key_joint_build(rec);
  return (int)rec[KGV_KC_STATUS];
}
int hs_kj_words() { return KGV_KJ_WORDS; }
// m: 5 limbs.  h: 5 words of packed digits; returns fix.
int hs_recode_joint(const uint32_t* m, uint32_t* h) {
  bool fix;
  recode_joint(h, fix, m);
  return fix;
}
// the GLV split of k: m1, m2 (5 limbs each) and the flags neg1, neg2
void hs_glv_split(const uint32_t* k, uint32_t* m1, uint32_t* m2, uint32_t* flags) {
  bool n1, n2;
  glv_split(m1, n1, m2, n2, k);
  flags[0] = n1;
  flags[1] = n2;
}
// R = kP * P + kG * G by ecmult_joint (which = 0) or ecmult_comb (which = 1) from a record of hs_joint_build.  Returns 1 for the point
// at infinity, else 0 and the canonical affine x, y of R in xy.
int hs_ecmult(const uint32_t* rec, const uint32_t* kP, const uint32_t* kG, int which, uint32_t* xy) {
  HostTab tab;
  gej R;
  if (which == 0) ecmult_joint(R, kP, kG, rec, rec + KGV_KJ_JOINT, tab, (const uint32_t*)nullptr, HostGLoad());
  else ecmult_comb(R, kP, kG, rec, tab, (const uint32_t*)nullptr, HostGLoad());
  return affine_out(R, xy);
}
}
