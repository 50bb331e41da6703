// Host build of the group law and of the wide-accumulator fold (portable primitive bodies) for GPU-less unit tests.
// TEST BUILD ONLY: never linked into the product library.
#include "../../rusty_kaspa_b200/csrc/kgv_secp.cuh"
#include <cstring>
using namespace kgv;

static void load(fe& x, const uint8_t* b) { memcpy(x.v, b, 32); }
static void store(uint8_t* b, const fe& x) { memcpy(b, x.v, 32); }
// gej as 97 bytes: x, y, z (little-endian limbs), inf
static void load_gej(gej& r, const uint8_t* b) { load(r.x, b); load(r.y, b + 32); load(r.z, b + 64); r.inf = b[96] != 0; }
static void store_gej(uint8_t* b, const gej& r) { store(b, r.x); store(b + 32, r.y); store(b + 64, r.z); b[96] = r.inf; }

extern "C" {
// r = v + top * 2^256 (mod p), weakly reduced
void hs_fe_fold(const uint8_t* v, int32_t top, uint8_t* r) {
  fex a;
  memcpy(a.v, v, 32);
  a.top = (uint32_t)top;
  fe z;
  fe_fold(z, a);
  store(r, z);
}
void hs_gej_double_n(uint8_t* p, int n) { gej r; load_gej(r, p); gej_double_n(r, n); store_gej(p, r); }
void hs_gej_add_ge(uint8_t* p, const uint8_t* bx, const uint8_t* by, uint8_t* hout) {
  gej r;
  fe x, y, h;
  load_gej(r, p); load(x, bx); load(y, by);
  gej_add_ge(r, x, y, &h);
  store_gej(p, r);
  store(hout, h);
}
}
