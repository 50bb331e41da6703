// Host driver of tests/test_scratch_carve.py: lays out scratch with kgv_carve / kgv_reserve_carved (kgv_internal.h) and prints, for every
// layout, the size the measuring pass gave, the size reserved and the carving pass's end, then every array's offset and requested bytes.
#include "../../rusty_kaspa_b200/csrc/kgv_internal.h"

#include <cstdlib>

static size_t g_need = 0;
// host stand-in of the device reserve: records the size asked for and keeps a 256-byte aligned buffer at least that large
int kgv_reserve(kgv_ctx*, uint8_t** buf, size_t* cap, size_t need) {
  g_need = need;
  if (*cap >= need && *buf) return KGV_OK;
  free(*buf);
  *cap = al256(need) + 256;
  *buf = (uint8_t*)aligned_alloc(256, *cap);
  return *buf ? KGV_OK : KGV_ERR_NOMEM;
}

struct Arr {
  const char* name;
  const void* p;
  size_t bytes;  // elements * size + pad
};

int main() {
  uint8_t* buf = nullptr;
  size_t cap = 0;
  for (size_t n : {0, 1, 7, 33, 1000}) {
    uint8_t* a;
    uint64_t* b;
    uint32_t* z;
    double* d;
    uint16_t* e;
    uint32_t* z2;
    uint8_t* f;
    size_t end = 0;
    auto lay = [&](kgv_carve& c) {
      a = c.take<uint8_t>(n + 3);
      b = c.take<uint64_t>(n);
      z = c.take<uint32_t>(0);
      d = c.take<double>(2 * n, 40);
      e = c.take<uint16_t>(n, 7);
      z2 = c.take<uint32_t>(0, 0);
      f = c.take<uint8_t>(1, 255);
      end = c.at;
    };
    kgv_carve m;
    lay(m);
    const bool null_measure = !a && !b && !z && !d && !e && !z2 && !f;
    const size_t measured = m.at;
    if (kgv_reserve_carved(nullptr, &buf, &cap, lay) != KGV_OK) return 1;
    const Arr arr[] = {{"a", a, n + 3}, {"b", b, 8 * n}, {"z", z, 0}, {"d", d, 16 * n + 40}, {"e", e, 2 * n + 7}, {"z2", z2, 0}, {"f", f, 256}};
    printf("layout %zu %zu %zu %zu %d\n", n, measured, g_need, end, null_measure ? 1 : 0);
    for (const Arr& x : arr) printf("array %s %td %zu\n", x.name, (const uint8_t*)x.p - buf, x.bytes);
  }
  free(buf);
  return 0;
}
