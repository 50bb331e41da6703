// Host build of the standardness rule bodies (kgv_standard.cuh) for GPU-less tests (TEST BUILD ONLY): the same functions the kernels of
// kgv_standard.cu call, over scripts laid out in one arena (script k at arena[off[k] .. off[k] + len[k])).
#include "../../rusty_kaspa_b200/csrc/kgv_standard.cuh"
using namespace kgv;

extern "C" {
// per script: out[k] = class | unspendable << 2 | (p2sh sig-op bound of the script taken as a signature script) << 8,
// ops[k] = the sig-op count of the script's own opcodes
void hs_scripts(const uint8_t* arena, const uint64_t* off, const uint32_t* len, const uint16_t* version, size_t n, uint64_t* out, uint64_t* ops) {
  for (size_t k = 0; k < n; k++) {
    const uint8_t* s = arena + off[k];
    out[k] = script_class(version[k], s, len[k]) | (uint64_t)script_is_unspendable(s, len[k]) << 2 | p2sh_sig_op_bound(s, len[k]) << 8;
    ops[k] = script_sig_ops(s, len[k]);
  }
}
// is_transaction_output_dust of output k (value[k], script k) at relay fee fee[k]
void hs_dust(const uint8_t* arena, const uint64_t* off, const uint32_t* len, const uint64_t* value, const uint64_t* fee, size_t n, uint8_t* out) {
  for (size_t k = 0; k < n; k++) out[k] = output_is_dust(value[k], arena + off[k], len[k], fee[k]);
}
// minimum_required_transaction_relay_fee: out[k] = the fee, ok[k] = 0 where mass * fee overflows
void hs_min_fee(const uint64_t* mass, const uint64_t* fee, size_t n, uint64_t* out, uint8_t* ok) {
  for (size_t k = 0; k < n; k++) ok[k] = min_relay_fee(mass[k], fee[k], out[k]);
}
}
