// kgv_standard.cuh — the rule bodies of the mempool's standardness policy, as KGV_HD functions (one script, one output, one number at a
// time) so that the host build (tests/hostsim/hostsim_standard.cpp) runs the same code as the kernels of kgv_standard.cu.
//
// Restates (reference paths):
//   ScriptClass::from_script                 crypto/txscript/src/script_class.rs:39-82
//   is_unspendable                           crypto/txscript/src/lib.rs:231-233
//   get_sig_op_count_upper_bound (P2SH)      crypto/txscript/src/lib.rs:176-226
//   is_transaction_output_dust               mining/src/mempool/check_transaction_standard.rs:116-163
//   minimum_required_transaction_relay_fee   mining/src/mempool/check_transaction_standard.rs:215-231
// Scripts are walked with script_next_op (kgv_script_std.cuh), the opcode deserialiser the device script engine uses: a parse error can
// only be a push running past the end, so it is always the last opcode of the walk.
#pragma once
#include "kgv_script_std.cuh"

namespace kgv {

constexpr uint64_t STD_MAX_P2SH_SIG_OPS = 15;             // MAX_STANDARD_P2SH_SIG_OPS
constexpr uint64_t STD_MAX_SIGNATURE_SCRIPT_SIZE = 1650;  // MAXIMUM_STANDARD_SIGNATURE_SCRIPT_SIZE
constexpr uint64_t STD_MAX_TRANSACTION_MASS = 100000;     // MAXIMUM_STANDARD_TRANSACTION_MASS
constexpr uint64_t STD_MAX_SOMPI = 29000000000ull * 100000000ull;
constexpr uint64_t STD_MAX_PUB_KEYS_PER_MULTISIG = 20;

enum : uint8_t { SCLASS_NONSTANDARD = 0, SCLASS_PUBKEY = 1, SCLASS_PUBKEY_ECDSA = 2, SCLASS_SCRIPT_HASH = 3 };

// ScriptClass::from_script: only version 0 scripts have a class, decided by their length and three bytes
KGV_HD uint8_t script_class(uint16_t version, const uint8_t* s, uint32_t n) {
  if (version != 0) return SCLASS_NONSTANDARD;
  if (n == 34 && s[0] == 0x20 && s[33] == 0xac) return SCLASS_PUBKEY;
  if (n == 35 && s[0] == 0x21 && s[34] == 0xab) return SCLASS_PUBKEY_ECDSA;
  if (n == 35 && s[0] == 0xaa && s[1] == 0x20 && s[34] == 0x87) return SCLASS_SCRIPT_HASH;
  return SCLASS_NONSTANDARD;
}

// is_unspendable: OP_RETURN as the first opcode, or a parse error anywhere
KGV_HD bool script_is_unspendable(const uint8_t* s, uint32_t n) {
  if (n && s[0] == 0x6a) return true;
  for (uint32_t pos = 0, op, doff, dlen; pos < n;)
    if (script_next_op(s, n, pos, op, doff, dlen)) return true;
  return false;
}

// a < b for the 128-bit products a1 * a2 and b1 * b2
KGV_HD bool mul128_less(uint64_t a1, uint64_t a2, uint64_t b1, uint64_t b2) {
#ifdef __CUDA_ARCH__
  const uint64_t ah = __umul64hi(a1, a2), bh = __umul64hi(b1, b2);
#else
  const uint64_t ah = (uint64_t)(((unsigned __int128)a1 * a2) >> 64), bh = (uint64_t)(((unsigned __int128)b1 * b2) >> 64);
#endif
  return ah < bh || (ah == bh && a1 * a2 < b1 * b2);
}

// is_transaction_output_dust.  floor(x / d) < f  <=>  x < f * d, so value * 1000 / (3 * size) < fee is compared as two exact 128-bit
// products: the reference's u64 path (value * 1000 fits) and its u128 path give the same answer.
KGV_HD bool output_is_dust(uint64_t value, const uint8_t* s, uint32_t n, uint64_t minimum_relay_transaction_fee) {
  if (script_is_unspendable(s, n)) return true;
  const uint64_t size = 8 + 2 + 8 + (uint64_t)n + 148;  // transaction_output_estimated_serialized_size + a P2PK input
  return mul128_less(value, 1000, minimum_relay_transaction_fee, 3 * size);
}

// get_sig_op_count_by_opcodes over the opcodes of s, stopping at the first parse error.  A multisig opcode counts the small integer
// before it (OP_1..OP_16), else 20 (also at position 0).  The reference's to_small_int asserts OP_1 <= op < OP_16 and so panics on
// OP_16; here OP_16 counts 16.
KGV_HD uint64_t script_sig_ops(const uint8_t* s, uint32_t n) {
  uint64_t c = 0;
  uint32_t prev = 0x100;  // no opcode before the first
  for (uint32_t pos = 0, op, doff, dlen; pos < n; prev = op) {
    if (script_next_op(s, n, pos, op, doff, dlen)) break;
    if (op == 0xac || op == 0xad || op == 0xab) c += 1;  // CHECKSIG, CHECKSIGVERIFY, CHECKSIGECDSA
    else if (op == 0xae || op == 0xaf || op == 0xa9)     // CHECKMULTISIG, CHECKMULTISIGVERIFY, CHECKMULTISIGECDSA
      c += prev >= 0x51 && prev <= 0x60 ? prev - 0x50 : STD_MAX_PUB_KEYS_PER_MULTISIG;
  }
  return c;
}

// get_sig_op_count_upper_bound for a P2SH entry: 0 unless the signature script is non-empty, parses and is push-only (every opcode
// <= 0x60); then the sig-ops of the data its last opcode pushes (empty for OP_0, OP_1NEGATE, OP_1..OP_16)
KGV_HD uint64_t p2sh_sig_op_bound(const uint8_t* ss, uint32_t n) {
  if (n == 0) return 0;
  uint32_t pos = 0, op, doff = 0, dlen = 0;
  while (pos < n)
    if (script_next_op(ss, n, pos, op, doff, dlen) || op > 0x60) return 0;
  return script_sig_ops(ss + doff, dlen);
}

// minimum_required_transaction_relay_fee: mass * fee / 1000, that or fee when it is 0, capped at MAX_SOMPI.  false when mass * fee
// overflows u64 (the reference's overflow check panics there).
KGV_HD bool min_relay_fee(uint64_t mass, uint64_t fee, uint64_t& out) {
  if (mass && fee > ~0ull / mass) return false;
  uint64_t m = mass * fee / 1000;
  if (m == 0) m = fee;
  out = m < STD_MAX_SOMPI ? m : STD_MAX_SOMPI;
  return true;
}

}  // namespace kgv
