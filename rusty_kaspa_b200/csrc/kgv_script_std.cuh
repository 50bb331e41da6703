// kgv_script_std.cuh — the three standard script classes, evaluated exactly as the reference's
// script engine would evaluate these shapes, but split into data-parallel phases:
//   plan    : per input, recognise the shape and lay out the signature checks it may need
//   (batch) : sighash + Schnorr/ECDSA verification of every candidate (sig, key) pair
//   resolve : per input, replay the engine's sequential logic over the pair verdicts
//
// Reference semantics followed (crypto/txscript/src):
//   lib.rs:399-449   execute: spk version > 0 accepts; sigscript push-only; P2SH save/restore stack
//   lib.rs:456-470   final stack must be exactly one truthy element (else EvalFalse)
//   lib.rs:488-571   CHECKMULTISIG: in-order key matching, early fail when keys run out, NullFail
//   lib.rs:574-643   check_*_signature: sig-op budget first, then lengths, then parse, then verify
//   opcodes/mod.rs:746-808  CHECKSIG(ECDSA): last signature byte is the hash type (InvalidSigHashType)
//   opcodes/mod.rs:141-190  minimal (canonical) push encodings
//   script_class.rs:58-82, standard/multisig.rs:18-70  the shapes themselves
// Any input that is not exactly one of these shapes is reported as KGV_SCRIPT_NONSTANDARD: the
// host script VM (csrc/host) decides it, so verdicts stay bit-exact for arbitrary scripts.
#pragma once
#include "../../include/kgv.h"
#include "kgv_blake2b.cuh"

namespace kgv {

enum : uint8_t { CLS_NONSTANDARD = 0, CLS_ACCEPT_VERSION = 1, CLS_P2PK = 2, CLS_P2PK_ECDSA = 3, CLS_MULTISIG = 4, CLS_MULTISIG_ECDSA = 5 };

// device-side populated entry: the script stays where it lives (batch arena or UTXO table slot)
struct DevEntry {
  uint64_t amount;
  uint64_t block_daa_score;
  const uint8_t* script;
  uint32_t script_len;
  uint16_t spk_version;
  uint8_t is_coinbase;
  uint8_t found;
};

struct InputPlan {
  uint32_t item_base;    // first item of this input in its (Schnorr or ECDSA) item list
  uint32_t redeem_off;   // multisig: offset of the redeem script inside the signature script
  uint16_t redeem_len;
  uint8_t cls;
  uint8_t m, n;          // multisig: required signatures, keys
  uint8_t n_items;       // 1 for P2PK, m*(n-m+1) for multisig
  uint8_t pad_[2];
};

KGV_HD bool sighash_type_allowed(uint32_t t) { return t == 1 || t == 2 || t == 4 || t == 0x81 || t == 0x82 || t == 0x84; }

// the next opcode of sc[0..n) at pos as parse_script deserialises it (opcodes/macros.rs:9-61): op, and its pushed data at sc[doff..doff+dlen)
// (dlen 0 for every opcode that is not OP_DATA_1..75 / OP_PUSHDATA1/2/4, OP_0 and OP_1..OP_16 included); pos moves past both.  Returns 0,
// or KGV_SCRIPT_MALFORMED_PUSH_SIZE / KGV_SCRIPT_MALFORMED_PUSH when the length bytes or the data run past the end - the last opcode then.
KGV_HD uint8_t script_next_op(const uint8_t* sc, uint32_t n, uint32_t& pos, uint32_t& op, uint32_t& doff, uint32_t& dlen) {
  op = sc[pos++];
  doff = pos; dlen = 0;
  if (op >= 0x01 && op <= 0x4b) {
    if (n - pos < op) return KGV_SCRIPT_MALFORMED_PUSH;
    dlen = op;
  } else if (op >= 0x4c && op <= 0x4e) {
    const uint32_t lb = op == 0x4c ? 1 : op == 0x4d ? 2 : 4;
    if (n - pos < lb) return KGV_SCRIPT_MALFORMED_PUSH_SIZE;
    uint64_t l = 0;
    for (uint32_t i = 0; i < lb; i++) l |= (uint64_t)sc[pos + i] << (8 * i);
    pos += lb;
    if ((uint64_t)(n - pos) < l) return KGV_SCRIPT_MALFORMED_PUSH;
    doff = pos; dlen = (uint32_t)l;
  }
  pos += dlen;
  return 0;
}

// one canonical direct data push at p[0..n): returns bytes consumed (0 if not canonical), data offset/len relative to p
KGV_HD uint32_t canonical_push(const uint8_t* p, uint32_t n, uint32_t& doff, uint32_t& dlen) {
  if (n == 0) return 0;
  uint32_t op = p[0];
  if (op >= 1 && op <= 75) {
    if (n < 1 + op) return 0;
    if (op == 1 && ((p[1] >= 1 && p[1] <= 16) || p[1] == 0x81)) return 0;
    doff = 1; dlen = op;
    return 1 + op;
  }
  if (op == 0x4c) {
    if (n < 2) return 0;
    uint32_t l = p[1];
    if (l <= 75 || n < 2 + l) return 0;
    doff = 2; dlen = l;
    return 2 + l;
  }
  if (op == 0x4d) {
    if (n < 3) return 0;
    uint32_t l = (uint32_t)p[1] | ((uint32_t)p[2] << 8);
    if (l <= 255 || n < 3 + l) return 0;
    doff = 3; dlen = l;
    return 3 + l;
  }
  return 0;
}

// Recognise the shape of one input. ss = signature script, e = the spent entry.
KGV_HD void plan_input(InputPlan& pl, const uint8_t* ss, uint32_t ss_len, const DevEntry& e) {
  pl.item_base = 0; pl.redeem_off = 0; pl.redeem_len = 0; pl.m = 0; pl.n = 0; pl.n_items = 0; pl.cls = CLS_NONSTANDARD;
  pl.pad_[0] = pl.pad_[1] = 0;
  if (e.spk_version > 0) { pl.cls = CLS_ACCEPT_VERSION; return; }
  const uint8_t* spk = e.script;
  uint32_t sl = e.script_len;
  if ((sl == 34 && spk[0] == 0x20 && spk[33] == 0xac) || (sl == 35 && spk[0] == 0x21 && spk[34] == 0xab)) {
    if (!(ss_len == 66 && ss[0] == 0x41)) return;
    pl.cls = sl == 34 ? CLS_P2PK : CLS_P2PK_ECDSA;
    pl.n_items = 1;
    return;
  }
  if (!(sl == 35 && spk[0] == 0xaa && spk[1] == 0x20 && spk[34] == 0x87)) return;
  // P2SH: m pushes of 65 bytes, then the canonical push of a standard multisig redeem script
  uint32_t off = 0, nsig = 0, roff = 0, rlen = 0;
  bool have = false;
  while (off < ss_len) {
    uint32_t doff, dlen;
    uint32_t used = canonical_push(ss + off, ss_len - off, doff, dlen);
    if (!used) return;
    if (off + used == ss_len) { roff = off + doff; rlen = dlen; have = true; break; }
    if (dlen != 65 || nsig == 20) return;
    nsig++;
    off += used;
  }
  if (!have || rlen < 3 || rlen > 520) return;
  const uint8_t* rd = ss + roff;
  uint32_t last = rd[rlen - 1];
  if (last != 0xae && last != 0xa9) return;
  bool ecdsa = last == 0xa9;
  if (rd[0] < 0x51 || rd[0] > 0x60) return;
  uint32_t m = rd[0] - 0x50, klen = ecdsa ? 33 : 32, nkeys = 0, p = 1;
  while (p < rlen - 2) {
    if (rd[p] != klen || p + 1 + klen > rlen - 2 || nkeys == 20) return;
    nkeys++;
    p += 1 + klen;
  }
  if (p != rlen - 2) return;
  uint32_t opn = rd[rlen - 2];
  if (opn < 0x51 || opn > 0x60 || opn - 0x50 != nkeys || m > nkeys || m != nsig) return;
  pl.cls = ecdsa ? CLS_MULTISIG_ECDSA : CLS_MULTISIG;
  pl.m = (uint8_t)m; pl.n = (uint8_t)nkeys;
  pl.n_items = (uint8_t)(m * (nkeys - m + 1));  // <= 10*11 = 110
  pl.redeem_off = roff; pl.redeem_len = (uint16_t)rlen;
}

// Location of the (sig, key) pair of item k of an input: signature i may only be matched against
// keys i .. n-m+i (lib.rs:540-547), so item k = i*(n-m+1) + (j-i).
KGV_HD void item_location(const InputPlan& pl, uint32_t k, const uint8_t* ss, const DevEntry& e, const uint8_t*& sig65, const uint8_t*& key) {
  if (pl.cls == CLS_P2PK || pl.cls == CLS_P2PK_ECDSA) {
    sig65 = ss + 1;
    key = e.script + 1;
    return;
  }
  uint32_t w = pl.n - pl.m + 1;
  uint32_t i = k / w, j = i + k % w;
  uint32_t klen = pl.cls == CLS_MULTISIG_ECDSA ? 33u : 32u;
  sig65 = ss + 66u * i + 1;
  key = ss + pl.redeem_off + 1 + (1 + klen) * j + 1;
}

// Replay of the engine over the pair verdicts st[0..n_items) (KGV_SIG_* codes). Returns a KGV_SCRIPT_* code.
KGV_HD uint32_t resolve_input(const InputPlan& pl, const uint8_t* ss, const DevEntry& e, uint32_t sig_op_count, const uint8_t* st) {
  if (pl.cls == CLS_ACCEPT_VERSION) return KGV_SCRIPT_OK;
  if (pl.cls == CLS_NONSTANDARD) return KGV_SCRIPT_NONSTANDARD;
  uint32_t remaining = sig_op_count;
  if (pl.cls == CLS_P2PK || pl.cls == CLS_P2PK_ECDSA) {
    if (!sighash_type_allowed(ss[65])) return KGV_SCRIPT_INVALID_SIGHASH_TYPE;
    if (remaining == 0) return KGV_SCRIPT_EXCEEDED_SIGOP_LIMIT;
    uint32_t v = st[0];
    if (v == KGV_SIG_PK_PARSE_ERR || v == KGV_SIG_SIG_PARSE_ERR) return KGV_SCRIPT_INVALID_SIGNATURE;
    return v == KGV_SIG_VALID ? KGV_SCRIPT_OK : KGV_SCRIPT_EVAL_FALSE;
  }
  // P2SH: BLAKE2b-256(redeem) must equal the hash in the spk, else the first stage ends false
  Blake2b hs;
  b2b_init(hs, B2B_UNKEYED);
  b2b_bytes(hs, ss + pl.redeem_off, pl.redeem_len);
  uint64_t d[4];
  b2b_final(hs, d);
  bool eq = true;
  for (int w = 0; w < 4; w++)
    for (int b = 0; b < 8; b++) eq = eq && ((uint8_t)(d[w] >> (8 * b)) == e.script[2 + 8 * w + b]);
  if (!eq) return KGV_SCRIPT_EVAL_FALSE;
  uint32_t m = pl.m, n = pl.n, w = n - m + 1, ki = 0;
  bool failed = false;
  for (uint32_t si = 0; si < m && !failed; si++) {
    if (!sighash_type_allowed(ss[66u * si + 65])) return KGV_SCRIPT_INVALID_SIGHASH_TYPE;
    for (;;) {
      if (n - ki < m - si) { failed = true; break; }
      uint32_t j = ki++;
      if (remaining == 0) return KGV_SCRIPT_EXCEEDED_SIGOP_LIMIT;
      remaining--;
      // j is within [si, n-m+si] here (ki >= si always, and the guard above bounds it from above)
      uint32_t v = st[si * w + (j - si)];
      if (v == KGV_SIG_PK_PARSE_ERR || v == KGV_SIG_SIG_PARSE_ERR) return KGV_SCRIPT_INVALID_SIGNATURE;
      if (v == KGV_SIG_VALID) break;
    }
  }
  return failed ? KGV_SCRIPT_NULL_FAIL : KGV_SCRIPT_OK;
}

// ---- per-transaction context rules (tx_validation_in_utxo_context.rs:75-155, mass/mod.rs:64-80,338-410)
KGV_HD uint64_t utxo_plurality(uint32_t script_len) { return (63ull + script_len + 99ull) / 100ull; }
KGV_HD bool ck_mul(uint64_t a, uint64_t b, uint64_t& r) {  // true on overflow (u64::checked_mul): the high half of the 128-bit product decides, no division
  r = a * b;
#if defined(__CUDA_ARCH__)
  return __umul64hi(a, b) != 0;
#else
  return (uint64_t)(((unsigned __int128)a * b) >> 64) != 0;
#endif
}
KGV_HD bool ck_add(uint64_t a, uint64_t b, uint64_t& r) { r = a + b; return r < a; }
KGV_HD uint64_t sat_add(uint64_t a, uint64_t b) { uint64_t r = a + b; return r < a ? ~0ull : r; }
KGV_HD uint64_t sat_sub(uint64_t a, uint64_t b) { return a > b ? a - b : 0; }

// returns false if the storage mass is incomputable
template <class EntryAt, class OutputAt>
KGV_HD bool storage_mass(uint64_t& mass, bool coinbase, uint32_t n_in, uint32_t n_out, EntryAt entry_at, OutputAt output_at, uint64_t C) {
  if (coinbase) { mass = 0; return true; }
  uint64_t outs_plur = 0, harm_outs = 0;
  for (uint32_t i = 0; i < n_out; i++) {
    uint64_t value; uint32_t slen;
    output_at(i, value, slen);
    uint64_t p = utxo_plurality(slen), v;
    outs_plur += p;
    if (ck_mul(C, p, v) || ck_mul(v, p, v)) return false;
    if (value == 0) return false;
    if (ck_add(harm_outs, v / value, harm_outs)) return false;
  }
  bool relaxed;
  if (outs_plur == 1) relaxed = true;
  else if (n_in > 2) relaxed = false;
  else {
    uint64_t ip = 0;
    for (uint32_t i = 0; i < n_in; i++) ip += utxo_plurality(entry_at(i).script_len);
    relaxed = ip == 1 || (outs_plur == 2 && ip == 2);
  }
  if (relaxed) {
    uint64_t harm_ins = 0;
    for (uint32_t i = 0; i < n_in; i++) {
      const DevEntry& e = entry_at(i);
      uint64_t p = utxo_plurality(e.script_len);
      if (e.amount == 0) return false;
      harm_ins = sat_add(harm_ins, C * p * p / e.amount);
    }
    mass = sat_sub(harm_outs, harm_ins);
    return true;
  }
  uint64_t ins_plur = 0, sum_ins = 0;
  for (uint32_t i = 0; i < n_in; i++) { ins_plur += utxo_plurality(entry_at(i).script_len); sum_ins += entry_at(i).amount; }
  if (ins_plur == 0) return false;
  uint64_t mean = sum_ins / ins_plur;
  if (mean == 0) return false;
  uint64_t q = C / mean, prod;
  mass = sat_sub(harm_outs, ck_mul(ins_plur, q, prod) ? ~0ull : prod);
  return true;
}

}  // namespace kgv
