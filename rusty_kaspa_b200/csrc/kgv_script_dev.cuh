// kgv_script_dev.cuh — the full script engine, one input per thread: a restatement of execute_input of the host engine
// (csrc/host/kgv_script_vm.cpp, itself pinned by the reference's script corpus) with the same check order and the same
// ScriptErr for every input.  KGV_HD: compiled by nvcc for the device and by g++ for tests/hostsim.
//
// Stack items are views, not copies (SItem): a pointer into bytes that stay immutable for the whole call (sigscript, spk,
// redeem script, output scripts, the per-input heap), or up to 8 bytes held inline (numbers, booleans, small-int pushes),
// optionally behind a 2-byte big-endian version prefix (OpTxInputSpk / OpTxOutputSpk).  DUP / PICK / OVER copy 16 bytes.
//
// Scratch bound (per input, ScriptSlot, global memory — no dynamically indexed local arrays, DESIGN.md §6):
//   * stack: data + alt items.  The host engine checks |data| + |alt| <= 244 after every opcode, and one opcode adds at most
//     3 items (OP_3DUP), so at most 247 are live; the alt stack grows down from the top of the same array.
//   * heap: only OP_SHA256 / OP_BLAKE2B make bytes that are neither a view nor inline (32 B each).  They are non-push opcodes, and
//     run_script stops a script at its 202nd such opcode (num_ops > MAX_OPS_PER_SCRIPT).  The sigscript is push-only (no
//     hashing); a P2SH spk is the fixed 35-byte shape with exactly one OP_BLAKE2B; the redeem script (or a plain spk) hashes at
//     most 201 times.  Plus one slot for a redeem script that was an inline item (a small-int push): 203 slots.
//   * condition stack: each OP_IF / OP_NOTIF is a counted opcode and the stack must be empty at the end of each script: <= 201.
// Signature checks read a per-input verdict log (2 bits per check, KGV_SIG_*): check k reads verdict k.  When the log runs out
// the engine writes the request (hash type, kind, key, signature) and stops with SE_NEEDS; re-running from the start with a longer
// log is deterministic.  Every check consumes one unit of the input's sig_op_count first, so an input makes at most 255 checks.
#pragma once
#include "../../include/kgv.h"
#include "kgv_blake2b.cuh"
#include "kgv_sha256.cuh"
#include "kgv_txhash.cuh"

#if defined(__CUDACC__)
#define KGV_SE_CALL static __device__ __noinline__
#else
#define KGV_SE_CALL static inline
#endif

namespace kgv {

enum : uint32_t {
  SE_STACK_CAP = 248, SE_COND_CAP = 204, SE_HEAP_SLOTS = 203, SE_LOG_BYTES = 64,
  SE_MAX_STACK = 244, SE_MAX_SCRIPT = 10000, SE_MAX_ELEMENT = 520, SE_MAX_OPS = 201, SE_MAX_KEYS = 20,
};
enum : uint8_t { SE_NEEDS = 254, SE_PENDING = 254, SE_SKIPPED = 253, SE_OVERFLOW = 252 };
enum : uint32_t { SI_INLINE = 1, SI_PREFIX = 2 };

struct SItem {
  uint64_t w;    // pointer, or the inline bytes (little-endian: byte i = w >> 8i)
  uint32_t len;  // bytes behind the prefix
  uint32_t fl;   // SI_*; with SI_PREFIX the version is in bits 16..31
};
struct ScriptSlot {
  SItem stk[SE_STACK_CAP];
  uint8_t heap[SE_HEAP_SLOTS][32];
  uint8_t cond[SE_COND_CAP];  // 0 false, 1 true, 2 skip
};
struct ScriptReq {  // the check an input is waiting for
  uint8_t hash_type, ecdsa, pad_[2];
  uint8_t key[33];
  uint8_t sig[64];
  uint8_t pad2_[3];
};

KGV_HD SItem si_inline(uint64_t w, uint32_t len) { SItem s; s.w = w; s.len = len; s.fl = SI_INLINE; return s; }
KGV_HD SItem si_view(const uint8_t* p, uint32_t len) { SItem s; s.w = (uint64_t)(uintptr_t)p; s.len = len; s.fl = 0; return s; }
KGV_HD uint32_t si_len(const SItem& a) { return a.len + ((a.fl & SI_PREFIX) ? 2u : 0u); }
KGV_HD uint32_t si_byte(const SItem& a, uint32_t i) {
  if (a.fl & SI_INLINE) return (uint32_t)(a.w >> (8 * i)) & 0xffu;
  if (a.fl & SI_PREFIX) {
    if (i == 0) return a.fl >> 24;
    if (i == 1) return (a.fl >> 16) & 0xffu;
    i -= 2;
  }
  return ((const uint8_t*)(uintptr_t)a.w)[i];
}
KGV_HD bool si_bool(const SItem& a) {  // data_stack.rs:206-214
  const uint32_t n = si_len(a);
  if (n == 0) return false;
  if (si_byte(a, n - 1) & 0x7f) return true;
  for (uint32_t i = 0; i + 1 < n; i++)
    if (si_byte(a, i)) return true;
  return false;
}
KGV_SE_CALL bool si_equal(SItem a, SItem b) {
  const uint32_t n = si_len(a);
  if (n != si_len(b)) return false;
  for (uint32_t i = 0; i < n; i++)
    if (si_byte(a, i) != si_byte(b, i)) return false;
  return true;
}
// serialize_i64 (data_stack.rs:109-137) into an inline item; false when it needs more than 8 bytes (SerializationError)
KGV_HD bool si_num(int64_t x, SItem& out) {
  const bool neg = x < 0;
  uint64_t p = neg ? (uint64_t)0 - (uint64_t)x : (uint64_t)x, w = 0;
  uint32_t n = 0;
  bool last_sat = false;
  while (p) {
    if (n == 8) return false;
    const uint64_t b = p & 0xff;
    last_sat = (b & 0x80) != 0;
    w |= b << (8 * n++);
    p >>= 8;
  }
  if (last_sat) {
    if (n == 8) return false;
    n++;
  }
  if (neg) w |= (uint64_t)0x80 << (8 * (n - 1));
  out = si_inline(w, n);
  return true;
}
// SizedEncodeInt<LEN>::deserialize (data_stack.rs:177-190)
KGV_HD uint8_t si_to_num(const SItem& v, uint32_t maxlen, int64_t& out) {
  const uint32_t n = si_len(v);
  if (n > maxlen) return KGV_SCRIPT_NUMBER_TOO_BIG;
  if (n > 8) return KGV_SCRIPT_NOT_MINIMAL_DATA;
  if (n == 0) { out = 0; return KGV_SCRIPT_OK; }
  const uint32_t msb = si_byte(v, n - 1);
  if ((msb & 0x7f) == 0 && (n == 1 || (si_byte(v, n - 2) & 0x80) == 0)) return KGV_SCRIPT_NOT_MINIMAL_DATA;
  int64_t acc = msb & 0x7f;
  for (uint32_t i = n - 1; i-- > 0;) acc = (int64_t)(((uint64_t)acc << 8) + si_byte(v, i));
  out = (msb & 0x80) ? -acc : acc;
  return KGV_SCRIPT_OK;
}
// SHA-256 / unkeyed BLAKE2b-256 of an item into 32 bytes
KGV_SE_CALL void si_sha256(SItem a, uint8_t* out) {
  uint32_t st[8] = {0x6a09e667u, 0xbb67ae85u, 0x3c6ef372u, 0xa54ff53au, 0x510e527fu, 0x9b05688cu, 0x1f83d9abu, 0x5be0cd19u};
  const uint32_t n = si_len(a), total = (n + 9 + 63) / 64 * 64;
  const uint64_t bits = (uint64_t)n * 8;
  for (uint32_t off = 0; off < total; off += 64) {
    uint32_t w[16];
#pragma unroll
    for (int i = 0; i < 16; i++) {
      uint32_t v = 0;
#pragma unroll
      for (int k = 0; k < 4; k++) {
        const uint32_t pos = off + 4 * i + k;
        uint32_t c;
        if (pos < n) c = si_byte(a, pos);
        else if (pos == n) c = 0x80;
        else if (pos >= total - 8) c = (uint32_t)(bits >> (8 * (total - 1 - pos))) & 0xff;
        else c = 0;
        v = (v << 8) | c;
      }
      w[i] = v;
    }
    sha256_compress(st, w);
  }
#pragma unroll
  for (int i = 0; i < 8; i++) { out[4 * i] = (uint8_t)(st[i] >> 24); out[4 * i + 1] = (uint8_t)(st[i] >> 16); out[4 * i + 2] = (uint8_t)(st[i] >> 8); out[4 * i + 3] = (uint8_t)st[i]; }
}
KGV_SE_CALL void si_blake2b(SItem a, uint8_t* out) {
  Blake2b h;
  b2b_init(h, B2B_UNKEYED);
  if (a.fl & SI_INLINE) {
    for (uint32_t i = 0; i < a.len; i++) b2b_byte(h, si_byte(a, i));
  } else {
    if (a.fl & SI_PREFIX) { b2b_byte(h, a.fl >> 24); b2b_byte(h, (a.fl >> 16) & 0xff); }
    b2b_bytes(h, (const uint8_t*)(uintptr_t)a.w, a.len);
  }
  uint64_t d[4];
  b2b_final(h, d);
#pragma unroll
  for (int i = 0; i < 32; i++) out[i] = (uint8_t)(d[i / 8] >> (8 * (i % 8)));
}

KGV_HD bool se_sighash_type_ok(uint32_t t) { return t == 1 || t == 2 || t == 4 || t == 0x81 || t == 0x82 || t == 0x84; }
KGV_HD bool se_is_disabled(uint32_t op) {
  switch (op) { case 0x7e: case 0x7f: case 0x80: case 0x81: case 0x83: case 0x84: case 0x85: case 0x86: case 0x8d: case 0x8e:
                case 0x95: case 0x96: case 0x97: case 0x98: case 0x99: return true; default: return false; }
}
KGV_HD uint8_t se_minimal_push(uint32_t op, const uint8_t* d, uint32_t n) {  // opcodes/mod.rs:141-190
  if (n == 0) return op != 0x00 ? KGV_SCRIPT_NOT_MINIMAL_DATA : KGV_SCRIPT_OK;
  if (n == 1 && d[0] >= 1 && d[0] <= 16) return op != 0x51u + d[0] - 1 ? KGV_SCRIPT_NOT_MINIMAL_DATA : KGV_SCRIPT_OK;
  if (n == 1 && d[0] == 0x81) return op != 0x4f ? KGV_SCRIPT_NOT_MINIMAL_DATA : KGV_SCRIPT_OK;
  if (n <= 75) return op != n ? KGV_SCRIPT_NOT_MINIMAL_DATA : KGV_SCRIPT_OK;
  if (n <= 255) return op != 0x4c ? KGV_SCRIPT_NOT_MINIMAL_DATA : KGV_SCRIPT_OK;
  if (n < 65535 && op != 0x4d) return KGV_SCRIPT_NOT_MINIMAL_DATA;
  return KGV_SCRIPT_OK;
}
KGV_HD bool se_add_ovf(int64_t a, int64_t b, int64_t& r) {
  r = (int64_t)((uint64_t)a + (uint64_t)b);
  return (a >= 0) == (b >= 0) && (r >= 0) != (a >= 0);
}
KGV_HD bool se_sub_ovf(int64_t a, int64_t b, int64_t& r) {
  r = (int64_t)((uint64_t)a - (uint64_t)b);
  return (a >= 0) != (b >= 0) && (r >= 0) != (a >= 0);
}

struct DevScriptEngine {
  const BatchView* b;
  const kgv_tx* t;
  const kgv_input* in;
  uint32_t idx;          // input index within the tx
  ScriptSlot* s;
  uint32_t nd, na, nc, heap;
  int num_ops;
  uint32_t sigops_remaining;
  const uint8_t* log;    // verdict log of this input (2 bits per check)
  uint32_t n_log, n_checks;
  ScriptReq* req;

  KGV_HD bool executing() const { return nc == 0 || s->cond[nc - 1] == 1; }
  KGV_HD SItem& top(uint32_t k = 0) { return s->stk[nd - 1 - k]; }
  KGV_HD uint8_t push(const SItem& x) {
    if (nd + na >= SE_STACK_CAP) return SE_OVERFLOW;  // unreachable by the bound above; reported as an internal error
    s->stk[nd++] = x;
    return KGV_SCRIPT_OK;
  }
  KGV_HD uint8_t push_num(int64_t x) {
    SItem v;
    if (!si_num(x, v)) return KGV_SCRIPT_SERIALIZATION;
    return push(v);
  }
  KGV_HD uint8_t push_bool(bool v) { return push(si_inline(v ? 1 : 0, v ? 1 : 0)); }
  KGV_HD uint8_t pop_nums(uint32_t n, uint32_t maxlen, int64_t& x0, int64_t& x1, int64_t& x2) {  // items bottom-first
    if (nd < n) return KGV_SCRIPT_INVALID_STACK_OPERATION;
    nd -= n;
    uint8_t e = si_to_num(s->stk[nd], maxlen, x0);
    if (e || n < 2) return e;
    if ((e = si_to_num(s->stk[nd + 1], maxlen, x1)) || n < 3) return e;
    return si_to_num(s->stk[nd + 2], maxlen, x2);
  }
  KGV_HD uint8_t pop_num(uint32_t maxlen, int64_t& x) { int64_t u, v; return pop_nums(1, maxlen, x, u, v); }
  KGV_HD uint8_t pop_bool(bool& v) {
    if (nd == 0) return KGV_SCRIPT_INVALID_STACK_OPERATION;
    v = si_bool(s->stk[--nd]);
    return KGV_SCRIPT_OK;
  }
  KGV_HD uint8_t* alloc32() { return heap < SE_HEAP_SLOTS ? s->heap[heap++] : nullptr; }

  // check_schnorr/ecdsa_signature (lib.rs:574-643): verdicts come from the log
  KGV_HD uint8_t check_sig(uint32_t hash_type, const SItem& key, const SItem& sig, uint32_t siglen, bool ecdsa, bool& valid) {
    if (sigops_remaining == 0) return KGV_SCRIPT_EXCEEDED_SIGOP_LIMIT;
    sigops_remaining--;
    if (siglen != 64) return KGV_SCRIPT_SIG_LENGTH;
    if (si_len(key) != (ecdsa ? 33u : 32u)) return KGV_SCRIPT_PUBKEY_FORMAT;
    const uint32_t k = n_checks++;
    if (k >= n_log) {
      req->hash_type = (uint8_t)hash_type;
      req->ecdsa = ecdsa ? 1 : 0;
      for (uint32_t i = 0; i < 33; i++) req->key[i] = i < si_len(key) ? (uint8_t)si_byte(key, i) : 0;
      for (uint32_t i = 0; i < 64; i++) req->sig[i] = (uint8_t)si_byte(sig, i);
      return SE_NEEDS;
    }
    const uint32_t v = (log[k >> 2] >> (2 * (k & 3))) & 3u;
    if (v == KGV_SIG_PK_PARSE_ERR || v == KGV_SIG_SIG_PARSE_ERR) return KGV_SCRIPT_INVALID_SIGNATURE;
    valid = v == KGV_SIG_VALID;
    return KGV_SCRIPT_OK;
  }

  KGV_HD uint8_t op_checksig(bool ecdsa) {  // opcodes/mod.rs:746-790
    if (nd < 2) return KGV_SCRIPT_INVALID_STACK_OPERATION;
    const SItem key = s->stk[nd - 1], sig = s->stk[nd - 2];
    nd -= 2;
    const uint32_t sl = si_len(sig);
    if (sl == 0) return push_bool(false);
    const uint32_t typ = si_byte(sig, sl - 1);
    if (!se_sighash_type_ok(typ)) return KGV_SCRIPT_INVALID_SIGHASH_TYPE;
    bool valid = false;
    const uint8_t e = check_sig(typ, key, sig, sl - 1, ecdsa, valid);
    if (e) return e;
    return push_bool(valid);
  }
  KGV_HD uint8_t op_checkmultisig(bool ecdsa) {  // lib.rs:488-571
    int64_t nk, ns;
    uint8_t e = pop_num(4, nk);
    if (e) return e;
    if (nk < 0 || nk > SE_MAX_KEYS) return KGV_SCRIPT_INVALID_PUBKEY_COUNT;
    num_ops += (int)nk;
    if (num_ops > (int)SE_MAX_OPS) return KGV_SCRIPT_TOO_MANY_OPERATIONS;
    if (nd < (uint32_t)nk) return KGV_SCRIPT_INVALID_STACK_OPERATION;
    nd -= (uint32_t)nk;
    const uint32_t kbase = nd;  // keys[i] = stk[kbase + i]; nothing is pushed before the result
    if ((e = pop_num(4, ns))) return e;
    if (ns < 0 || ns > nk) return KGV_SCRIPT_INVALID_SIGNATURE_COUNT;
    if (nd < (uint32_t)ns) return KGV_SCRIPT_INVALID_STACK_OPERATION;
    nd -= (uint32_t)ns;
    const uint32_t sbase = nd, nsig = (uint32_t)ns, nkey = (uint32_t)nk;
    bool failed = false;
    uint32_t ki = 0;
    for (uint32_t si = 0; si < nsig && !failed; si++) {
      const SItem sg = s->stk[sbase + si];
      const uint32_t sl = si_len(sg);
      if (sl == 0) { failed = true; break; }
      const uint32_t typ = si_byte(sg, sl - 1);
      if (!se_sighash_type_ok(typ)) return KGV_SCRIPT_INVALID_SIGHASH_TYPE;
      for (;;) {
        if (nkey - ki < nsig - si) { failed = true; break; }
        const SItem key = s->stk[kbase + ki++];
        bool valid = false;
        if ((e = check_sig(typ, key, sg, sl - 1, ecdsa, valid))) return e;
        if (valid) break;
      }
    }
    if (failed) {
      for (uint32_t si = 0; si < nsig; si++)
        if (si_len(s->stk[sbase + si])) return KGV_SCRIPT_NULL_FAIL;
    }
    return push_bool(!failed);
  }
  KGV_HD uint8_t push_spk(uint16_t version, const uint8_t* script, uint32_t n) {  // lib.rs:645-653
    SItem v = si_view(script, n);
    v.fl = SI_PREFIX | ((uint32_t)version << 16);
    return push(v);
  }
  KGV_HD uint8_t verify_top() { bool v; uint8_t e = pop_bool(v); if (e) return e; return v ? KGV_SCRIPT_OK : KGV_SCRIPT_VERIFY; }

  KGV_HD uint8_t exec(uint32_t op, const uint8_t* data, uint32_t dlen) {
    int64_t a = 0, b2 = 0, c = 0, r = 0;
    uint8_t e;
    if (op == 0x00) return push(si_inline(0, 0));
    if (op <= 0x4e) return push(si_view(data, dlen));
    if (op == 0x4f) return push_num(-1);
    if (op >= 0x51 && op <= 0x60) return push_num((int64_t)op - 0x50);
    switch (op) {
      case 0x50: case 0x62: case 0x65: case 0x66: case 0x89: case 0x8a: return KGV_SCRIPT_OPCODE_RESERVED;
      case 0x61: return KGV_SCRIPT_OK;
      case 0x63: case 0x64: {  // OpIf / OpNotIf
        uint8_t cv = 2;
        if (executing()) {
          if (nd == 0) return KGV_SCRIPT_EMPTY_STACK;
          const SItem buf = s->stk[--nd];
          const uint32_t n = si_len(buf);
          if (n > 1) return KGV_SCRIPT_EXPECTED_BOOLEAN;
          bool truth;
          if (n == 0) truth = false;
          else if (si_byte(buf, 0) == 1) truth = true;
          else return KGV_SCRIPT_EXPECTED_BOOLEAN;
          cv = (truth == (op == 0x63)) ? 1 : 0;
        }
        if (nc >= SE_COND_CAP) return SE_OVERFLOW;
        s->cond[nc++] = cv;
        return KGV_SCRIPT_OK;
      }
      case 0x67: if (nc == 0) return KGV_SCRIPT_COND_STACK_EMPTY; if (s->cond[nc - 1] != 2) s->cond[nc - 1] ^= 1; return KGV_SCRIPT_OK;
      case 0x68: if (nc == 0) return KGV_SCRIPT_COND_STACK_EMPTY; nc--; return KGV_SCRIPT_OK;
      case 0x69: return verify_top();
      case 0x6a: return KGV_SCRIPT_EARLY_RETURN;
      case 0x6b:  // OpToAltStack
        if (nd == 0) return KGV_SCRIPT_INVALID_STACK_OPERATION;
        if (nd + na >= SE_STACK_CAP) return SE_OVERFLOW;
        s->stk[SE_STACK_CAP - 1 - na++] = s->stk[--nd];
        return KGV_SCRIPT_OK;
      case 0x6c:  // OpFromAltStack
        if (na == 0) return KGV_SCRIPT_EMPTY_STACK;
        return push(s->stk[SE_STACK_CAP - na--]);
      case 0x6d: if (nd < 2) return KGV_SCRIPT_INVALID_STACK_OPERATION; nd -= 2; return KGV_SCRIPT_OK;
      case 0x6e: case 0x6f: case 0x76: {  // 2DUP 3DUP DUP
        const uint32_t k = op == 0x6e ? 2 : op == 0x6f ? 3 : 1;
        if (nd < k) return KGV_SCRIPT_INVALID_STACK_OPERATION;
        for (uint32_t i = 0; i < k; i++) if ((e = push(s->stk[nd - k]))) return e;
        return KGV_SCRIPT_OK;
      }
      case 0x70: case 0x78: {  // 2OVER OVER
        const uint32_t k = op == 0x70 ? 2 : 1;
        if (nd < 2 * k) return KGV_SCRIPT_INVALID_STACK_OPERATION;
        for (uint32_t i = 0; i < k; i++) if ((e = push(s->stk[nd - 2 * k]))) return e;
        return KGV_SCRIPT_OK;
      }
      case 0x71: case 0x7b: {  // 2ROT ROT: the k items at depth 3k..2k move to the top
        const uint32_t k = op == 0x71 ? 2 : 1;
        if (nd < 3 * k) return KGV_SCRIPT_INVALID_STACK_OPERATION;
        for (uint32_t i = 0; i < k; i++) {
          const uint32_t from = nd - 3 * k;
          const SItem x = s->stk[from];
          for (uint32_t j = from; j + 1 < nd; j++) s->stk[j] = s->stk[j + 1];
          s->stk[nd - 1] = x;
        }
        return KGV_SCRIPT_OK;
      }
      case 0x72: case 0x7c: {  // 2SWAP SWAP
        const uint32_t k = op == 0x72 ? 2 : 1;
        if (nd < 2 * k) return KGV_SCRIPT_INVALID_STACK_OPERATION;
        for (uint32_t i = 0; i < k; i++) {
          const SItem x = s->stk[nd - 2 * k + i];
          s->stk[nd - 2 * k + i] = s->stk[nd - k + i];
          s->stk[nd - k + i] = x;
        }
        return KGV_SCRIPT_OK;
      }
      case 0x73: if (nd == 0) return KGV_SCRIPT_INVALID_STACK_OPERATION; if (si_bool(top())) return push(top()); return KGV_SCRIPT_OK;
      case 0x74: return push_num((int64_t)nd);
      case 0x75: if (nd == 0) return KGV_SCRIPT_INVALID_STACK_OPERATION; nd--; return KGV_SCRIPT_OK;
      case 0x77: if (nd < 2) return KGV_SCRIPT_INVALID_STACK_OPERATION; s->stk[nd - 2] = s->stk[nd - 1]; nd--; return KGV_SCRIPT_OK;
      case 0x79: case 0x7a: {  // PICK ROLL
        if ((e = pop_num(4, a))) return e;
        if (a < 0 || (uint64_t)a >= nd) return op == 0x79 ? KGV_SCRIPT_PICK_INVALID : KGV_SCRIPT_ROLL_INVALID;
        const uint32_t pos = nd - (uint32_t)a - 1;
        const SItem x = s->stk[pos];
        if (op == 0x7a) {
          for (uint32_t j = pos; j + 1 < nd; j++) s->stk[j] = s->stk[j + 1];
          nd--;
        }
        return push(x);
      }
      case 0x7d: {  // TUCK
        if (nd < 2) return KGV_SCRIPT_INVALID_STACK_OPERATION;
        const SItem x = s->stk[nd - 1], y = s->stk[nd - 2];
        s->stk[nd - 2] = x; s->stk[nd - 1] = y;
        return push(x);
      }
      case 0x7e: case 0x7f: case 0x80: case 0x81: case 0x83: case 0x84: case 0x85: case 0x86: case 0x8d: case 0x8e:
      case 0x95: case 0x96: case 0x97: case 0x98: case 0x99: return KGV_SCRIPT_OPCODE_DISABLED;
      case 0x82: if (nd == 0) return KGV_SCRIPT_INVALID_STACK_OPERATION; return push_num((int64_t)si_len(top()));
      case 0x87: case 0x88: {
        if (nd < 2) return KGV_SCRIPT_INVALID_STACK_OPERATION;
        const bool eq = si_equal(s->stk[nd - 1], s->stk[nd - 2]);
        nd -= 2;
        if (op == 0x87) return push_bool(eq);
        return eq ? KGV_SCRIPT_OK : KGV_SCRIPT_VERIFY;
      }
      case 0x8b: if ((e = pop_num(8, a))) return e; if (a == INT64_MAX) return KGV_SCRIPT_NUMBER_TOO_BIG; return push_num(a + 1);
      case 0x8c: if ((e = pop_num(8, a))) return e; if (a == INT64_MIN) return KGV_SCRIPT_NUMBER_TOO_BIG; return push_num(a - 1);
      case 0x8f: if ((e = pop_num(8, a))) return e; if (a == INT64_MIN) return KGV_SCRIPT_NUMBER_TOO_BIG; return push_num(-a);
      case 0x90: if ((e = pop_num(8, a))) return e; if (a == INT64_MIN) return KGV_SCRIPT_NUMBER_TOO_BIG; return push_num(a < 0 ? -a : a);
      case 0x91: if ((e = pop_num(8, a))) return e; return push_num(a == 0);
      case 0x92: if ((e = pop_num(8, a))) return e; return push_num(a != 0);
      case 0x93: if ((e = pop_nums(2, 8, a, b2, c))) return e; if (se_add_ovf(a, b2, r)) return KGV_SCRIPT_NUMBER_TOO_BIG; return push_num(r);
      case 0x94: if ((e = pop_nums(2, 8, a, b2, c))) return e; if (se_sub_ovf(a, b2, r)) return KGV_SCRIPT_NUMBER_TOO_BIG; return push_num(r);
      case 0x9a: if ((e = pop_nums(2, 8, a, b2, c))) return e; return push_num(a != 0 && b2 != 0);
      case 0x9b: if ((e = pop_nums(2, 8, a, b2, c))) return e; return push_num(a != 0 || b2 != 0);
      case 0x9c: if ((e = pop_nums(2, 8, a, b2, c))) return e; return push_num(a == b2);
      case 0x9d: if ((e = pop_nums(2, 8, a, b2, c))) return e; return a == b2 ? KGV_SCRIPT_OK : KGV_SCRIPT_VERIFY;
      case 0x9e: if ((e = pop_nums(2, 8, a, b2, c))) return e; return push_num(a != b2);
      case 0x9f: if ((e = pop_nums(2, 8, a, b2, c))) return e; return push_num(a < b2);
      case 0xa0: if ((e = pop_nums(2, 8, a, b2, c))) return e; return push_num(a > b2);
      case 0xa1: if ((e = pop_nums(2, 8, a, b2, c))) return e; return push_num(a <= b2);
      case 0xa2: if ((e = pop_nums(2, 8, a, b2, c))) return e; return push_num(a >= b2);
      case 0xa3: if ((e = pop_nums(2, 8, a, b2, c))) return e; return push_num(a < b2 ? a : b2);
      case 0xa4: if ((e = pop_nums(2, 8, a, b2, c))) return e; return push_num(a > b2 ? a : b2);
      case 0xa5: if ((e = pop_nums(3, 8, a, b2, c))) return e; return push_num(a >= b2 && a < c);
      case 0xa8: case 0xaa: {  // OpSHA256 / OpBlake2b
        if (nd == 0) return KGV_SCRIPT_INVALID_STACK_OPERATION;
        const SItem x = s->stk[--nd];
        uint8_t* out = alloc32();
        if (!out) return SE_OVERFLOW;
        if (op == 0xa8) si_sha256(x, out);
        else si_blake2b(x, out);
        return push(si_view(out, 32));
      }
      case 0xa9: return op_checkmultisig(true);
      case 0xab: return op_checksig(true);
      case 0xac: return op_checksig(false);
      case 0xad: if ((e = op_checksig(false))) return e; return verify_top();
      case 0xae: return op_checkmultisig(false);
      case 0xaf: if ((e = op_checkmultisig(false))) return e; return verify_top();
      case 0xb0: case 0xb1: {  // CLTV / CSV (opcodes/mod.rs:816-908)
        if (nd == 0) return KGV_SCRIPT_INVALID_STACK_OPERATION;
        const SItem x = s->stk[--nd];
        const uint32_t n = si_len(x);
        if (n > 8) return KGV_SCRIPT_NUMBER_TOO_BIG;
        uint64_t v = 0;
        for (uint32_t i = n; i-- > 0;) v = (v << 8) | si_byte(x, i);
        if (op == 0xb0) {
          const uint64_t LT = 500000000000ull;
          const bool both_lo = t->lock_time < LT && v < LT, both_hi = t->lock_time >= LT && v >= LT;
          if (!(both_lo || both_hi)) return KGV_SCRIPT_UNSATISFIED_LOCKTIME;
          if (v > t->lock_time) return KGV_SCRIPT_UNSATISFIED_LOCKTIME;
          if (in->sequence == ~0ull) return KGV_SCRIPT_UNSATISFIED_LOCKTIME;
          return KGV_SCRIPT_OK;
        }
        const uint64_t DIS = 1ull << 63, MASK = 0xffffffffull;
        if (v & DIS) return KGV_SCRIPT_OK;
        if (in->sequence & DIS) return KGV_SCRIPT_UNSATISFIED_LOCKTIME;
        if ((v & MASK) > (in->sequence & MASK)) return KGV_SCRIPT_UNSATISFIED_LOCKTIME;
        return KGV_SCRIPT_OK;
      }
      case 0xb2: case 0xb5: case 0xb6: case 0xb7: case 0xb8: case 0xba: case 0xbb: case 0xbc: case 0xbd: case 0xc0: case 0xc1: return KGV_SCRIPT_OPCODE_RESERVED;
      case 0xb3: return push_num((int64_t)t->n_inputs);
      case 0xb4: return push_num((int64_t)t->n_outputs);
      case 0xb9: return push_num((int64_t)idx);
      case 0xbe: case 0xbf: {  // OpTxInputAmount / OpTxInputSpk
        if ((e = pop_num(4, a))) return e;
        if (a < 0 || (uint64_t)a >= t->n_inputs) return KGV_SCRIPT_INVALID_INPUT_INDEX;
        const DevEntry& u = b->entries[t->first_input + (uint32_t)a];
        if (op == 0xbe) { if (u.amount > (uint64_t)INT64_MAX) return KGV_SCRIPT_NUMBER_TOO_BIG; return push_num((int64_t)u.amount); }
        return push_spk(u.spk_version, u.script, u.script_len);
      }
      case 0xc2: case 0xc3: {  // OpTxOutputAmount / OpTxOutputSpk
        if ((e = pop_num(4, a))) return e;
        if (a < 0 || (uint64_t)a >= t->n_outputs) return KGV_SCRIPT_INVALID_OUTPUT_INDEX;
        const kgv_output& o = b->outputs[t->first_output + (uint32_t)a];
        if (op == 0xc2) { if (o.value > (uint64_t)INT64_MAX) return KGV_SCRIPT_NUMBER_TOO_BIG; return push_num((int64_t)o.value); }
        return push_spk(o.spk_version, b->bytes + o.script_off, o.script_len);
      }
      default: return KGV_SCRIPT_INVALID_OPCODE;  // 0xa6 0xa7 0xc4..0xff
    }
  }

  // execute_script (lib.rs:363-397)
  KGV_HD uint8_t run_script(const uint8_t* sc, uint32_t n, bool verify_only_push) {
    uint8_t res = KGV_SCRIPT_OK;
    uint32_t pos = 0;
    while (pos < n) {
      uint32_t op, doff, dlen;
      if ((res = script_next_op(sc, n, pos, op, doff, dlen))) break;  // macros.rs:9-61 (kgv_script_std.cuh)
      const uint8_t* data = op >= 0x01 && op <= 0x4e ? sc + doff : nullptr;
      if (se_is_disabled(op)) { res = KGV_SCRIPT_OPCODE_DISABLED; break; }
      if (op == 0x65 || op == 0x66) { res = KGV_SCRIPT_OPCODE_RESERVED; break; }
      if (verify_only_push && op > 0x60) { res = KGV_SCRIPT_NOT_PUSH_ONLY; break; }
      if (op > 0x60) {  // execute_opcode (lib.rs:322-344)
        if (++num_ops > (int)SE_MAX_OPS) { res = KGV_SCRIPT_TOO_MANY_OPERATIONS; break; }
      } else if (dlen > SE_MAX_ELEMENT) { res = KGV_SCRIPT_ELEMENT_TOO_BIG; break; }
      if (executing() || (op >= 0x63 && op <= 0x68)) {
        if (op > 0 && op <= 0x4e) { res = se_minimal_push(op, data, dlen); if (res) break; }
        res = exec(op, data, dlen);
        if (res) break;
      }
      if (na + nd > SE_MAX_STACK) { res = KGV_SCRIPT_STACK_SIZE_EXCEEDED; break; }
    }
    if (res == KGV_SCRIPT_OK && nc != 0) return KGV_SCRIPT_UNBALANCED_CONDITIONAL;
    na = 0;
    num_ops = 0;
    return res;
  }
  KGV_HD uint8_t check_error_condition(bool final_script) {  // lib.rs:456-470
    if (final_script) {
      if (nd > 1) return KGV_SCRIPT_CLEAN_STACK;
      if (nd == 0) return KGV_SCRIPT_EMPTY_STACK;
    }
    bool v;
    const uint8_t e = pop_bool(v);
    if (e) return e;
    return v ? KGV_SCRIPT_OK : KGV_SCRIPT_EVAL_FALSE;
  }
  // execute (lib.rs:399-449)
  KGV_HD uint8_t execute(const DevEntry& entry) {
    if (entry.spk_version > 0) return KGV_SCRIPT_OK;
    const uint8_t* ss = b->bytes + in->sigscript_off;
    const uint32_t ssl = in->sigscript_len;
    const uint8_t* spk = entry.script;
    const uint32_t spkl = entry.script_len;
    if (ssl == 0 && spkl == 0) return KGV_SCRIPT_EVAL_FALSE;
    if (ssl > SE_MAX_SCRIPT || spkl > SE_MAX_SCRIPT) return KGV_SCRIPT_SCRIPT_SIZE;
    const bool p2sh = spkl == 35 && spk[0] == 0xaa && spk[1] == 0x20 && spk[34] == 0x87;
    uint8_t e;
    if (ssl && (e = run_script(ss, ssl, true))) return e;
    // The host engine saves the whole stack before a P2SH spk and restores it after.  The spk is exactly
    // OP_BLAKE2B <32 bytes> OP_EQUAL, which only replaces the top item and pushes above it, so keeping the depth and
    // the top item is the same restore.
    const uint32_t saved_nd = nd;
    SItem saved_top = si_inline(0, 0);
    if (p2sh && nd) saved_top = top();
    if (spkl && (e = run_script(spk, spkl, false))) return e;
    if (p2sh) {
      if ((e = check_error_condition(false))) return e;
      nd = saved_nd;
      if (nd == 0) return KGV_SCRIPT_EMPTY_STACK;
      s->stk[nd - 1] = saved_top;
      SItem sc = s->stk[--nd];
      if (sc.fl & SI_INLINE) {  // a small-int push: give the redeem script bytes of its own
        uint8_t* p = alloc32();
        if (!p) return SE_OVERFLOW;
        for (uint32_t i = 0; i < sc.len; i++) p[i] = (uint8_t)si_byte(sc, i);
        sc = si_view(p, sc.len);
      }
      if ((e = run_script((const uint8_t*)(uintptr_t)sc.w, sc.len, false))) return e;
    }
    return check_error_condition(true);
  }
};

// One input from the start: returns a KGV_SCRIPT_* code, SE_NEEDS (request written to *req) or SE_OVERFLOW.
KGV_HD uint8_t script_run_input(const BatchView& b, uint32_t tx, uint32_t in_abs, ScriptSlot* slot, const uint8_t* log, uint32_t n_log, ScriptReq* req) {
  DevScriptEngine g;
  g.b = &b;
  g.t = &b.txs[tx];
  g.in = &b.inputs[in_abs];
  g.idx = in_abs - g.t->first_input;
  g.s = slot;
  g.nd = g.na = g.nc = g.heap = 0;
  g.num_ops = 0;
  g.sigops_remaining = g.in->sig_op_count;
  g.log = log;
  g.n_log = n_log;
  g.n_checks = 0;
  g.req = req;
  return g.execute(b.entries[in_abs]);
}

}  // namespace kgv
