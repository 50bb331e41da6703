"""CPU restatement of header validation in isolation (test infrastructure, never the thing under test):
  consensus/core/src/hashing/header.rs:7-35          block hash / pre-PoW hash (keyed BLAKE2b "BlockHash")
  consensus/pow/src/xoshiro.rs, matrix.rs           xoshiro256++, the 64x64 nibble matrix, compute_rank, heavy_hash
  crypto/hashes/src/pow_hashers.rs                  cSHAKE256 "ProofOfWorkHash" / "HeavyHash" (start states from tools/derive_cshake_states.py)
  math/src/lib.rs:64-79, uint.rs:67-84              Uint256::from_compact_target_bits and its shift (modulo 256 in a release build)
  consensus/pow/src/lib.rs:56-75                    calc_block_level_check_pow, calc_level_from_pow
  consensus/src/pipeline/header_processor/pre_ghostdag_validation.rs:17-24,30-68,102-106   the isolation rules, in order

A header is a dict: version, parents_by_level (expanded: list of lists of 32-byte hashes), hash_merkle_root, accepted_id_merkle_root,
utxo_commitment, timestamp, bits, nonce, daa_score, blue_score, blue_work (int), pruning_point.  Pure Python: a header costs ~15 ms
(mostly the rank), so bulk comparisons use the C restatement (tests/oracle_pow/ok_pow.c)."""
import hashlib
import os
import struct
import sys

sys.path.insert(0, os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "tools"))
import derive_cshake_states as dcs  # noqa: E402

MASK = (1 << 64) - 1
_STATES = dcs.derive()
POW_START, HEAVY_START = _STATES["ProofOfWorkHash"], _STATES["HeavyHash"]
ORIGIN = b"\xfe" * 32

# statuses (KGV_HEADER_* in include/kgv.h)
OK, WRONG_BLOCK_VERSION, TIME_TOO_FAR_INTO_THE_FUTURE, NO_PARENTS, TOO_MANY_PARENTS, ORIGIN_PARENT, INVALID_POW = range(7)
SKIP_POW = 1


def serialize(h, nonce=None, timestamp=None):
    """The bytes hash_override_nonce_time feeds the hasher."""
    out = [struct.pack("<H", h["version"]), struct.pack("<Q", len(h["parents_by_level"]))]
    for lvl in h["parents_by_level"]:
        out.append(struct.pack("<Q", len(lvl)))
        out.extend(lvl)
    bw = h["blue_work"].to_bytes(24, "big").lstrip(b"\0")
    out += [h["hash_merkle_root"], h["accepted_id_merkle_root"], h["utxo_commitment"],
            struct.pack("<QIQQQ", h["timestamp"] if timestamp is None else timestamp, h["bits"], h["nonce"] if nonce is None else nonce,
                        h["daa_score"], h["blue_score"]),
            struct.pack("<Q", len(bw)), bw, h["pruning_point"]]
    return b"".join(out)


def block_hash(h, nonce=None, timestamp=None):
    return hashlib.blake2b(serialize(h, nonce, timestamp), digest_size=32, key=b"BlockHash").digest()


def pre_pow_hash(h):
    return block_hash(h, 0, 0)


def _words(b32):
    return list(struct.unpack("<4Q", b32))


def _squeeze(st):
    return b"".join(w.to_bytes(8, "little") for w in st[:4])


def pow_hash(pre_pow, timestamp, nonce):
    st = list(POW_START)
    for i, w in enumerate(_words(pre_pow)):
        st[i] ^= w
    st[4] ^= timestamp
    st[9] ^= nonce
    return _squeeze(dcs.keccak_f1600(st))


def kheavy_hash(b32):
    st = list(HEAVY_START)
    for i, w in enumerate(_words(b32)):
        st[i] ^= w
    return _squeeze(dcs.keccak_f1600(st))


class Xoshiro:
    def __init__(self, seed32):
        self.s = _words(seed32)

    def u64(self):
        s0, s1, s2, s3 = self.s
        rl = lambda v, r: ((v << r) | (v >> (64 - r))) & MASK
        res = (s0 + rl((s0 + s3) & MASK, 23)) & MASK
        t = (s1 << 17) & MASK
        s2 ^= s0
        s3 ^= s1
        s1 ^= s2
        s0 ^= s3
        s2 ^= t
        s3 = rl(s3, 45)
        self.s = [s0, s1, s2, s3]
        return res


def rand_matrix(gen):
    m = []
    for _ in range(64):
        row = []
        for _ in range(4):
            v = gen.u64()
            row += [(v >> (4 * k)) & 0xF for k in range(16)]
        m.append(row)
    return m


def compute_rank(m):
    """matrix.rs compute_rank, operation for operation (Python floats are IEEE doubles, and nothing here fuses)."""
    eps = 1e-9
    a = [[float(x) for x in row] for row in m]
    rank, sel = 0, [False] * 64
    for i in range(64):
        j = 0
        while j < 64 and not (not sel[j] and abs(a[j][i]) > eps):
            j += 1
        if j != 64:
            rank += 1
            sel[j] = True
            for p in range(i + 1, 64):
                a[j][p] /= a[j][i]
            for k in range(64):
                if k != j and abs(a[k][i]) > eps:
                    for p in range(i + 1, 64):
                        a[k][p] -= a[j][p] * a[k][i]
    return rank


def generate_matrix(seed32):
    """Matrix::generate: returns (matrix, tries)."""
    gen, tries = Xoshiro(seed32), 0
    while True:
        m = rand_matrix(gen)
        tries += 1
        if compute_rank(m) == 64:
            return m, tries


def heavy_hash(m, h32):
    vec = []
    for b in h32:
        vec += [b >> 4, b & 0xF]
    prod = bytearray(32)
    for i in range(32):
        s1 = sum(m[2 * i][j] * vec[j] for j in range(64)) & 0xFFFF
        s2 = sum(m[2 * i + 1][j] * vec[j] for j in range(64)) & 0xFFFF
        prod[i] = ((((s1 >> 10) << 4) | (s2 >> 10)) & 0xFF) ^ h32[i]
    return kheavy_hash(bytes(prod))


def compact_target(bits):
    """Uint256::from_compact_target_bits; the shift by 8 * (exponent - 3) wraps modulo 256 (uint.rs overflowing_shl)."""
    e = bits >> 24
    if e <= 3:
        mant, sh = (bits & 0xFFFFFF) >> (8 * (3 - e)), 0
    else:
        mant, sh = bits & 0xFFFFFF, 8 * (e - 3)
    if mant > 0x7FFFFF:
        return 0
    return (mant << (sh % 256)) & ((1 << 256) - 1)


def level_from_pow(pow_value, max_block_level):
    return max(max_block_level - pow_value.bit_length(), 0)


def check_pow(h, max_block_level, matrix=None):
    """(pre_pow_hash, pow value (int), passed, level) as calc_block_level_check_pow (genesis: max level, passed) and State::check_pow."""
    pre = pre_pow_hash(h)
    m = matrix if matrix is not None else generate_matrix(pre)[0]
    pw = int.from_bytes(heavy_hash(m, pow_hash(pre, h["timestamp"], h["nonce"])), "little")
    if not h["parents_by_level"]:
        return pre, pw, True, max_block_level
    return pre, pw, pw <= compact_target(h["bits"]), level_from_pow(pw, max_block_level)


def validate_in_isolation(h, rules, pow_result=None):
    """validate_header_in_isolation with now_ms given: (status, a, b, level, passed).  rules: dict block_version, max_block_parents,
    max_block_level, timestamp_deviation_tolerance, now_ms, flags."""
    _, _, passed, level = pow_result if pow_result is not None else check_pow(h, rules["max_block_level"])
    if h["version"] != rules["block_version"]:
        return WRONG_BLOCK_VERSION, h["version"], 0, level, passed
    max_time = (rules["now_ms"] + rules["timestamp_deviation_tolerance"] * 1000) & MASK
    if h["timestamp"] > max_time:
        return TIME_TOO_FAR_INTO_THE_FUTURE, h["timestamp"], max_time, level, passed
    direct = h["parents_by_level"][0] if h["parents_by_level"] else []
    if not direct:
        return NO_PARENTS, 0, 0, level, passed
    if len(direct) > rules["max_block_parents"]:
        return TOO_MANY_PARENTS, len(direct), rules["max_block_parents"], level, passed
    if any(p == ORIGIN for p in direct):
        return ORIGIN_PARENT, 0, 0, level, passed
    if not passed and not (rules["flags"] & SKIP_POW):
        return INVALID_POW, 0, 0, level, passed
    return OK, 0, 0, level, passed


# ---- the C restatement (tests/oracle_pow/ok_pow.c) and the host build of the device code (tests/hostsim/hostsim_pow.cpp) ----
_TESTS = os.path.dirname(os.path.abspath(__file__))
_CSRC = os.path.join(os.path.dirname(_TESTS), "rusty_kaspa_b200", "csrc")


def _build(src, out, cmd, deps=()):
    import subprocess
    if not os.path.exists(out) or any(os.path.getmtime(d) > os.path.getmtime(out) for d in (src,) + tuple(deps)):
        subprocess.run(cmd, check=True, capture_output=True)
    return out


def c_oracle():
    import ctypes
    d = os.path.join(_TESTS, "oracle_pow")
    src, out = os.path.join(d, "ok_pow.c"), os.path.join(d, "libok_pow.so")
    lib = ctypes.CDLL(_build(src, out, ["gcc", "-O2", "-std=c11", "-fPIC", "-shared", "-pthread", "-o", out, src, "-lm"]))
    vp, u64, u32 = ctypes.c_void_p, ctypes.c_uint64, ctypes.c_uint32
    lib.ok_pow_validate_batch.argtypes = [vp, ctypes.c_size_t, vp, vp, vp, vp, vp, vp, vp, ctypes.c_int]
    lib.ok_pow_header_hash.argtypes = [vp, vp, vp, u64, u64, vp]
    lib.ok_pow_rank_u16.argtypes, lib.ok_pow_rank_u16.restype = [vp], u32
    lib.ok_pow_generate.argtypes, lib.ok_pow_generate.restype = [vp, vp], u32
    lib.ok_pow_heavy_hash.argtypes = [vp, vp, vp]
    lib.ok_pow_compact_target.argtypes = [u32, vp]
    lib.ok_keccak_f1600.argtypes = [vp]
    lib.ok_pow_grind.argtypes, lib.ok_pow_grind.restype = [vp, vp, vp, u64, u64, ctypes.POINTER(u64)], ctypes.c_int
    return lib


def hostsim():
    import ctypes
    d = os.path.join(_TESTS, "hostsim")
    src, out = os.path.join(d, "hostsim_pow.cpp"), os.path.join(d, "libhostsim_pow.so")
    hdrs = [os.path.join(_CSRC, f) for f in ("kgv_pow.cuh", "kgv_keccak.cuh", "kgv_blake2b.cuh", "kgv_muhash.cuh")]
    lib = ctypes.CDLL(_build(src, out, ["g++", "-O2", "-std=c++17", "-shared", "-fPIC", "-o", out, src], hdrs))
    vp, u64, u32 = ctypes.c_void_p, ctypes.c_uint64, ctypes.c_uint32
    lib.hs_keccak_f1600.argtypes = [vp]
    lib.hs_pow_hash.argtypes = [vp, u64, u64, vp]
    lib.hs_header_hash.argtypes = [vp, vp, vp, u64, u64, vp]
    lib.hs_rank.argtypes, lib.hs_rank.restype = [vp], u32
    lib.hs_generate.argtypes, lib.hs_generate.restype = [vp, vp], u32
    lib.hs_generate_scripted.argtypes, lib.hs_generate_scripted.restype = [vp, u32, vp], u32
    lib.hs_heavy_hash.argtypes = [vp, vp, vp]
    lib.hs_compact_target.argtypes = [u32, vp]
    lib.hs_validate.argtypes = [vp] * 7
    return lib


def oracle_validate(lib, batch, rules, threads=None):
    """The C restatement over a headers.HeaderBatch: (HEADER_RESULT_DTYPE[n], hashes, pow values, pre-PoW hashes), (n, 32) uint8 each."""
    import ctypes
    import numpy as np
    from rusty_kaspa_b200.headers import HEADER_RESULT_DTYPE
    n = len(batch)
    res = np.zeros(max(n, 1), dtype=HEADER_RESULT_DTYPE)
    hs, pw, pre = (np.zeros((max(n, 1), 32), dtype=np.uint8) for _ in range(3))
    par = batch.parents if batch.parents.size else np.zeros((1, 32), dtype=np.uint8)
    ll = batch.level_len if batch.level_len.size else np.zeros(1, dtype=np.uint32)
    lib.ok_pow_validate_batch(batch.headers.ctypes.data, n, par.ctypes.data, ll.ctypes.data, ctypes.addressof(rules), res.ctypes.data, hs.ctypes.data,
                              pw.ctypes.data, pre.ctypes.data, threads or os.cpu_count() or 1)
    return res[:n], hs[:n], pw[:n], pre[:n]


GOLDEN = os.path.join(_TESTS, "golden")
FIXTURES = ("goref_1060_blocks.json.gz", "headers_goref_notx_5000.json.gz", "headers_goref_custom_pruning_depth.json.gz")


def fixture_headers(name):
    from rusty_kaspa_b200.blocks_json import load_headers_json
    return load_headers_json(os.path.join(GOLDEN, name))


def fixture_rules(params, **kw):
    from rusty_kaspa_b200.headers import HeaderRules
    d = dict(timestamp_deviation_tolerance=params["timestamp_deviation_tolerance"], max_block_parents=params["blockrate"]["max_block_parents"],
             max_block_level=params["max_block_level"], now_ms=2**63, skip_pow=bool(params.get("skip_proof_of_work")))
    d.update(kw)
    return HeaderRules(**d)
