"""Derives the two cSHAKE256 start states of kHeavyHash (NIST SP 800-185, section 3.3) and prints them as the constants of
rusty_kaspa_b200/csrc/kgv_keccak.cuh.

cSHAKE256(X, L, N = "", S) absorbs bytepad(encode_string(N) || encode_string(S), 136) || X, then pads with the two-bit suffix 00 and
pad10*1.  The first part is one full 136-byte block that does not depend on X, so it is absorbed once here.  A message of fixed length
then fits in the next block: the device XORs its words into the start state and runs one permutation.  The padding of that block,
0x04 at the message length and 0x80 at byte 135, is folded into the constant as well.

  "ProofOfWorkHash": message = pre_pow_hash (32) || timestamp u64 || 32 zero bytes || nonce u64 = 80 bytes
  "HeavyHash":       message = 32 bytes

    python tools/derive_cshake_states.py        # prints the C table
"""
RATE = 136
MASK = (1 << 64) - 1

_RC = [0x0000000000000001, 0x0000000000008082, 0x800000000000808A, 0x8000000080008000, 0x000000000000808B, 0x0000000080000001,
       0x8000000080008081, 0x8000000000008009, 0x000000000000008A, 0x0000000000000088, 0x0000000080008009, 0x000000008000000A,
       0x000000008000808B, 0x800000000000008B, 0x8000000000008089, 0x8000000000008003, 0x8000000000008002, 0x8000000000000080,
       0x000000000000800A, 0x800000008000000A, 0x8000000080008081, 0x8000000000008080, 0x0000000080000001, 0x8000000080008008]
# rotation offsets r[x][y] of the rho step (FIPS 202, 3.2.2), lane index x + 5y
_ROT = [[0, 36, 3, 41, 18], [1, 44, 10, 45, 2], [62, 6, 43, 15, 61], [28, 55, 25, 21, 56], [27, 20, 39, 8, 14]]


def _rol(v, r):
    return ((v << r) | (v >> (64 - r))) & MASK if r else v


def keccak_f1600(a):
    """The 24-round permutation on 25 u64 lanes (lane x + 5y), in place; returns a."""
    for rc in _RC:
        c = [a[x] ^ a[x + 5] ^ a[x + 10] ^ a[x + 15] ^ a[x + 20] for x in range(5)]
        d = [c[(x - 1) % 5] ^ _rol(c[(x + 1) % 5], 1) for x in range(5)]
        for i in range(25):
            a[i] ^= d[i % 5]
        b = [0] * 25
        for x in range(5):
            for y in range(5):
                b[y + 5 * ((2 * x + 3 * y) % 5)] = _rol(a[x + 5 * y], _ROT[x][y])
        for y in range(5):
            row = b[5 * y:5 * y + 5]
            for x in range(5):
                a[x + 5 * y] = row[x] ^ ((~row[(x + 1) % 5]) & row[(x + 2) % 5])
        a[0] ^= rc
    return a


def left_encode(x):
    n = max(1, (x.bit_length() + 7) // 8)
    return bytes([n]) + x.to_bytes(n, "big")


def encode_string(s):
    return left_encode(8 * len(s)) + s


def bytepad(x, w):
    z = left_encode(w) + x
    return z + bytes((-len(z)) % w)


def absorb(state, block):
    for i in range(len(block) // 8):
        state[i] ^= int.from_bytes(block[8 * i:8 * i + 8], "little")


def cshake256_start_state(custom, msg_len):
    """State a fixed-length message of msg_len (< 136) bytes is XORed into (little-endian words) before the one permutation that
    yields cSHAKE256(msg, N = "", S = custom)."""
    prefix = bytepad(encode_string(b"") + encode_string(custom), RATE)
    st = [0] * 25
    for k in range(0, len(prefix), RATE):
        absorb(st, prefix[k:k + RATE])
        keccak_f1600(st)
    st[msg_len // 8] ^= 0x04 << (8 * (msg_len % 8))
    st[(RATE - 1) // 8] ^= 0x80 << (8 * ((RATE - 1) % 8))
    return st


POW_STATE = ("ProofOfWorkHash", 80)
HEAVY_STATE = ("HeavyHash", 32)


def derive():
    return {name: cshake256_start_state(name.encode(), n) for name, n in (POW_STATE, HEAVY_STATE)}


def c_table(name, words):
    rows = ["    " + ", ".join("0x%016xull" % w for w in words[k:k + 5]) + "," for k in range(0, 25, 5)]
    return "KGV_CONST_TABLE uint64_t %s[25] = {\n%s\n};" % (name, "\n".join(rows))


if __name__ == "__main__":
    s = derive()
    print("// cSHAKE256(N = \"\", S = \"ProofOfWorkHash\"), 80-byte message, padding folded in")
    print(c_table("kPowHashStart", s["ProofOfWorkHash"]))
    print("// cSHAKE256(N = \"\", S = \"HeavyHash\"), 32-byte message, padding folded in")
    print(c_table("kHeavyHashStart", s["HeavyHash"]))
