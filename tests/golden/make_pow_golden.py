#!/usr/bin/env python3
"""Extracts the reference's proof-of-work known answers and two header-complete DAG fixtures into tests/golden/.

Run with a rusty-kaspa source tree at hand:
    python tests/golden/make_pow_golden.py <rusty-kaspa source tree>   (or set RUSTY_KASPA_SRC)
Sources, parsed at run time and recorded in the fixtures:
  consensus/pow/src/matrix.rs   test_generate_matrix (seed [42; 32] and the expected matrix), test_heavy_hash (its matrix, input and
                                expected hash), test_compute_rank (the zero matrix, the u16 matrix drawn from seed [42; 32] and the same
                                matrix with row 0 replaced by row 1, and the ranks asserted for them)
  testing/integration/testdata/dags_for_json_tests/{goref-notx-5000-blocks,goref_custom_pruning_depth}/blocks.json.gz
                                every header, all fields and the expanded parents_by_level as written, with its hash; the params line kept
Outputs: pow_kat.json, headers_goref_notx_5000.json.gz, headers_goref_custom_pruning_depth.json.gz.
"""
import gzip
import json
import os
import re
import sys

REF = sys.argv[1] if len(sys.argv) > 1 else os.environ.get("RUSTY_KASPA_SRC", "")
OUT = os.path.dirname(os.path.abspath(__file__))
MATRIX = "consensus/pow/src/matrix.rs"
DAGS = "testing/integration/testdata/dags_for_json_tests"
MASK = (1 << 64) - 1


def read(rel):
    with open(os.path.join(REF, rel)) as f:
        return f.read()


def lineno(src, needle):
    return src[:src.index(needle)].count("\n") + 1


def matrix_literal(src, fn):
    i = src.index("Matrix([", src.index(fn))
    body = src[i + len("Matrix(["):src.index("]);", i)]
    rows = [[int(x) for x in r.split(",") if x.strip()] for r in re.findall(r"\[([0-9,\s]+)\]", body)]
    assert len(rows) == 64 and all(len(r) == 64 for r in rows), fn
    return rows


def byte_literal(src, fn, name):
    i = src.index("[", src.index(name, src.index(fn)))
    b = [int(x) for x in src[i + 1:src.index("]", i)].split(",") if x.strip()]
    assert len(b) == 32, (fn, name)
    return bytes(b).hex()


def xoshiro_u64s(seed_byte, n):
    """XoShiRo256PlusPlus (consensus/pow/src/xoshiro.rs) seeded with Hash::from_bytes([seed_byte; 32]): what test_compute_rank draws."""
    s = [int.from_bytes(bytes([seed_byte] * 8), "little")] * 4
    rl = lambda v, r: ((v << r) | (v >> (64 - r))) & MASK
    out = []
    for _ in range(n):
        out.append((s[0] + rl((s[0] + s[3]) & MASK, 23)) & MASK)
        t = (s[1] << 17) & MASK
        s[2] ^= s[0]; s[3] ^= s[1]; s[1] ^= s[2]; s[0] ^= s[3]; s[2] ^= t; s[3] = rl(s[3], 45)
    return out


def kat():
    src = read(MATRIX)
    rank_fn = src[src.index("fn test_compute_rank"):src.index("fn test_heavy_hash")]
    # the asserted ranks and the mutation, read from the test rather than assumed
    asserted = [int(x) for x in re.findall(r"compute_rank\(\),\s*(\d+)\)", rank_fn)]
    assert asserted == [0, 64, 63] and "matrix.0[0] = matrix.0[1];" in rank_fn and "[42; 32]" in rank_fn and "rng.u64() as u16" in rank_fn
    vals = [v & 0xFFFF for v in xoshiro_u64s(42, 64 * 64)]
    full = [vals[64 * r:64 * r + 64] for r in range(64)]
    dup = [list(full[1])] + [list(r) for r in full[1:]]
    gen_fn = src[src.index("fn test_generate_matrix"):]
    assert "Hash::from_bytes([42; 32])" in gen_fn
    return {"source": {"file": MATRIX, "test_compute_rank": lineno(src, "fn test_compute_rank"), "test_heavy_hash": lineno(src, "fn test_heavy_hash"),
                       "test_generate_matrix": lineno(src, "fn test_generate_matrix")},
            "generate_matrix": {"seed": bytes([42] * 32).hex(), "matrix": matrix_literal(src, "fn test_generate_matrix")},
            "heavy_hash": {"matrix": matrix_literal(src, "fn test_heavy_hash"), "input": byte_literal(src, "fn test_heavy_hash", "let hash"),
                           "expected": byte_literal(src, "fn test_heavy_hash", "expected_hash")},
            "compute_rank": [{"name": "zero", "matrix": [[0] * 64 for _ in range(64)], "rank": asserted[0]},
                             {"name": "xoshiro_u16_seed42", "matrix": full, "rank": asserted[1]},
                             {"name": "row0_is_row1", "matrix": dup, "rank": asserted[2]}]}


def headers_only(rel, out):
    with gzip.open(os.path.join(REF, rel), "rt") as f:
        lines = [l for l in f.read().splitlines() if l.strip()]
    keep = [lines[0]] + [json.dumps({"header": json.loads(l)["header"]}, separators=(",", ":")) for l in lines[1:]]
    with gzip.GzipFile(os.path.join(OUT, out), "wb", compresslevel=9, mtime=0) as g:
        g.write(("\n".join(keep) + "\n").encode())
    return len(keep) - 1


if __name__ == "__main__":
    if not REF or not os.path.isdir(REF):
        sys.exit(__doc__)
    with open(os.path.join(OUT, "pow_kat.json"), "w") as f:
        json.dump(kat(), f, separators=(",", ":"))
        f.write("\n")
    for d, out in (("goref-notx-5000-blocks", "headers_goref_notx_5000.json.gz"), ("goref_custom_pruning_depth", "headers_goref_custom_pruning_depth.json.gz")):
        print(out, headers_only(os.path.join(DAGS, d, "blocks.json.gz"), out), "headers")
