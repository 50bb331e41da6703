#!/usr/bin/env python3
"""Extracts the reference's own cases for the mempool's standardness policy into tests/golden/standard_cases.json.

Run where the reference sources are available (the GPU machines do not have them):
    python tests/golden/make_standard_golden.py <rusty-kaspa source tree>   (or set RUSTY_KASPA_SRC)
Sources, parsed at run time and recorded in the fixture:
  mining/src/mempool/check_transaction_standard.rs  the three constants; test_calc_min_required_tx_relay_fee (8 rows),
                                                    test_is_transaction_output_dust (7 rows), test_check_transaction_standard_in_isolation
                                                    (7 named transactions, built as the test builds them)
  mining/src/mempool/config.rs                      the default relay fee and standard versions
  consensus/core/src/constants.rs                   TX_VERSION, MAX_SOMPI, SOMPI_PER_KASPA, MAX_SCRIPT_PUBLIC_KEY_VERSION
The generator asserts the names and counts it finds, so a change of those tests breaks it instead of silently shrinking the fixture.
"""
import json
import os
import re
import sys

REF = sys.argv[1] if len(sys.argv) > 1 else os.environ.get("RUSTY_KASPA_SRC", "")
OUT = os.path.dirname(os.path.abspath(__file__))
STD = "mining/src/mempool/check_transaction_standard.rs"
CFG = "mining/src/mempool/config.rs"
CONSTS = "consensus/core/src/constants.rs"
U64 = 2**64 - 1


def read(rel):
    with open(os.path.join(REF, rel)) as f:
        return f.read()


def lineno(src, needle):
    return src[:src.index(needle)].count("\n") + 1


def num(s):
    return int(s.replace("_", ""), 0)


def constants():
    std, cfg, con = read(STD), read(CFG), read(CONSTS)
    c = lambda src, name: re.search(r"const %s: \w+ = ([^;]+);" % name, src).group(1)
    tx_version = num(c(con, "TX_VERSION"))
    sompi = num(c(con, "SOMPI_PER_KASPA"))
    max_sompi = re.fullmatch(r"([\d_]+) \* SOMPI_PER_KASPA", c(con, "MAX_SOMPI"))
    assert c(cfg, "DEFAULT_MINIMUM_STANDARD_TRANSACTION_VERSION") == "TX_VERSION" and c(cfg, "DEFAULT_MAXIMUM_STANDARD_TRANSACTION_VERSION") == "TX_VERSION"
    return {"MAX_STANDARD_P2SH_SIG_OPS": num(c(std, "MAX_STANDARD_P2SH_SIG_OPS")),
            "MAXIMUM_STANDARD_SIGNATURE_SCRIPT_SIZE": num(c(std, "MAXIMUM_STANDARD_SIGNATURE_SCRIPT_SIZE")),
            "MAXIMUM_STANDARD_TRANSACTION_MASS": num(c(std, "MAXIMUM_STANDARD_TRANSACTION_MASS")),
            "DEFAULT_MINIMUM_RELAY_TRANSACTION_FEE": num(c(cfg, "DEFAULT_MINIMUM_RELAY_TRANSACTION_FEE")),
            "DEFAULT_MINIMUM_STANDARD_TRANSACTION_VERSION": tx_version, "DEFAULT_MAXIMUM_STANDARD_TRANSACTION_VERSION": tx_version,
            "TX_VERSION": tx_version, "SOMPI_PER_KASPA": sompi, "MAX_SOMPI": num(max_sompi.group(1)) * sompi,
            "MAX_SCRIPT_PUBLIC_KEY_VERSION": num(c(con, "MAX_SCRIPT_PUBLIC_KEY_VERSION"))}


def value_of(expr, k):
    names = {"DEFAULT_MINIMUM_RELAY_TRANSACTION_FEE": k["DEFAULT_MINIMUM_RELAY_TRANSACTION_FEE"], "MAXIMUM_STANDARD_TRANSACTION_MASS":
             k["MAXIMUM_STANDARD_TRANSACTION_MASS"], "MAX_SOMPI": k["MAX_SOMPI"], "u64::MAX": U64}
    return names[expr] if expr in names else num(expr)


def relay_fee_rows(src, k):
    body = src[src.index("fn test_calc_min_required_tx_relay_fee()"):src.index("fn test_is_transaction_output_dust()")]
    rows = [{"name": m.group(1), "size": value_of(m.group(2), k), "minimum_relay_transaction_fee": value_of(m.group(3), k), "want": value_of(m.group(4), k)}
            for m in re.finditer(r'name: "([^"]+)",\s*size: ([\w:]+),\s*minimum_relay_transaction_fee: ([\w:]+),\s*want: ([\w:]+),?\s*\}', body)]
    assert len(rows) == 8, rows
    return {"source": "%s:%d (test_calc_min_required_tx_relay_fee)" % (STD, lineno(src, "fn test_calc_min_required_tx_relay_fee()")), "rows": rows}


def dust_rows(src, k):
    body = src[src.index("fn test_is_transaction_output_dust()"):src.index("fn test_check_transaction_standard_in_isolation()")]
    spk = body[body.index("let script_public_key = ScriptPublicKey::new("):body.index("let invalid_script_public_key")]
    spk = bytes(int(x, 16) for x in re.findall(r"0x([0-9a-fA-F]{2})\b", spk[spk.index("smallvec!["):]))
    inv = re.search(r"let invalid_script_public_key = ScriptPublicKey::new\(0, smallvec!\[([^\]]*)\]\);", body).group(1)
    inv = bytes(int(x, 0) for x in inv.split(","))
    assert len(spk) == 36 and inv == b"\x01", (len(spk), inv)
    scripts = {"script_public_key": spk.hex(), "invalid_script_public_key": inv.hex()}
    rows = []
    for m in re.finditer(r'name: "([^"]+)",\s*tx_out: TransactionOutput::new\(([\w:]+), (\w+)(?:\.clone\(\))?\),\s*minimum_relay_transaction_fee: ([\w:]+),\s*'
                         r'is_dust: (true|false),', body):
        rows.append({"name": m.group(1), "value": value_of(m.group(2), k), "script": scripts[m.group(3)], "spk_version": 0,
                     "minimum_relay_transaction_fee": value_of(m.group(4), k), "is_dust": m.group(5) == "true"})
    assert len(rows) == 7 and any(r["value"] == U64 and r["minimum_relay_transaction_fee"] == U64 for r in rows), rows
    return {"source": "%s:%d (test_is_transaction_output_dust)" % (STD, lineno(src, "fn test_is_transaction_output_dust()")), "rows": rows}


# the transactions of test_check_transaction_standard_in_isolation, by name: the edit each makes to the typical P2PK transaction
ISOLATION = {
    "Typical pay-to-pubkey transaction": {},
    "Transaction version too high": {"version": "TX_VERSION + 1"},
    "Transaction size is too large": {"output0": {"value": 0, "script_zeros": "MAXIMUM_STANDARD_TRANSACTION_MASS as usize + 1"}},
    "Signature script size is too large": {"version": "TX_VERSION + 1", "input0_sigscript_zeros": "MAXIMUM_STANDARD_SIGNATURE_SCRIPT_SIZE as usize + 1"},
    "Valid but non standard public key script": {"output0": {"value": "SOMPI_PER_KASPA", "script_ops": ["OpTrue"]}},
    "Dust output": {"output0": {"value": 0}},
    "Null-data transaction": {"output0": {"value": "SOMPI_PER_KASPA", "script_ops": ["OpReturn"]}},
}
OPS = {"OpTrue": 0x51, "OpReturn": 0x6a}


def isolation_cases(src, k):
    body = src[src.index("fn test_check_transaction_standard_in_isolation()"):]
    # the shared pieces, checked against the text they come from
    for needle in ("TransactionOutpoint::new(kaspa_hashes::Hash::from_u64_word(1), 1)", "let dummy_sig_script = vec![0u8; 65];",
                   "TransactionInput::new(dummy_prev_out, dummy_sig_script, MAX_TX_IN_SEQUENCE_NUM, 1)", "let addr_hash = vec![1u8; 32];",
                   "Address::new(Prefix::Testnet, Version::PubKey, &addr_hash)", "TransactionOutput::new(SOMPI_PER_KASPA, dummy_script_public_key)",
                   "NonContextualMasses::new(mass, mass)"):
        assert needle in body, needle
    # pay_to_address_script of a Version::PubKey address: OP_DATA_32 <32-byte key> OP_CHECKSIG (script_class.rs is_pay_to_pubkey)
    p2pk = bytes([0x20]) + bytes([1] * 32) + bytes([0xac])
    value = lambda v: k[v] if isinstance(v, str) else v
    size = lambda e: {"MAXIMUM_STANDARD_TRANSACTION_MASS as usize + 1": k["MAXIMUM_STANDARD_TRANSACTION_MASS"] + 1,
                      "MAXIMUM_STANDARD_SIGNATURE_SCRIPT_SIZE as usize + 1": k["MAXIMUM_STANDARD_SIGNATURE_SCRIPT_SIZE"] + 1}[e]
    cases = []
    for m in re.finditer(r'Test \{\s*name: "([^"]+)",\s*mtx: new_mtx\((.*?),\s*(\d+),\s*\),\s*is_standard: (true|false),\s*\}', body, re.S):
        name, tx_src, mass, std = m.group(1), m.group(2), int(m.group(3)), m.group(4) == "true"
        assert name in ISOLATION, name
        edit = ISOLATION[name]
        version = "TX_VERSION + 1" if re.search(r"Transaction::new\(\s*TX_VERSION \+ 1,", tx_src) else "TX_VERSION"
        assert version == edit.get("version", "TX_VERSION"), name
        tx = {"version": k["TX_VERSION"] + (1 if version != "TX_VERSION" else 0), "lock_time": 0, "subnetwork_id": bytes(20).hex(), "gas": 0,
              "payload": "", "mass": 0,
              "inputs": [{"txid": (1).to_bytes(8, "little").hex() + bytes(24).hex(), "index": 1, "sigscript_zeros": 65, "sequence": U64, "sig_op_count": 1}],
              "outputs": [{"value": k["SOMPI_PER_KASPA"], "spk_version": 0, "script": p2pk.hex()}]}
        if "input0_sigscript_zeros" in edit:
            assert "vec![0u8; MAXIMUM_STANDARD_SIGNATURE_SCRIPT_SIZE as usize + 1]" in tx_src, name
            tx["inputs"][0]["sigscript_zeros"] = size(edit["input0_sigscript_zeros"])
        o = edit.get("output0")
        if o is not None:
            out = tx["outputs"][0]
            out["value"] = value(o["value"])
            assert re.search(r"TransactionOutput::new\(\s*%s" % ("0" if o["value"] == 0 else o["value"]), tx_src), name
            if "script_zeros" in o:
                assert "ScriptVec::from_vec(vec![0u8; MAXIMUM_STANDARD_TRANSACTION_MASS as usize + 1])" in tx_src, name
                del out["script"]
                out["script_zeros"] = size(o["script_zeros"])
            if "script_ops" in o:
                assert all("add_op(%s)" % op in tx_src for op in o["script_ops"]), name
                out["script"] = bytes(OPS[op] for op in o["script_ops"]).hex()
        cases.append({"name": name, "line": lineno(src, 'name: "%s"' % name), "compute_mass": mass, "transient_mass": mass, "is_standard": std, "tx": tx})
    assert [c["name"] for c in cases] == list(ISOLATION), [c["name"] for c in cases]
    return {"source": "%s:%d (test_check_transaction_standard_in_isolation)" % (STD, lineno(src, "fn test_check_transaction_standard_in_isolation()")),
            "p2pk_script": p2pk.hex(), "cases": cases}


if __name__ == "__main__":
    if not REF or not os.path.isdir(REF):
        sys.exit("usage: make_standard_golden.py <rusty-kaspa source tree>")
    src = read(STD)
    k = constants()
    out = {"constants": k, "relay_fee": relay_fee_rows(src, k), "dust": dust_rows(src, k), "isolation": isolation_cases(src, k)}
    with open(os.path.join(OUT, "standard_cases.json"), "w") as f:
        json.dump(out, f, indent=1)
    print("wrote standard_cases.json")
