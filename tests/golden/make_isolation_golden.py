#!/usr/bin/env python3
"""Extracts the reference's own cases for the isolation and lock-time finality rules into tests/golden/isolation_cases.json.

Run where the reference sources are available (the GPU machines do not have them):
    python tests/golden/make_isolation_golden.py <rusty-kaspa source tree>   (or set RUSTY_KASPA_SRC)
Sources, parsed at run time and recorded in the fixture:
  consensus/src/processes/transaction_validator/tx_validation_in_isolation.rs  validate_tx_in_isolation_test: the valid coinbase, the valid
                                                                               transaction, every mutation and the error it must raise
  consensus/src/pipeline/body_processor/body_validation_in_context.rs          the check_for_lock_time_and_sequence cases (NotFinalized)
  consensus/core/src/config/params.rs, consensus/core/src/config/bps.rs,
  consensus/core/src/constants.rs                                              mainnet values of the rule parameters and constants
"""
import json
import os
import re
import sys

REF = sys.argv[1] if len(sys.argv) > 1 else os.environ.get("RUSTY_KASPA_SRC", "")
OUT = os.path.dirname(os.path.abspath(__file__))
ISO = "consensus/src/processes/transaction_validator/tx_validation_in_isolation.rs"
CTX = "consensus/src/pipeline/body_processor/body_validation_in_context.rs"
PARAMS = "consensus/core/src/config/params.rs"


def read(rel):
    with open(os.path.join(REF, rel)) as f:
        return f.read()


def hexbytes(s):
    return bytes(int(x, 16) for x in re.findall(r"0x([0-9a-fA-F]{2})\b", re.sub(r"//[^\n]*", "", s)))


def lineno(src, needle):
    return src[:src.index(needle)].count("\n") + 1


def mainnet_rules():
    src = read(PARAMS)
    body = src[src.index("pub const MAINNET_PARAMS: Params = Params {"):src.index("pub const TESTNET_PARAMS")]
    num = lambda name: int(re.search(r"\n\s*%s:\s*([\d_]+)," % name, body).group(1).replace("_", ""))
    bps = int(re.search(r"blockrate: BlockrateParams::new::<(\d+)>\(\)", body).group(1))
    table = read("consensus/core/src/config/bps.rs")
    k = dict((int(a), int(b)) for a, b in re.findall(r"(\d+) => (\d+)", table[table.index("pub const fn ghostdag_k()"):]))[bps]
    consts = read("consensus/core/src/constants.rs")
    const = lambda name: re.search(r"pub const %s: u\d+ = ([^;]+);" % name, consts).group(1)
    return {n: num(n) for n in ("max_tx_inputs", "max_tx_outputs", "max_signature_script_len", "max_script_public_key_len", "mass_per_tx_byte",
                                "mass_per_script_pub_key_byte", "mass_per_sig_op", "coinbase_payload_script_public_key_max_len")} | {
        "ghostdag_k": k, "bps": bps,
        "LOCK_TIME_THRESHOLD": int(const("LOCK_TIME_THRESHOLD").replace("_", "")),
        "TRANSIENT_BYTE_TO_MASS_FACTOR": int(const("TRANSIENT_BYTE_TO_MASS_FACTOR")),
        "MAX_SOMPI": int(re.fullmatch(r"([\d_]+) \* SOMPI_PER_KASPA", const("MAX_SOMPI")).group(1).replace("_", "")) * int(const("SOMPI_PER_KASPA").replace("_", "")),
        "TX_VERSION": int(const("TX_VERSION"))}


def tx_json(version, inputs, outputs, lock_time, subnetwork, gas, payload):
    return {"version": version, "lock_time": lock_time, "subnetwork_id": subnetwork.hex(), "gas": gas, "payload": payload.hex(), "mass": 0,
            "inputs": [{"txid": t.hex(), "index": i, "sigscript": s.hex(), "sequence": q, "sig_op_count": c} for t, i, s, q, c in inputs],
            "outputs": [{"value": v, "spk_version": 0, "script": s.hex()} for v, s in outputs]}


# every mutation line of the test, as the structured edit the consumers apply
MUTATIONS = {
    "tx.subnetwork_id = SubnetworkId::from_byte(3);": {"subnetwork_id": (bytes([3]) + bytes(19)).hex()},
    "tx.inputs = vec![];": {"inputs": "empty"},
    "tx.inputs = (0..params.max_tx_inputs + 1).map(|_| valid_tx.inputs[0].clone()).collect();": {"inputs": "repeat_first", "count": "max_tx_inputs+1"},
    "tx.inputs[0].signature_script = vec![0; params.max_signature_script_len + 1];": {"sigscript0_zeros": "max_signature_script_len+1"},
    "tx.outputs = (0..params.max_tx_outputs + 1).map(|_| valid_tx.outputs[0].clone()).collect();": {"outputs": "repeat_first", "count": "max_tx_outputs+1"},
    "tx.outputs[0].script_public_key = ScriptPublicKey::new(0, scriptvec![0u8; params.max_script_public_key_len + 1]);":
        {"spk0_zeros": "max_script_public_key_len+1"},
    "tx.inputs.push(tx.inputs[0].clone());": {"inputs": "push_first"},
    "tx.gas = 1;": {"gas": 1},
    "tx.payload = vec![0];": {"payload": "00"},
    "tx.version = TX_VERSION + 1;": {"version": "TX_VERSION+1"},
}


def isolation_cases():
    src = read(ISO)
    body = src[src.index("fn validate_tx_in_isolation_test()"):]
    over = dict((k, int(v)) for k, v in re.findall(r"params\.(max_tx_\w+) = (\d+);", body))
    cb_src = body[body.index("let valid_cb = Transaction::new("):body.index("tv.validate_tx_in_isolation(&valid_cb)")]
    spk = cb_src[cb_src.index("scriptvec!("):cb_src.index(")", cb_src.index("scriptvec!("))]
    cb_value = int(re.search(r"value: (0x[0-9a-fA-F]+|\d+)", cb_src).group(1), 0)
    cb_payload = bytes(int(x) for x in re.search(r"vec!\[(\d+(?:,\s*\d+)*)\]", cb_src[cb_src.index("SUBNETWORK_ID_COINBASE"):]).group(1).split(","))
    valid_cb = tx_json(0, [], [(cb_value, hexbytes(spk))], 0, bytes([1]) + bytes(19), 0, cb_payload)
    tx_src = body[body.index("let valid_tx = Transaction::new("):body.index("tv.validate_tx_in_isolation(&valid_tx)")]
    txid = hexbytes(tx_src[tx_src.index("TransactionId::from_slice(&["):tx_src.index("]),")])
    sig = hexbytes(tx_src[tx_src.index("signature_script: vec!["):tx_src.index("],", tx_src.index("signature_script: vec!["))])
    outs = []
    for m in re.finditer(r"value: (0x[0-9a-fA-F]+|\d+),\s*script_public_key: ScriptPublicKey::new\(\s*0,\s*scriptvec!\((.*?)\),\s*\),", tx_src, re.S):
        outs.append((int(m.group(1), 0), hexbytes(m.group(2))))
    assert len(txid) == 32 and len(sig) == 140 and len(outs) == 2, (len(txid), len(sig), len(outs))
    assert "sequence: u64::MAX" in tx_src and "sig_op_count: 0" in tx_src and "index: 0" in tx_src
    valid_tx = tx_json(0, [(txid, 0, sig, 2**64 - 1, 0)], outs, 0, bytes(20), 0, b"")
    cases = []
    for m in re.finditer(r"let mut tx(?:: Transaction)? = valid_tx(?:\.clone\(\))?;\s*\n\s*(.*?)\n\s*assert_match!\(tv\.validate_tx_in_isolation\(&tx\), (.*?)\);", body, re.S):
        line = re.sub(r"\s+", " ", m.group(1).strip())
        assert line in MUTATIONS, line
        res = m.group(2)
        err = "Ok" if res == "Ok(())" else re.match(r"Err\(TxRuleError::(\w+)", res).group(1)
        cases.append({"line": lineno(src, m.group(1).strip()), "mutation": MUTATIONS[line], "source": line, "error": err})
    assert len(cases) == len(MUTATIONS), len(cases)
    return {"source": "%s:%d-%d (validate_tx_in_isolation_test)" % (ISO, lineno(src, "fn validate_tx_in_isolation_test()"), src.count("\n")),
            "rule_overrides": over, "valid_coinbase": valid_cb, "valid_tx": valid_tx, "cases": cases}


def finality_cases():
    """check_for_lock_time_and_sequence(consensus, parent, hash, lock_time, sequence, should_pass): the lock time relative to the block's DAA
    score (tip_daa_score) or past median time, a single input with that sequence"""
    src = read(CTX)
    out = []
    for m in re.finditer(r"check_for_lock_time_and_sequence\(\s*&consensus,\s*valid_block_child\.header\.hash,\s*(\d+)\.into\(\),\s*(tip_daa_score|past_median_time)"
                         r"\s*([+-]\s*\d+)?,\s*(0|u64::MAX),\s*(true|false),?\s*\)", src):
        out.append({"line": lineno(src, m.group(0)), "against": "daa_score" if m.group(2) == "tip_daa_score" else "past_median_time",
                    "lock_time_offset": int(m.group(3).replace(" ", "")) if m.group(3) else 0, "sequence": 0 if m.group(4) == "0" else 2**64 - 1,
                    "passes": m.group(5) == "true"})
    assert len(out) == 8 and sum(not c["passes"] for c in out) == 4, out
    tpl = src[src.index("async fn check_for_lock_time_and_sequence("):]
    assert "TransactionOutpoint::new(1.into(), 0), vec![], sequence, 0)" in tpl and "NotFinalized" in tpl
    return {"source": "%s:%d-%d (check_for_lock_time_and_sequence)" % (CTX, lineno(src, "let tip_daa_score = valid_block_child.header.daa_score + 1;"), src.count("\n")),
            "tx": "one input (outpoint (1, 0), empty signature script, the case's sequence, sig_op_count 0), no outputs, native subnetwork",
            "failure": "NotFinalized", "cases": out}


if __name__ == "__main__":
    if not REF or not os.path.isdir(REF):
        sys.exit("usage: make_isolation_golden.py <rusty-kaspa source tree>")
    with open(os.path.join(OUT, "isolation_cases.json"), "w") as f:
        json.dump({"mainnet": mainnet_rules(), "isolation": isolation_cases(), "finality": finality_cases()}, f, indent=1)
    print("wrote isolation_cases.json")
