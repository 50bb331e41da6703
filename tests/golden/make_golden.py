#!/usr/bin/env python3
"""Extracts the reference's own known-answer vectors for the validation hot path into JSON fixtures.

Run in the build container (needs /root/reference; the GPU box does not have it):
    python tests/golden/make_golden.py
Outputs (committed): tests/golden/{hashers,tx_hashing,sighash,check_scripts_kat,muhash}.json, simpa_goref_1060.json.gz,
simpa_goref_pruning_5000.json.gz, script_tests.json.gz

Everything is parsed out of the reference's Rust test sources / test data at run time — nothing is
retyped by hand — and each fixture records the file:line range it came from:
  crypto/hashes/src/hashers.rs:142-233                     incremental domain hashers
  consensus/core/src/hashing/tx.rs:118-203                 tx id / tx hash (8 vectors)
  consensus/core/src/hashing/sighash.rs:293-690            sighash (29 vectors)
  consensus/src/processes/transaction_validator/tx_validation_in_utxo_context.rs:228-709
                                                           real mainnet Schnorr P2PK / 2-of-4 P2SH multisig spends
  testing/integration/testdata/dags_for_json_tests/goref-1060-tx-265-blocks/blocks.json.gz
                                                           simpa-generated DAG: 224 signed inputs, all valid
  crypto/muhash/src/lib.rs:17-21,189-238,290-327,430-444   MuHash known answers (empty, 3 vectors, pre-computed, serialize, parse)
  crypto/muhash/src/u3072.rs:455-555                       MuHash field edge cases (overflowing values, (p-1)^2, inverse edge case)
  consensus/core/src/utxo/utxo_diff.rs:270-568             UtxoDiff algebra rule table (diff_from / with_diff)
"""
import gzip
import json
import os
import re
import sys

REF = "/root/reference"
OUT = os.path.dirname(os.path.abspath(__file__))


def read(rel):
    with open(os.path.join(REF, rel)) as f:
        return f.read()


def dump(name, obj):
    if name.endswith(".gz"):
        with gzip.GzipFile(os.path.join(OUT, name), "wb", mtime=0) as f:
            f.write(json.dumps(obj, separators=(",", ":")).encode())
    else:
        with open(os.path.join(OUT, name), "w") as f:
            json.dump(obj, f, indent=1)
    print("wrote", name)


# ------------------------------------------------------------------------------------ hashers
def hashers():
    src = read("crypto/hashes/src/hashers.rs")
    body = src[src.index("fn test_vectors()"):]
    inputs_src = body[body.index("let input_data = ["):body.index("fn run_test_vector")]
    # the five inputs, in order
    inputs = [b"", bytes([1])]
    m = re.search(r"&\[\s*((?:\d+,\s*)+\d+),?\s*\]\[\.\.\]", inputs_src[inputs_src.index("&[1][..]") + 8:])
    inputs.append(bytes(int(x) for x in re.findall(r"\d+", m.group(1))))
    assert "&[42; 64]" in inputs_src and "&[0; 8][..]" in inputs_src
    inputs += [bytes([42]) * 64, bytes(8)]
    vectors = []
    for m in re.finditer(r"run_test_vector\(\s*&input_data,\s*(\w+)::new,\s*&\[(.*?)\],\s*\);", body, re.S):
        vectors.append({"hasher": m.group(1), "expected": re.findall(r'"([0-9a-f]{64})"', m.group(2))})
    assert len(vectors) >= 6 and all(len(v["expected"]) == 5 for v in vectors)
    dump("hashers.json", {"source": "crypto/hashes/src/hashers.rs:142-233",
                          "note": "the hasher is NOT reset between inputs: expected[i] = H(input[0] || ... || input[i])",
                          "inputs_hex": [b.hex() for b in inputs], "vectors": vectors})


# ------------------------------------------------------------------------------------ tx id / hash
def tx_hashing():
    src = read("consensus/core/src/hashing/tx.rs")
    body = src[src.index("fn test_transaction_hashing()"):]
    exp = re.findall(r'expected_id:\s*"([0-9a-f]{64})",\s*expected_hash:\s*"([0-9a-f]{64})"', body)
    assert len(exp) == 8
    # transactions exactly as constructed by the test (tx.rs:125-193); TransactionInput::new(outpoint, sigscript, sequence, sig_op_count)
    assert "TransactionInput::new(TransactionOutpoint::new(Hash::from_u64_word(0), 2), vec![1, 2], 7, 5)" in body
    sub = lambda b: bytes([b]) + bytes(19)
    in_a = [{"txid": bytes(32).hex(), "index": 2, "sigscript": "0102", "sequence": 7, "sig_op_count": 5}]
    in_b = [{"txid": "59b3d6dc6cdc660c389c3fdb5704c48c598d279cdf1bab54182db586a4c95dd5", "index": 2, "sigscript": "0102", "sequence": 7, "sig_op_count": 5}]
    assert in_b[0]["txid"] in body
    out = [{"value": 1564, "spk_version": 7, "script": "0102030405"}]
    mk = lambda ver, ins, outs, lock, subnet, gas, payload: {"version": ver, "inputs": ins, "outputs": outs, "lock_time": lock,
                                                             "subnetwork_id": subnet.hex(), "gas": gas, "payload": payload, "mass": 0}
    txs = [mk(0, [], [], 0, sub(0), 0, ""), mk(1, in_a, [], 0, sub(0), 0, ""), mk(1, in_a, out, 0, sub(0), 0, ""),
           mk(2, in_a, out, 54, sub(0), 3, ""), mk(2, in_b, out, 54, sub(0), 3, ""), mk(2, in_b, out, 54, sub(1), 3, ""),
           mk(2, in_b, out, 54, sub(2), 3, ""), mk(2, in_b, out, 54, sub(2), 3, "010203")]
    dump("tx_hashing.json", {"source": "consensus/core/src/hashing/tx.rs:118-203",
                             "vectors": [{"tx": t, "expected_id": e[0], "expected_hash": e[1]} for t, e in zip(txs, exp)]})


# ------------------------------------------------------------------------------------ sighash
def sighash():
    src = read("consensus/core/src/hashing/sighash.rs")
    body = src[src.index("fn test_signature_hash()"):]
    prev = re.search(r'TransactionId::from_str\("([0-9a-f]{64})"\)', body).group(1)
    spks = re.findall(r'hex_decode\("([0-9a-f]+)"', body)[:2]
    ht = {"SIG_HASH_ALL": 1, "SIG_HASH_NONE": 2, "SIG_HASH_SINGLE": 4, "SIG_HASH_ALL_ANYONE_CAN_PAY": 0x81,
          "SIG_HASH_NONE_ANYONE_CAN_PAY": 0x82, "SIG_HASH_SINGLE_ANYONE_CAN_PAY": 0x84}
    vectors = []
    for m in re.finditer(r'TestVector \{\s*name: "([^"]+)",\s*populated_tx: &(\w+),\s*hash_type: (\w+),\s*input_index: (\d+),\s*'
                         r'action: ModifyAction::(\w+)(?:\((\d+)\))?,\s*expected_hash: "([0-9a-f]{64})"', body):
        vectors.append({"name": m.group(1), "tx": "native" if m.group(2).startswith("native") else "subnetwork", "hash_type": ht[m.group(3)],
                        "input_index": int(m.group(4)), "action": m.group(5), "action_arg": int(m.group(6)) if m.group(6) else None,
                        "expected": m.group(7)})
    assert len(vectors) == 29, len(vectors)
    ins = [{"txid": prev, "index": i, "sigscript": "", "sequence": i, "sig_op_count": 0} for i in range(3)]
    outs = [{"value": 300, "spk_version": 0, "script": spks[1]}, {"value": 300, "spk_version": 0, "script": spks[0]}]
    native = {"version": 0, "inputs": ins, "outputs": outs, "lock_time": 1615462089000, "subnetwork_id": bytes(20).hex(), "gas": 0, "payload": "", "mass": 0}
    subnet = dict(native, subnetwork_id=(bytes(range(1, 11)) + bytes(10)).hex(), gas=250, payload=bytes(range(10, 21)).hex())
    entries = [{"amount": 100, "spk_version": 0, "script": spks[0]}, {"amount": 200, "spk_version": 0, "script": spks[1]},
               {"amount": 300, "spk_version": 0, "script": spks[1]}]
    dump("sighash.json", {"source": "consensus/core/src/hashing/sighash.rs:293-690",
                          "actions": {"Output": "outputs[i].value = 100", "Input": "inputs[i].index = 2", "AmountSpent": "entries[i].amount = 666",
                                      "PrevScriptPublicKey": "entries[i].script += 010203", "Sequence": "inputs[i].sequence = 12345",
                                      "Payload": "payload = 06060604020001030307", "Gas": "gas = 1234",
                                      "SubnetworkId": "subnetwork_id = 06060604020001030307 + 10 zero bytes"},
                          "native": native, "subnetwork": subnet, "entries": entries, "vectors": vectors})


# ------------------------------------------------------------------------------------ check_scripts KATs
def check_scripts_kat():
    rel = "consensus/src/processes/transaction_validator/tx_validation_in_utxo_context.rs"
    src = read(rel)
    names = ["check_signature_test", "check_incorrect_signature_test", "check_multi_signature_test",
             "check_last_sig_incorrect_multi_signature_test", "check_first_sig_incorrect_multi_signature_test",
             "check_empty_incorrect_multi_signature_test", "check_non_push_only_script_sig_test"]
    cases = []
    for nm in names:
        start = src.index("fn %s()" % nm)
        end = src.index("#[test]", start) if "#[test]" in src[start:] else len(src)
        body = src[start:end]
        line0 = src[:start].count("\n") + 1
        prev = re.search(r'TransactionId::from_str\("([0-9a-f]{64})"\)', body).group(1)
        hexes = re.findall(r'hex_decode\(\s*"([0-9a-f]*)"', body)
        sigscript, spk1, spk2 = hexes[0], hexes[1], (hexes[2] if len(hexes) > 2 else None)
        var = {"script_pub_key_1": spk1, "script_pub_key_2": spk2}
        inp = re.search(r"index: (\d+) \},\s*signature_script,\s*sequence: (\d+),\s*sig_op_count: (\d+)", body)
        outs = [{"value": int(v), "spk_version": 0, "script": var[k]} for v, k in
                re.findall(r"TransactionOutput \{ value: (\d+), script_public_key: ScriptPublicKey::new\(0, (script_pub_key_\d)", body)]
        ent = re.search(r"amount: (\d+),\s*script_public_key: ScriptPublicKey::new\(0, (script_pub_key_\d)\S*\),\s*block_daa_score: (\d+),\s*is_coinbase: (\w+)", body)
        tx = {"version": 0, "inputs": [{"txid": prev, "index": int(inp.group(1)), "sigscript": sigscript, "sequence": int(inp.group(2)),
                                         "sig_op_count": int(inp.group(3))}],
              "outputs": outs, "lock_time": 0, "subnetwork_id": bytes(20).hex(), "gas": 0, "payload": "", "mass": 0}
        entry = {"amount": int(ent.group(1)), "spk_version": 0, "script": var[ent.group(2)], "block_daa_score": int(ent.group(3)),
                 "is_coinbase": ent.group(4) == "true"}
        # expected results: the single-input tx, then the tx with its last input duplicated (lib.rs par_iter split)
        def expectation(fragment):
            m = re.search(r"TxScriptError::(\w+)", fragment)
            if m:
                return m.group(1)
            if ".expect(" in fragment:
                return "Ok"
            return "AnyError"
        split = body.index("duplicate_input(&tx")
        first, second = body[body.index("PopulatedTransaction::new("):split], body[split:]
        cases.append({"name": nm, "source": "%s:%d" % (rel, line0), "tx": tx, "entries": [entry],
                      "expected": expectation(first[first.index("check_scripts"):] if "check_scripts" in first else first),
                      "expected_duplicated_input": expectation(second)})
    dump("check_scripts_kat.json", {"source": rel + ":228-709",
                                    "note": "expected = TxScriptError variant wrapped in TxRuleError::SignatureInvalid, 'Ok', or 'AnyError' "
                                            "(test only asserts is_err). *_duplicated_input: same tx with its last input (and entry) appended again.",
                                    "cases": cases})


# ------------------------------------------------------------------------------------ simpa DAG fixture
def _simpa_fixture(rel, out_name, note_extra=""):
    with gzip.open(os.path.join(REF, rel), "rt") as f:
        lines = f.read().splitlines()
    params = json.loads(lines[0])
    blocks = [json.loads(l) for l in lines[1:]]

    def conv_tx(t):
        return {"version": t["version"],
                "inputs": [{"txid": i["previousOutpoint"]["transactionId"], "index": i["previousOutpoint"]["index"],
                            "sigscript": i["signatureScript"], "sequence": i["sequence"], "sig_op_count": i["sigOpCount"]} for i in t["inputs"]],
                "outputs": [{"value": o["value"], "spk_version": int(o["scriptPublicKey"][:4], 16), "script": o["scriptPublicKey"][4:]} for o in t["outputs"]],
                "lock_time": t["lockTime"], "subnetwork_id": t["subnetworkId"], "gas": t["gas"], "payload": t["payload"], "mass": t.get("mass", 0)}

    out_blocks = []
    for b in blocks:
        h = b["header"]
        out_blocks.append({"hash": h["hash"], "daa_score": h["daaScore"], "hash_merkle_root": h["hashMerkleRoot"],
                           "accepted_id_merkle_root": h["acceptedIdMerkleRoot"], "utxo_commitment": h["utxoCommitment"],
                           "parents": h["parentsByLevel"][0] if h["parentsByLevel"] else [], "blue_work": h["blueWork"], "blue_score": h["blueScore"],
                           "transactions": [conv_tx(t) for t in b["transactions"]]})
    dump(out_name, {"source": rel, "coinbase_maturity": params.get("blockrate", {}).get("coinbase_maturity", params.get("coinbase_maturity")),
                    "storage_mass_parameter": params.get("storage_mass_parameter"),
                    "note": "simpa-generated DAG (simpa/generate-json-tests-data.sh); the reference's json_test replays it and asserts "
                            "every block ends UTXO-valid, so every signed input here must verify. tx ids are NOT stored: they must be "
                            "recomputed (hashing/tx.rs) to resolve the inputs' previous outpoints.  Header fields kept: hashMerkleRoot "
                            "(calc_hash_merkle_root), utxoCommitment (MuHash of the UTXO set in the block's past), acceptedIdMerkleRoot (KIP-15 "
                            "form), level-0 parents and blueWork (selected parent = max (blue_work, hash), processes/ghostdag/ordering.rs)." + note_extra,
                    "blocks": out_blocks})


def simpa_fixture():
    _simpa_fixture("testing/integration/testdata/dags_for_json_tests/goref-1060-tx-265-blocks/blocks.json.gz", "simpa_goref_1060.json.gz")
    _simpa_fixture("testing/integration/testdata/dags_for_json_tests/goref_custom_pruning_depth/blocks.json.gz", "simpa_goref_pruning_5000.json.gz",
                   "  5 001 blocks, 4 790 signed single-input transactions (json_test `goref_custom_pruning_depth_test`).")


# ------------------------------------------------------------------------------------ script engine rows
def script_tests():
    """crypto/txscript/test-data/script_tests.json (872 rows of which 850 are tests, 'short form' assembly) -> raw script bytes.
    The assembler restates opcodes::parse_short_form (crypto/txscript/src/opcodes/macros.rs:138-175) and
    ScriptBuilder::{add_i64,add_data,add_op} (script_builder.rs:88-243); the opcode-name table is parsed out of
    crypto/txscript/src/opcodes/mod.rs."""
    src = read("crypto/txscript/src/opcodes/mod.rs")
    names = {}
    for m in re.finditer(r"opcode\s+(?:\|\w+\|\s+)?(\w+)<(0x[0-9a-fA-F]+),", src):
        names[m.group(1)] = int(m.group(2), 16)
    assert len(names) == 256, len(names)
    by_token = {}
    for name, num in names.items():
        by_token[name.upper()] = num
        if name in ("OpFalse", "OpTrue") or (num != 0x00 and (num < 0x51 or num > 0x60)):
            by_token.setdefault(name[2:].upper(), num)

    def ser_i64(v, maxlen=8):
        neg, p, out, sat = v < 0, abs(v), bytearray(), False
        while p:
            b = p & 0xFF
            sat = bool(b & 0x80)
            out.append(b)
            p >>= 8
        if sat:
            out.append(0)
        if neg:
            out[-1] |= 0x80
        assert len(out) <= maxlen
        return bytes(out)

    class Rejected(Exception):
        pass

    def add_data(script, data):
        n = len(data)
        if n == 0 or (n == 1 and (data[0] <= 16 or data[0] == 0x81)):
            size = 1
        else:
            size = n + (1 if n <= 75 else 2 if n <= 255 else 3 if n <= 65535 else 5)
        if len(script) + size > 10000:
            raise Rejected("DataRejected")
        if n > 520:
            raise Rejected("ElementExceedsMaxSize")
        if n == 0:
            script.append(0x00)
        elif n == 1 and 1 <= data[0] <= 16:
            script.append(0x50 + data[0])
        elif n == 1 and data[0] == 0x81:
            script.append(0x4F)
        else:
            if n <= 75:
                script.append(n)
            elif n <= 255:
                script += bytes([0x4C, n])
            else:
                script += bytes([0x4D, n & 0xFF, n >> 8])
            script += data

    def assemble(text):
        script = bytearray()
        for line in text.splitlines():
            line = line.split("#")[0]
            for tok in line.split():
                try:
                    v = int(tok)
                    if not (-2**63 <= v < 2**63) or not re.fullmatch(r"[+-]?\d+", tok):
                        raise ValueError
                    if v == -2**63:
                        add_data(script, ser_i64(v, 9))
                    elif v == 0:
                        script.append(0x00)
                    elif v == -1 or 1 <= v <= 16:
                        script.append(0x50 + v)
                    else:
                        add_data(script, ser_i64(v))
                    continue
                except ValueError:
                    pass
                if tok.startswith("0x") and re.fullmatch(r"(?:[0-9a-fA-F]{2})*", tok[2:]):
                    script += bytes.fromhex(tok[2:])
                elif len(tok) >= 2 and tok[0] == "'" and tok[-1] == "'":
                    add_data(script, tok[1:-1].encode())
                else:
                    t = tok.replace("_", "").upper()
                    if t not in by_token:
                        raise KeyError("cannot parse token %r" % tok)
                    if len(script) >= 10000:
                        raise Rejected("OpCodeRejected")
                    script.append(by_token[t])
        return bytes(script)

    rows = json.load(open(os.path.join(REF, "crypto/txscript/test-data/script_tests.json")))
    out = []
    for r in rows:
        if len(r) < 4:
            continue
        sig_txt, spk_txt, _flags, expected = r[0], r[1], r[2], r[3]
        row = {"sig_text": sig_txt, "spk_text": spk_txt, "expected": expected}
        try:
            row["sigscript"] = assemble(sig_txt).hex()
            row["spk"] = assemble(spk_txt).hex()
        except Rejected as e:
            row["builder_error"] = str(e)  # ScriptBuilderError: the reference test maps ElementExceedsMaxSize to PUSH_SIZE
        out.append(row)
    assert len(out) == 850, len(out)  # 872 JSON rows, 22 of them comments
    dump("script_tests.json.gz", {"source": "crypto/txscript/test-data/script_tests.json via opcodes::parse_short_form; harness crypto/txscript/src/lib.rs:1366-1555",
                                  "spending_tx": "create_spending_transaction (lib.rs:1366-1397): version 1, one input spending output 0 of a version-1 'coinbase' "
                                                 "(input outpoint (0^32, 0xffffffff), sigscript 0000, sequence u64::MAX, sig_op_count 20, one 0-value output with the spk), "
                                                 "sequence u64::MAX, sig_op_count 20, one 0-value output with an empty spk; entry: amount 0, daa 0, coinbase",
                                  "rows": out})


# ------------------------------------------------------------------------------------ muhash
def muhash():
    src = read("crypto/muhash/src/lib.rs")
    ints = lambda txt: bytes(int(x, 0) for x in re.findall(r"0x[0-9a-fA-F]+|\d+", txt))
    m = re.search(r"pub const EMPTY_MUHASH: Hash = Hash::from_bytes\(\[(.*?)\]\);", src, re.S)
    empty = ints(m.group(1))
    assert len(empty) == 32
    vecs = []
    tv = src[src.index("const TEST_VECTORS: [TestVector; 3] = ["):src.index("fn element_from_byte")]
    for m in re.finditer(r"data: &\[(.*?)\],\s*multiset_hash: Hash::from_bytes\(\[(.*?)\]\),\s*cumulative_hash: Hash::from_bytes\(\[(.*?)\]\),", tv, re.S):
        d, mh, ch = ints(m.group(1)), ints(m.group(2)), ints(m.group(3))
        assert len(mh) == 32 and len(ch) == 32
        vecs.append({"data": d.hex(), "multiset_hash": mh.hex(), "cumulative_hash": ch.hex()})
    assert len(vecs) == 3
    pre = re.search(r'fn test_new_pre_computed\(\) \{\s*let expected = "([0-9a-f]{64})";', src).group(1)
    ser_src = src[src.index("fn test_serialize()"):]
    ser = ints(re.search(r"let expected = \[(.*?)\];", ser_src, re.S).group(1))
    assert len(ser) == 384
    u3072 = read("crypto/muhash/src/u3072.rs")
    prime_diff = int(re.search(r"pub const PRIME_DIFF: Limb = (\d+);", u3072).group(1))
    # the field's own edge tests (u3072.rs:455-555): 64-bit limbs, little-endian
    limbs = lambda txt: [int(x) for x in re.findall(r"\d+", txt)]
    edge = limbs(re.search(r"fn test_inverse_edge_case\(\) \{.*?limbs: \[(.*?)\],", u3072, re.S).group(1))
    assert len(edge) == 48
    assert "limbs[0] = Limb::MAX - i;" in u3072 and "(0..PRIME_DIFF).into_par_iter()" in u3072  # exhuastive_test_div_overflow
    assert "max.limbs[0] -= u3072::PRIME_DIFF;" in u3072 and "max *= copy_max;" in u3072  # test_mul_max
    dump("muhash.json", {"source": "crypto/muhash/src/lib.rs:17-21 (EMPTY_MUHASH), :189-238 (TEST_VECTORS), :290-298 (test_new_pre_computed), "
                                   ":301-327 (test_serialize), :430-444 (test_parse_muhash_fail); crypto/muhash/src/u3072.rs:22 (PRIME_DIFF)",
                         "prime_diff": prime_diff, "empty_muhash": empty.hex(), "test_vectors": vecs,
                         "pre_computed": {"add": ["00" + "00" * 31, "01" + "00" * 31], "remove": ["02" + "00" * 31], "finalized": pre},
                         "serialize": {"add": ["01" + "00" * 31, "02" + "00" * 31], "serialized": ser.hex()},
                         "parse_fail": {"overflow": "9b28ef" + "ff" * 381, "ok": "0028ef" + "ff" * 381, "all_ff_overflows": True},
                         "u3072_edges": {
                             "source": "crypto/muhash/src/u3072.rs:455-484 (exhuastive_test_div_overflow), :486-493 (test_mul_max), "
                                       ":521-555 (test_inverse_edge_case)",
                             "inverse_edge_case": b"".join(x.to_bytes(8, "little") for x in edge).hex(),
                             "mul_max": {"a": ((2**3072 - 1) - prime_diff).to_bytes(384, "little").hex(), "a_times_a": "01" + "00" * 383},
                             "div_overflow": {"x_i": "2^3072 - 1 - i for i in 0..prime_diff", "x_over_1": "prime_diff - 1 - i",
                                              "x_over_x": "1 for every i but prime_diff - 1 (x = p, which is 0)"}}})


# ------------------------------------------------------------------------------------ utxo diff algebra
def utxo_diff_rules():
    """consensus/core/src/utxo/utxo_diff.rs:270-568 test_utxo_diff_rules: the table of (this, other) -> diff_from / with_diff results.
    One outpoint (0^32, 0), two entries: entry1 = (amount 10, daa 0, coinbase), entry2 = (amount 20, daa 1, coinbase)."""
    src = read("consensus/core/src/utxo/utxo_diff.rs")
    body = src[src.index("let tests = ["):src.index("// Run the tests")]

    def diff(txt):
        d = {"add": [], "remove": []}
        for kind, ent in re.findall(r"insert_(add|remove)_point\(outpoint0, utxo_entry(\d)\.clone\(\)\)", txt):
            d[kind].append(int(ent))
        return d

    def result(txt):
        txt = txt.strip()
        if txt.startswith("Ok("):
            return {"ok": diff(txt)}
        m = re.match(r"Err\(UtxoAlgebraError::(\w+)\(", txt)
        return {"err": m.group(1)}

    tests = []
    for m in re.finditer(r'Test \{\s*name: "(.*?)",\s*this: (.*?),\s*other: (.*?),\s*expected_diff_from_result: (.*?),\s*expected_with_diff_result: (.*?),\s*\},', body, re.S):
        tests.append({"name": m.group(1), "this": diff(m.group(2)), "other": diff(m.group(3)), "diff_from": result(m.group(4)), "with_diff": result(m.group(5))})
    assert len(tests) == len(re.findall(r"Test \{", body)) and len(tests) >= 20, len(tests)
    dump("utxo_diff_rules.json", {"source": "consensus/core/src/utxo/utxo_diff.rs:270-568 (test_utxo_diff_rules)",
                                  "entries": {"1": {"amount": 10, "block_daa_score": 0, "is_coinbase": True}, "2": {"amount": 20, "block_daa_score": 1, "is_coinbase": True}},
                                  "note": "errors compare by variant (and outpoint) only, utxo_error.rs:29-43; after every Ok result the reference also checks the "
                                          "round trip this.with_diff(diff_from) == other and this.diff_from(with_diff) == other",
                                  "tests": tests})


# ------------------------------------------------------------------------------------ storage mass (KIP-9) cases
def storage_mass():
    """consensus/core/src/mass/mod.rs:516-729: test_storage_mass (explicit expected values, evaluated by a tiny interpreter of the test's
    own statements) and test_storage_mass_pluralities (pairs of transactions that must have EQUAL, non-zero mass)."""
    src = read("consensus/core/src/mass/mod.rs")
    consts = read("consensus/core/src/constants.rs")
    sompi = int(re.search(r"SOMPI_PER_KASPA: u64 = ([\d_]+);", consts).group(1).replace("_", ""))
    assert re.search(r"STORAGE_MASS_PARAMETER: u64 = SOMPI_PER_KASPA \* 10_000;", consts)
    env0 = {"SOMPI_PER_KASPA": sompi, "STORAGE_MASS_PARAMETER": sompi * 10_000}
    unit = int(re.search(r"const UTXO_UNIT_SIZE: u64 = (\d+);", src).group(1))

    def ev(expr, env):
        e = expr.strip().replace("_u64", "").replace("u64", "")
        e = re.sub(r"(\d+)\.pow\((\d+)\)", r"(\1**\2)", e)
        e = re.sub(r"(?<=\d)_(?=\d)", "", e)
        e = e.replace("/", "//")
        return int(eval(e, {"__builtins__": {}}, dict(env)))

    def amounts(txt, env):
        txt = txt.strip()
        m = re.match(r"\[(.+)(?:;| REP)\s*(\d+)\]$", txt)  # [x; n]
        if m:
            return [ev(m.group(1), env)] * int(m.group(2))
        return [ev(x, env) for x in txt.strip("[]").split(",") if x.strip()]

    # ---- test_storage_mass: statements in order
    body = src[src.index("fn test_storage_mass()"):src.index("fn generate_tx_from_amounts")]
    cases, cur, param, env = [], {}, None, dict(env0)
    body = re.sub(r"//[^\n]*", "", body)
    body = re.sub(r"\[(\w+); (\d+)\]", r"[\1 REP \2]", body)  # [x; n] must survive the split on ';'
    for stmt in body.split(";"):
        st = " ".join(stmt.split())
        m = re.search(r"let (?:mut )?(tx\d?) = generate_tx_from_amounts\(&(\[.*?\]), &(\[.*?\])\)", st)
        if m:
            cur[m.group(1)] = {"ins": amounts(m.group(2), env), "outs": amounts(m.group(3), env)}
            continue
        m = re.search(r"let mut (tx\d) = (tx\d?)\.clone\(\)", st)
        if m:
            cur[m.group(1)] = {"ins": list(cur[m.group(2)]["ins"]), "outs": list(cur[m.group(2)]["outs"])}
            continue
        m = re.search(r"let (\w+) = ([^;]+)$", st)
        if m and m.group(1) in ("storage_mass_parameter", "base_value"):
            env[m.group(1)] = ev(m.group(2), env)
            continue
        m = re.search(r"(tx\d?)\.tx\.outputs\[(\d+)\]\.value = (.+)$", st)
        if m:
            cur[m.group(1)]["outs"][int(m.group(2))] = ev(m.group(3), env)
            continue
        if re.search(r"for out in tx\.tx\.outputs\.iter_mut\(\) \{ out\.value \+= 1 \}", st) or "out.value += 1" in st:
            cur["tx"]["outs"] = [v + 1 for v in cur["tx"]["outs"]]  # (the closing brace shares the statement with what follows)
        m = re.search(r"tx\.entries\[0\]\.as_mut\(\)\.unwrap\(\)\.amount \+= tx\.tx\.outputs\.len\(\)", st)
        if m:
            cur["tx"]["ins"][0] += len(cur["tx"]["outs"])
            continue
        if "tx.tx.outputs.pop()" in st:
            cur["tx"]["outs"].pop()
            continue
        m = re.search(r"let storage_mass = MassCalculator::new\(0, 0, 0, (.+?)\)\.calc_contextual_masses\(&(tx\d?)\.as_verifiable\(\)\)\.unwrap\(\)", st)
        if m:
            pending = {"ins": list(cur[m.group(2)]["ins"]), "outs": list(cur[m.group(2)]["outs"]), "storage_mass_parameter": ev(m.group(1), env)}
            continue
        m = re.search(r"assert_eq!\(storage_mass, (.+)\)$", st)
        if m:
            e = m.group(1)
            pending["expected"] = ev(e, env)
            cases.append(pending)
    assert len(cases) == 8 and [c["expected"] for c in cases][:1] == [0] and cases[5]["expected"] == 9000000000 and cases[7]["expected"] == 5000000000, cases

    # ---- test_storage_mass_pluralities
    pb = src[src.index("fn test_storage_mass_pluralities()"):src.index("fn generate_script_for_plurality")]
    pl = []
    for m in re.finditer(r'PluralityTestCase \{\s*name: "([^"]+)",\s*inputs_tx1: &(\[.*?\]),\s*outputs_tx1: &(\[.*?\]),\s*inputs_tx2: &(\[.*?\]),\s*outputs_tx2: &(\[.*?\]),\s*'
                         r'plurality_index: Some\((\d+)\),\s*desired_plurality: Some\((\d+)\),\s*override_output: (true|false),\s*storage_mass_parameter: ([^,]+),', pb, re.S):
        pl.append({"name": m.group(1), "inputs_tx1": amounts(m.group(2), env0), "outputs_tx1": amounts(m.group(3), env0), "inputs_tx2": amounts(m.group(4), env0),
                   "outputs_tx2": amounts(m.group(5), env0), "plurality_index": int(m.group(6)), "desired_plurality": int(m.group(7)), "override_output": m.group(8) == "true",
                   "storage_mass_parameter": ev(m.group(9), env0), "script_len_for_plurality": (int(m.group(7)) - 1) * unit})
    assert len(pl) == len(re.findall(r"PluralityTestCase \{", pb)) - 0 and len(pl) >= 8, len(pl)
    dump("storage_mass.json", {"source": "consensus/core/src/mass/mod.rs:516-729 (test_storage_mass_pluralities, test_storage_mass)",
                               "note": "every script public key is empty (plurality 1) except the one the plurality cases override: script = (desired_plurality-1)*100 bytes "
                                       "(generate_script_for_plurality). Plurality cases assert mass(tx1) == mass(tx2) != 0.",
                               "cases": cases, "plurality_cases": pl})


# ------------------------------------------------------------------------------------ body_validation_in_isolation example block
def body_validation_block():
    """consensus/src/pipeline/body_processor/body_validation_in_isolation.rs:153-462 (validate_body_in_isolation_test): the example block (a Rust
    literal) with the hash_merkle_root its header commits to, and the three set-check mutations the test applies with the error each must raise."""
    src = read("consensus/src/pipeline/body_processor/body_validation_in_isolation.rs")
    body = src[src.index("fn validate_body_in_isolation_test()"):src.index("async fn merkle_root_missing_parents_known_invalid_test")]
    body = re.sub(r"//[^\n]*", "", body)
    hdr = body[body.index("Header::new_finalized("):body.index("vec![\n                Transaction::new(")]
    merkle = bytes(int(x, 16) for x in re.findall(r"0x([0-9a-f]{2})\b", hdr[hdr.rindex("Hash::from_slice(&["):hdr.index("]),", hdr.rindex("Hash::from_slice(&["))]))
    assert len(merkle) == 32
    txs_src = body[body.index("vec![\n                Transaction::new("):body.index("body_processor.validate_body_in_isolation(&example_block.clone()")]
    toks = re.findall(r"0x[0-9a-fA-F]+|\d[\d_]*|[A-Za-z_][A-Za-z_0-9]*(?:::[A-Za-z_][A-Za-z_0-9]*)*!?|[\[\](){},:;&.]", txs_src)
    pos = [0]

    def peek():
        return toks[pos[0]]

    def take(x=None):
        t = toks[pos[0]]
        assert x is None or t == x, (t, x, toks[pos[0] - 5:pos[0] + 5])
        pos[0] += 1
        return t

    def num(t):
        return int(t, 16) if t.startswith("0x") else int(t.replace("_", ""))

    def byte_list(close):  # after the opening bracket
        out = []
        while peek() != close:
            t = take()
            if t != ",":
                out.append(num(t))
        take(close)
        return bytes(out)

    def value():
        t = take()
        if t in ("vec!", "scriptvec!"):
            opener = take()
            close = "]" if opener == "[" else ")"
            if peek() in ("TransactionInput", "TransactionOutput", "Transaction::new"):
                items = []
                while peek() != close:
                    if peek() == ",":
                        take()
                        continue
                    items.append(value())
                take(close)
                return items
            return byte_list(close)
        if t == "Transaction::new":
            take("(")
            args = []
            while peek() != ")":
                if peek() == ",":
                    take()
                    continue
                args.append(value())
            take(")")
            ver, ins, outs, lock, subnet, gas, payload = args
            return {"version": ver, "inputs": ins, "outputs": outs, "lock_time": lock, "subnetwork_id": subnet, "gas": gas, "payload": payload}
        if t in ("TransactionInput", "TransactionOutput", "TransactionOutpoint"):
            take("{")
            d = {}
            while peek() != "}":
                if peek() == ",":
                    take()
                    continue
                k = take()
                take(":")
                d[k] = value()
            take("}")
            return d
        if t in ("TransactionId::from_slice", "Hash::from_slice"):
            take("("); take("&"); take("[")
            b = byte_list("]")
            take(")")
            return b
        if t == "ScriptPublicKey::new":
            take("(")
            ver = value(); take(",")
            sc = value()
            if peek() == ",":
                take()
            take(")")
            return {"spk_version": ver, "script": sc}
        if t == "u64::MAX":
            return 2**64 - 1
        if t == "SUBNETWORK_ID_NATIVE":
            return bytes(20)
        if t == "SUBNETWORK_ID_COINBASE":
            return bytes([1]) + bytes(19)
        return num(t)

    txs = value()
    assert len(txs) >= 4 and not txs[0]["inputs"] and len(txs[1]["inputs"]) == 2, [len(t["inputs"]) for t in txs]
    js = []
    for t in txs:
        js.append({"version": t["version"], "lock_time": t["lock_time"], "subnetwork_id": t["subnetwork_id"].hex(), "gas": t["gas"], "payload": t["payload"].hex(), "mass": 0,
                   "inputs": [{"txid": i["previous_outpoint"]["transaction_id"].hex(), "index": i["previous_outpoint"]["index"], "sigscript": i["signature_script"].hex(),
                               "sequence": i["sequence"], "sig_op_count": i["sig_op_count"]} for i in t["inputs"]],
                   "outputs": [{"value": o["value"], "spk_version": o["script_public_key"]["spk_version"], "script": o["script_public_key"]["script"].hex()} for o in t["outputs"]]})
    # the mutations of the test and the error each must raise (lines 423-460)
    for needle in ("txs.push(txs[1].clone());", "txs[2].inputs[0].previous_outpoint = txs[1].inputs[0].previous_outpoint;",
                   "txs[3].inputs[0].previous_outpoint = TransactionOutpoint { transaction_id: txs[2].id(), index: 0 };"):
        assert needle in body, needle
    order = [body.index("RuleError::DuplicateTransactions(_)"), body.index("RuleError::DoubleSpendInSameBlock(_)"), body.index("RuleError::ChainedTransaction(_)")]
    assert order == sorted(order)
    dump("body_validation_block.json", {"source": "consensus/src/pipeline/body_processor/body_validation_in_isolation.rs:153-462 (validate_body_in_isolation_test)",
                                        "hash_merkle_root": merkle.hex(), "txs": js,
                                        "mutations": [{"do": "push a clone of txs[1]", "error": "DuplicateTransactions"},
                                                      {"do": "txs[2].inputs[0].previous_outpoint = txs[1].inputs[0].previous_outpoint", "error": "DoubleSpendInSameBlock"},
                                                      {"do": "txs[3].inputs[0].previous_outpoint = (txs[2].id(), 0)", "error": "ChainedTransaction"}]})


if __name__ == "__main__":
    if not os.path.isdir(REF):
        sys.exit("needs /root/reference (run in the build container)")
    hashers()
    tx_hashing()
    sighash()
    check_scripts_kat()
    simpa_fixture()
    script_tests()
    muhash()
    utxo_diff_rules()
    storage_mass()
    body_validation_block()
