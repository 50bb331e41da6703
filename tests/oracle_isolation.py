"""CPU restatement of the isolation rules, lock-time finality and non-contextual masses (test infrastructure).

Written from the reference's Rust, one transaction at a time, in its order and with its data structures:
  validate_tx_in_isolation          consensus/src/processes/transaction_validator/tx_validation_in_isolation.rs:16-26 (a set for duplicates)
  check_tx_is_finalized             tx_validation_in_header_context.rs
  calc_non_contextual_masses        consensus/core/src/mass/mod.rs:248-269, transaction_estimated_serialized_size :13-59
Transactions are the dicts of rusty_kaspa_b200.txbatch.  Results are (status, index) with the KGV_TX_* numbers of include/kgv.h.
"""
MAX_SOMPI = 29_000_000_000 * 100_000_000
LOCK_TIME_THRESHOLD = 500_000_000_000
TRANSIENT_BYTE_TO_MASS_FACTOR = 4
TX_VERSION = 0
U64 = (1 << 64) - 1
COINBASE = bytes([1]) + bytes(19)
NATIVE = bytes(20)

STATUS = {"Ok": 0, "NoTxInputs": 14, "TooManyInputs": 15, "TooBigSignatureScript": 16, "TooManyOutputs": 17, "TooBigScriptPublicKey": 18,
          "CoinbaseHasInputs": 19, "CoinbaseNonZeroMassCommitment": 20, "CoinbaseTooManyOutputs": 21, "CoinbaseScriptPublicKeyTooLong": 22,
          "TxOutZero": 23, "TxOutTooHigh": 24, "OutputsValueOverflow": 25, "TotalTxOutTooHigh": 26, "TxDuplicateInputs": 27, "TxHasGas": 28,
          "SubnetworksDisabled": 29, "UnknownTxVersion": 30, "NotFinalized": 31}
NAME = {v: k for k, v in STATUS.items()}


class RuleError(Exception):
    def __init__(self, name, index=0):
        super().__init__(name, index)
        self.status, self.index = STATUS[name], index


def is_coinbase(tx):
    return bytes(tx["subnetwork_id"]) == COINBASE


def _first(seq, pred):
    for i, x in enumerate(seq):
        if pred(x):
            return i
    return None


def _isolation(tx, r):
    cb = is_coinbase(tx)
    ins, outs = tx["inputs"], tx["outputs"]
    # check_transaction_inputs_in_isolation
    if not cb and not ins:
        raise RuleError("NoTxInputs")
    if len(ins) > r["max_tx_inputs"]:
        raise RuleError("TooManyInputs")
    i = _first(ins, lambda x: len(x["sigscript"]) > r["max_signature_script_len"])
    if i is not None:
        raise RuleError("TooBigSignatureScript", i)
    # check_transaction_outputs_in_isolation
    if not cb and len(outs) > r["max_tx_outputs"]:
        raise RuleError("TooManyOutputs")
    i = _first(outs, lambda o: len(o["script"]) > r["max_script_public_key_len"])
    if i is not None:
        raise RuleError("TooBigScriptPublicKey", i)
    # check_coinbase_in_isolation
    if cb:
        if ins:
            raise RuleError("CoinbaseHasInputs")
        if tx.get("mass", 0) > 0:
            raise RuleError("CoinbaseNonZeroMassCommitment")
        if len(outs) > r["ghostdag_k"] + 2:
            raise RuleError("CoinbaseTooManyOutputs")
        i = _first(outs, lambda o: len(o["script"]) > r["coinbase_payload_script_public_key_max_len"])
        if i is not None:
            raise RuleError("CoinbaseScriptPublicKeyTooLong", i)
    # check_transaction_output_value_ranges
    total = 0
    for i, o in enumerate(outs):
        if o["value"] == 0:
            raise RuleError("TxOutZero", i)
        if o["value"] > MAX_SOMPI:
            raise RuleError("TxOutTooHigh", i)
        total += o["value"]
        if total > U64:
            raise RuleError("OutputsValueOverflow")
        if total > MAX_SOMPI:
            raise RuleError("TotalTxOutTooHigh")
    # check_duplicate_transaction_inputs
    seen = set()
    for x in ins:
        key = (bytes(x["txid"]), x["index"])
        if key in seen:
            raise RuleError("TxDuplicateInputs")
        seen.add(key)
    if tx["gas"] > 0:
        raise RuleError("TxHasGas")
    if not cb and bytes(tx["subnetwork_id"]) != NATIVE:
        raise RuleError("SubnetworksDisabled")
    if tx["version"] != TX_VERSION:
        raise RuleError("UnknownTxVersion")


def _finality(tx, daa_score, past_median_time):
    lt = tx["lock_time"]
    if lt == 0:
        return
    ref = daa_score if lt < LOCK_TIME_THRESHOLD else past_median_time
    if lt < ref:
        return
    i = _first(tx["inputs"], lambda x: x["sequence"] != U64)
    if i is not None:
        raise RuleError("NotFinalized", i)


def ok_tx_isolation(tx, rules):
    """validate_tx_in_isolation: (status, index)"""
    try:
        _isolation(tx, rules)
    except RuleError as e:
        return e.status, e.index
    return 0, 0


def ok_tx_finality(tx, daa_score, past_median_time):
    """check_tx_is_finalized as validate_tx_in_header_context_with_args picks its argument: (status, index)"""
    try:
        _finality(tx, daa_score, past_median_time)
    except RuleError as e:
        return e.status, e.index
    return 0, 0


def ok_tx_validate(tx, rules, daa_score, past_median_time, finality=True):
    """isolation, then (finality=True) the finality check: what kgv_validate_txs_in_isolation reports"""
    st = ok_tx_isolation(tx, rules)
    if st[0] or not finality:
        return st
    return ok_tx_finality(tx, daa_score, past_median_time)


def estimated_serialized_size(tx):
    size = 2 + 8
    size += sum(32 + 4 + 8 + len(x["sigscript"]) + 8 for x in tx["inputs"])
    size += 8
    size += sum(8 + 2 + 8 + len(o["script"]) for o in tx["outputs"])
    size += 8 + 20 + 8 + 32 + 8 + len(tx["payload"])
    return size


def ok_tx_non_contextual_masses(tx, rules):
    """calc_non_contextual_masses in u64 arithmetic that wraps: (compute_mass, transient_mass)"""
    if is_coinbase(tx):
        return 0, 0
    size = estimated_serialized_size(tx)
    spk = sum(2 + len(o["script"]) for o in tx["outputs"])
    sigops = sum(x["sig_op_count"] for x in tx["inputs"])
    compute = (size * rules["mass_per_tx_byte"] + spk * rules["mass_per_script_pub_key_byte"] + sigops * rules["mass_per_sig_op"]) & U64
    return compute, (size * TRANSIENT_BYTE_TO_MASS_FACTOR) & U64


# ---- the reference's own cases (tests/golden/isolation_cases.json, written by tests/golden/make_isolation_golden.py)
def _tx_from_json(j):
    return {"version": j["version"], "lock_time": j["lock_time"], "subnetwork_id": bytes.fromhex(j["subnetwork_id"]), "gas": j["gas"],
            "payload": bytes.fromhex(j["payload"]), "mass": j["mass"],
            "inputs": [{"txid": bytes.fromhex(i["txid"]), "index": i["index"], "sigscript": bytes.fromhex(i["sigscript"]), "sequence": i["sequence"],
                        "sig_op_count": i["sig_op_count"]} for i in j["inputs"]],
            "outputs": [{"value": o["value"], "spk_version": o["spk_version"], "script": bytes.fromhex(o["script"])} for o in j["outputs"]]}


def _apply(tx, m, rules):
    t = dict(tx, inputs=[dict(i) for i in tx["inputs"]], outputs=[dict(o) for o in tx["outputs"]])
    count = lambda key: rules[key.split("+")[0]] + 1
    if "subnetwork_id" in m:
        t["subnetwork_id"] = bytes.fromhex(m["subnetwork_id"])
    if m.get("inputs") == "empty":
        t["inputs"] = []
    if m.get("inputs") == "repeat_first":
        t["inputs"] = [dict(tx["inputs"][0]) for _ in range(count(m["count"]))]
    if m.get("inputs") == "push_first":
        t["inputs"].append(dict(t["inputs"][0]))
    if m.get("outputs") == "repeat_first":
        t["outputs"] = [dict(tx["outputs"][0]) for _ in range(count(m["count"]))]
    if "sigscript0_zeros" in m:
        t["inputs"][0]["sigscript"] = bytes(count(m["sigscript0_zeros"]))
    if "spk0_zeros" in m:
        t["outputs"][0]["script"] = bytes(count(m["spk0_zeros"]))
    if "gas" in m:
        t["gas"] = m["gas"]
    if "payload" in m:
        t["payload"] = bytes.fromhex(m["payload"])
    if m.get("version") == "TX_VERSION+1":
        t["version"] = TX_VERSION + 1
    return t


def golden():
    import json
    import os
    with open(os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "isolation_cases.json")) as f:
        return json.load(f)


def mainnet_rules(g=None):
    g = g or golden()
    return {k: g["mainnet"][k] for k in ("max_tx_inputs", "max_tx_outputs", "max_signature_script_len", "max_script_public_key_len", "mass_per_tx_byte",
                                         "mass_per_script_pub_key_byte", "mass_per_sig_op", "ghostdag_k", "coinbase_payload_script_public_key_max_len")}


def isolation_golden_cases(g=None):
    """[(name, tx, expected error name)] of validate_tx_in_isolation_test, and the rules that test uses (mainnet with its overrides)"""
    g = g or golden()
    iso = g["isolation"]
    rules = dict(mainnet_rules(g), **iso["rule_overrides"])
    cb, tx = _tx_from_json(iso["valid_coinbase"]), _tx_from_json(iso["valid_tx"])
    cases = [("valid_cb", cb, "Ok"), ("valid_tx", tx, "Ok")]
    cases += [("line %d: %s" % (c["line"], c["source"]), _apply(tx, c["mutation"], rules), c["error"]) for c in iso["cases"]]
    return cases, rules


def finality_golden_cases(daa_score=1000, past_median_time=1_700_000_000_000, g=None):
    """[(name, tx, expected error name, daa_score, past_median_time)] of the check_for_lock_time_and_sequence cases, at a context of our choosing"""
    g = g or golden()
    out = []
    for c in g["finality"]["cases"]:
        base = daa_score if c["against"] == "daa_score" else past_median_time
        tx = {"version": 0, "inputs": [{"txid": bytes([1]) + bytes(31), "index": 0, "sigscript": b"", "sequence": c["sequence"], "sig_op_count": 0}],
              "outputs": [], "lock_time": base + c["lock_time_offset"], "subnetwork_id": NATIVE, "gas": 0, "payload": b"", "mass": 0}
        out.append(("line %d" % c["line"], tx, "Ok" if c["passes"] else g["finality"]["failure"], daa_score, past_median_time))
    return out
