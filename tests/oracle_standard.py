"""CPU restatement of the mempool's standardness policy (test infrastructure).

Written from the reference's Rust, one transaction at a time, in its order and with its data structures:
  check_transaction_standard_in_isolation   mining/src/mempool/check_transaction_standard.rs:41-105
  is_transaction_output_dust                :116-163 (the u64 path and the u128 path, with their divisions)
  check_transaction_standard_in_context     :172-211 (the fee check inside the input loop, as written)
  minimum_required_transaction_relay_fee    :215-231 (an overflowing mass * fee raises OverflowError, where the reference panics)
  ScriptClass::from_script                  crypto/txscript/src/script_class.rs:39-82
  parse_script / is_unspendable / get_sig_op_count_upper_bound   crypto/txscript/src/lib.rs:100-104, 176-233, opcodes/macros.rs:9-61
Where the reference's to_small_int panics (OP_16 before a multisig opcode, opcodes/mod.rs:1065-1073) the library counts 16, and so does
this restatement.  Transactions are the dicts of rusty_kaspa_b200.txbatch.  Results are (status, index, detail) with the KGV_TX_* numbers
of include/kgv.h.
"""
import json
import os

MAX_STANDARD_P2SH_SIG_OPS = 15
MAXIMUM_STANDARD_SIGNATURE_SCRIPT_SIZE = 1650
MAXIMUM_STANDARD_TRANSACTION_MASS = 100_000
DEFAULT_MINIMUM_RELAY_TRANSACTION_FEE = 1000
MAX_SOMPI = 29_000_000_000 * 100_000_000
MAX_PUB_KEYS_PER_MUTLTISIG = 20
U64 = (1 << 64) - 1

STATUS = {"Ok": 0, "RejectVersion": 32, "RejectComputeMass": 33, "RejectTransientMass": 34, "RejectSignatureScriptSize": 35,
          "RejectScriptPublicKeyVersion": 36, "RejectOutputScriptClass": 37, "RejectDust": 38, "RejectStorageMass": 39,
          "RejectInputScriptClass": 40, "RejectSignatureCount": 41, "RejectInsufficientFee": 42}
NAME = {v: k for k, v in STATUS.items()}
NON_STANDARD, PUB_KEY, PUB_KEY_ECDSA, SCRIPT_HASH = 0, 1, 2, 3


class Policy:
    def __init__(self, minimum_relay_transaction_fee=DEFAULT_MINIMUM_RELAY_TRANSACTION_FEE, minimum_standard_transaction_version=0,
                 maximum_standard_transaction_version=0):
        self.fee = minimum_relay_transaction_fee
        self.min_version, self.max_version = minimum_standard_transaction_version, maximum_standard_transaction_version


def parse_script(script):
    """[(opcode, data)] and whether the walk ended in a parse error (a malformed push is always the last item: it ran out of bytes)"""
    ops, i, n = [], 0, len(script)
    while i < n:
        op = script[i]
        i += 1
        if 0x01 <= op <= 0x4b:  # OpData1..OpData75: fixed length
            data = script[i:i + op]
            i += op
            if len(data) != op:
                return ops, True
        elif 0x4c <= op <= 0x4e:  # OpPushData1/2/4: a little-endian length, then the data
            w = {0x4c: 1, 0x4d: 2, 0x4e: 4}[op]
            lb = script[i:i + w]
            i += w
            if len(lb) != w:
                return ops, True
            ln = int.from_bytes(lb, "little")
            data = script[i:i + ln]
            i += ln
            if len(data) != ln:
                return ops, True
        else:
            data = b""
        ops.append((op, bytes(data)))
    return ops, False


def script_class(version, script):
    if version != 0:
        return NON_STANDARD
    s = bytes(script)
    if len(s) == 34 and s[0] == 0x20 and s[33] == 0xac:
        return PUB_KEY
    if len(s) == 35 and s[0] == 0x21 and s[34] == 0xab:
        return PUB_KEY_ECDSA
    if len(s) == 35 and s[0] == 0xaa and s[1] == 0x20 and s[34] == 0x87:
        return SCRIPT_HASH
    return NON_STANDARD


def is_unspendable(script):
    ops, err = parse_script(bytes(script))
    return err or (len(ops) > 0 and ops[0][0] == 0x6a)


def is_transaction_output_dust(value, script, minimum_relay_transaction_fee):
    if is_unspendable(script):
        return True
    total_serialized_size = 8 + 2 + 8 + len(script) + 148
    # the u64 path (checked_mul(1000) is Some) and the u128 path compute the same integer quotient; Python's integers are exact for both
    return (value * 1000) // (3 * total_serialized_size) < minimum_relay_transaction_fee


def _to_small_int(op):
    return 0 if op == 0x00 else op - 0x50


def sig_op_count_by_opcodes(ops, err):
    n = 0
    for i, (op, _) in enumerate(ops):
        if op in (0xac, 0xad, 0xab):
            n += 1
        elif op in (0xae, 0xaf, 0xa9):
            if i == 0:
                n += MAX_PUB_KEYS_PER_MUTLTISIG
                continue
            prev = ops[i - 1][0]
            n += _to_small_int(prev) if 0x51 <= prev <= 0x60 else MAX_PUB_KEYS_PER_MUTLTISIG
    return n  # a parse error ends the list of parsed opcodes, so the count stops there either way


def sig_op_count_upper_bound_p2sh(signature_script):
    ops, err = parse_script(bytes(signature_script))
    if err or not ops or any(op > 0x60 for op, _ in ops):  # empty, a parse error, or an opcode that is not a push
        return 0
    return sig_op_count_by_opcodes(*parse_script(ops[-1][1]))


def minimum_required_transaction_relay_fee(mass, fee):
    if mass * fee > U64:
        raise OverflowError("mass * minimum_relay_transaction_fee overflows u64")
    m = mass * fee // 1000
    if m == 0:
        m = fee
    return min(m, MAX_SOMPI)


def check_in_isolation(tx, compute_mass, transient_mass, policy):
    if tx["version"] > policy.max_version or tx["version"] < policy.min_version:
        return STATUS["RejectVersion"], 0, tx["version"]
    if compute_mass > MAXIMUM_STANDARD_TRANSACTION_MASS:
        return STATUS["RejectComputeMass"], 0, compute_mass
    if transient_mass > MAXIMUM_STANDARD_TRANSACTION_MASS:
        return STATUS["RejectTransientMass"], 0, transient_mass
    for i, inp in enumerate(tx["inputs"]):
        if len(inp["sigscript"]) > MAXIMUM_STANDARD_SIGNATURE_SCRIPT_SIZE:
            return STATUS["RejectSignatureScriptSize"], i, len(inp["sigscript"])
    for i, o in enumerate(tx["outputs"]):
        if o["spk_version"] > 0:
            return STATUS["RejectScriptPublicKeyVersion"], i, 0
        if script_class(o["spk_version"], o["script"]) == NON_STANDARD:
            return STATUS["RejectOutputScriptClass"], i, 0
        if is_transaction_output_dust(o["value"], o["script"], policy.fee):
            return STATUS["RejectDust"], i, o["value"]
    return 0, 0, 0


def check_in_context(tx, entries, storage_mass, compute_mass, fee, policy):
    """entries: one dict per input (spk_version, script).  Raises OverflowError where the reference panics."""
    if storage_mass > MAXIMUM_STANDARD_TRANSACTION_MASS:
        return STATUS["RejectStorageMass"], 0, storage_mass
    for i, (inp, e) in enumerate(zip(tx["inputs"], entries)):
        c = script_class(e["spk_version"], e["script"])
        if c == NON_STANDARD:
            return STATUS["RejectInputScriptClass"], i, 0
        if c == SCRIPT_HASH:
            n = sig_op_count_upper_bound_p2sh(inp["sigscript"])
            if n > MAX_STANDARD_P2SH_SIG_OPS:
                return STATUS["RejectSignatureCount"], i, n
        minimum_fee = minimum_required_transaction_relay_fee(compute_mass, policy.fee)
        if fee < minimum_fee:
            return STATUS["RejectInsufficientFee"], 0, minimum_fee
    return 0, 0, 0


# ---- the reference's own cases (tests/golden/standard_cases.json, made by tests/golden/make_standard_golden.py)
def golden():
    with open(os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "standard_cases.json")) as f:
        return json.load(f)


def tx_from_golden(t):
    """a txbatch dict from the fixture's record (long zero scripts are stored by length)"""
    ins = [{"txid": bytes.fromhex(i["txid"]), "index": i["index"], "sigscript": bytes(i["sigscript_zeros"]) if "sigscript_zeros" in i else bytes.fromhex(i["sigscript"]),
            "sequence": i["sequence"], "sig_op_count": i["sig_op_count"]} for i in t["inputs"]]
    outs = [{"value": o["value"], "spk_version": o["spk_version"], "script": bytes(o["script_zeros"]) if "script_zeros" in o else bytes.fromhex(o["script"])}
            for o in t["outputs"]]
    return {"version": t["version"], "lock_time": t["lock_time"], "subnetwork_id": bytes.fromhex(t["subnetwork_id"]), "gas": t["gas"],
            "payload": bytes.fromhex(t["payload"]), "mass": t["mass"], "inputs": ins, "outputs": outs}


# the NonStandardError each isolation case raises (the reference's test asserts only is_standard)
ISOLATION_EXPECTED = {"Typical pay-to-pubkey transaction": ("Ok", 0), "Transaction version too high": ("RejectVersion", 0),
                      "Transaction size is too large": ("RejectOutputScriptClass", 0), "Signature script size is too large": ("RejectVersion", 0),
                      "Valid but non standard public key script": ("RejectOutputScriptClass", 0), "Dust output": ("RejectDust", 0),
                      "Null-data transaction": ("RejectOutputScriptClass", 0)}
