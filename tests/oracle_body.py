"""CPU restatement of the block body rules (test infrastructure), on top of oracle_isolation.py and oracle/pyref.py.

Written from the reference's Rust, one block at a time, in its order and with its data structures (Python sets for HashSet):
  validate_body_in_isolation   consensus/src/pipeline/body_processor/body_validation_in_isolation.rs:13-131
  validate_body_in_context     body_validation_in_context.rs:20-80 (without check_parent_bodies_exist, a statuses-store query)
  deserialize_coinbase_payload consensus/src/processes/coinbase.rs:185-220
A block is {"transactions": [tx dicts of rusty_kaspa_b200.txbatch], "hash_merkle_root", "daa_score", "blue_score", "past_median_time",
"expected_subsidy"}.  A verdict is the kgv_body_result of include/kgv.h as a dict; `first_tx` / `first_input` are the block's first tx and
input index within a batch, which the three set checks report their offender against (as kgv_block_set_checks does).
"""
import pyref
import oracle_isolation as oi

U64 = (1 << 64) - 1
MIN_PAYLOAD_LENGTH = 8 + 8 + 2 + 1

STATUS = {"Ok": 0, "NoTransactions": 1, "BadMerkleRoot": 2, "FirstTxNotCoinbase": 3, "MultipleCoinbases": 4, "TxInIsolationValidationFailed": 5,
          "ExceedsComputeMassLimit": 6, "ExceedsTransientMassLimit": 7, "ExceedsStorageMassLimit": 8, "DuplicateTransactions": 9,
          "DoubleSpendInSameBlock": 10, "ChainedTransaction": 11, "BadCoinbasePayload": 12, "BadCoinbasePayloadBlueScore": 13, "WrongSubsidy": 14,
          "TxInContextFailed": 15}
NAME = {v: k for k, v in STATUS.items()}
PAYLOAD_ERR = {"PayloadLenBelowMin": 1, "PayloadLenAboveMax": 2, "PayloadScriptPublicKeyLenAboveMax": 3, "PayloadCantContainScriptPublicKey": 4}


class BodyError(Exception):
    def __init__(self, name, index=0, tx_status=0, fail_input=0, a=0, b=0):
        super().__init__(name)
        self.verdict = {"status": STATUS[name], "index": index, "tx_status": tx_status, "fail_input": fail_input, "a": a, "b": b}


def sat_add(a, b):
    return min(a + b, U64)


def calc_hash_merkle_root(txs):
    return pyref.merkle_root([pyref.tx_hash(t) for t in txs])


def _in_isolation(block, rules, max_block_mass, first_tx, first_input):
    txs = block["transactions"]
    # check_has_transactions
    if not txs:
        raise BodyError("NoTransactions")
    # check_hash_merkle_root
    if calc_hash_merkle_root(txs) != bytes(block["hash_merkle_root"]):
        raise BodyError("BadMerkleRoot")
    # check_only_one_coinbase
    if not oi.is_coinbase(txs[0]):
        raise BodyError("FirstTxNotCoinbase")
    for i, tx in enumerate(txs[1:]):
        if oi.is_coinbase(tx):
            raise BodyError("MultipleCoinbases", i)
    # check_transactions_in_isolation
    for p, tx in enumerate(txs):
        st, idx = oi.ok_tx_isolation(tx, rules)
        if st:
            raise BodyError("TxInIsolationValidationFailed", p, st, idx)
    # check_block_mass
    compute = transient = storage = 0
    for p, tx in enumerate(txs):
        c, t = oi.ok_tx_non_contextual_masses(tx, rules)
        compute, transient, storage = sat_add(compute, c), sat_add(transient, t), sat_add(storage, tx.get("mass", 0))
        if compute > max_block_mass:
            raise BodyError("ExceedsComputeMassLimit", p, a=compute, b=max_block_mass)
        if transient > max_block_mass:
            raise BodyError("ExceedsTransientMassLimit", p, a=transient, b=max_block_mass)
        if storage > max_block_mass:
            raise BodyError("ExceedsStorageMassLimit", p, a=storage, b=max_block_mass)
    # check_duplicate_transactions
    ids = set()
    for p, tx in enumerate(txs):
        tid = pyref.tx_id(tx)
        if tid in ids:
            raise BodyError("DuplicateTransactions", first_tx + p)
        ids.add(tid)
    # check_block_double_spends
    existing = set()
    k = first_input
    for tx in txs:
        for x in tx["inputs"]:
            key = (bytes(x["txid"]), x["index"])
            if key in existing:
                raise BodyError("DoubleSpendInSameBlock", k)
            existing.add(key)
            k += 1
    # check_no_chained_transactions
    created = set()
    for tx in txs:
        tid = pyref.tx_id(tx)
        for index in range(len(tx["outputs"])):
            created.add((tid, index))
    k = first_input
    for tx in txs:
        for x in tx["inputs"]:
            if (bytes(x["txid"]), x["index"]) in created:
                raise BodyError("ChainedTransaction", k)
            k += 1
    return compute, transient, storage


def deserialize_coinbase_payload(payload, max_coinbase_payload_len, max_spk_len):
    """(blue_score, subsidy); raises BodyError("BadCoinbasePayload") with the CoinbaseError's code and two numbers"""
    def bad(name, a, b):
        return BodyError("BadCoinbasePayload", tx_status=PAYLOAD_ERR[name], a=a, b=b)
    if len(payload) < MIN_PAYLOAD_LENGTH:
        raise bad("PayloadLenBelowMin", len(payload), MIN_PAYLOAD_LENGTH)
    if len(payload) > max_coinbase_payload_len:
        raise bad("PayloadLenAboveMax", len(payload), max_coinbase_payload_len)
    blue_score = int.from_bytes(payload[0:8], "little")
    subsidy = int.from_bytes(payload[8:16], "little")
    spk_len = payload[18]
    if spk_len > max_spk_len:
        raise bad("PayloadScriptPublicKeyLenAboveMax", spk_len, max_spk_len)
    if len(payload) - MIN_PAYLOAD_LENGTH < spk_len:
        raise bad("PayloadCantContainScriptPublicKey", len(payload), MIN_PAYLOAD_LENGTH + spk_len)
    return blue_score, subsidy


def _in_context(block, rules, max_coinbase_payload_len):
    txs = block["transactions"]
    # check_coinbase_blue_score_and_subsidy
    blue_score, subsidy = deserialize_coinbase_payload(bytes(txs[0]["payload"]), max_coinbase_payload_len, rules["coinbase_payload_script_public_key_max_len"])
    if blue_score != block["blue_score"]:
        raise BodyError("BadCoinbasePayloadBlueScore", a=blue_score, b=block["blue_score"])
    if subsidy != block["expected_subsidy"]:
        raise BodyError("WrongSubsidy", a=block["expected_subsidy"], b=subsidy)
    # check_block_transactions_in_context
    for p, tx in enumerate(txs):
        st, idx = oi.ok_tx_finality(tx, block["daa_score"], block.get("past_median_time", 0))
        if st:
            raise BodyError("TxInContextFailed", p, st, idx)


OK = {"status": 0, "index": 0, "tx_status": 0, "fail_input": 0, "a": 0, "b": 0}


def ok_validate_body(block, rules, max_block_mass, max_coinbase_payload_len, isolation_only=False, first_tx=0, first_input=0):
    """(verdict dict, (compute, transient, storage) masses: zeros unless the verdict is Ok)"""
    try:
        masses = _in_isolation(block, rules, max_block_mass, first_tx, first_input)
        if not isolation_only:
            _in_context(block, rules, max_coinbase_payload_len)
    except BodyError as e:
        return e.verdict, (0, 0, 0)
    return dict(OK), masses


def ok_validate_bodies(blocks, rules, max_block_mass, max_coinbase_payload_len, isolation_only=False):
    """the window form: blocks laid out one after the other in one batch"""
    out, t, i = [], 0, 0
    for b in blocks:
        out.append(ok_validate_body(b, rules, max_block_mass, max_coinbase_payload_len, isolation_only, t, i))
        t += len(b["transactions"])
        i += sum(len(x["inputs"]) for x in b["transactions"])
    return out


def coinbase_payload(blue_score, subsidy, script=b"", spk_version=0, extra=b""):
    """serialize_coinbase_payload (coinbase.rs:141-161)"""
    return blue_score.to_bytes(8, "little") + subsidy.to_bytes(8, "little") + spk_version.to_bytes(2, "little") + bytes([len(script)]) + script + extra


# ---- the reference's own example block and the mutations of validate_body_in_isolation_test (:409-460)
REFERENCE_MUTATIONS = ("BadMerkleRoot", "ExceedsComputeMassLimit", "DuplicateTransactions", "MultipleCoinbases", "DoubleSpendInSameBlock",
                       "FirstTxNotCoinbase", "TxInIsolationValidationFailed", "ChainedTransaction")


def reference_example_blocks():
    """[(name, block, expected error name)]: the example block, then each mutation the reference's test applies to it.  Every mutation but
    the first recomputes the header's merkle root, as the test does."""
    import copy
    import json
    import os
    with open(os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "body_validation_block.json")) as f:
        g = json.load(f)
    base = [oi._tx_from_json(t) for t in g["txs"]]

    def block(txs, root=None):
        return {"transactions": txs, "hash_merkle_root": root if root is not None else calc_hash_merkle_root(txs), "daa_score": 0, "blue_score": 0,
                "past_median_time": 0, "expected_subsidy": 0}
    out = [("example block", block(copy.deepcopy(base), bytes.fromhex(g["hash_merkle_root"])), "Ok")]
    for name in REFERENCE_MUTATIONS:
        txs = copy.deepcopy(base)
        if name == "BadMerkleRoot":
            txs[1]["version"] += 1
            out.append((name, block(txs, bytes.fromhex(g["hash_merkle_root"])), name))
            continue
        if name == "ExceedsComputeMassLimit":
            txs[1]["inputs"][0]["sig_op_count"] = txs[1]["inputs"][1]["sig_op_count"] = 255
        elif name == "DuplicateTransactions":
            txs.append(copy.deepcopy(txs[1]))
        elif name == "MultipleCoinbases":
            txs[1]["subnetwork_id"] = oi.COINBASE
        elif name == "DoubleSpendInSameBlock":
            txs[2]["inputs"][0]["txid"], txs[2]["inputs"][0]["index"] = txs[1]["inputs"][0]["txid"], txs[1]["inputs"][0]["index"]
        elif name == "FirstTxNotCoinbase":
            txs[0]["subnetwork_id"] = oi.NATIVE
        elif name == "TxInIsolationValidationFailed":
            txs[1]["inputs"] = []
        elif name == "ChainedTransaction":
            txs[3]["inputs"][0]["txid"], txs[3]["inputs"][0]["index"] = pyref.tx_id(txs[2]), 0
        out.append((name, block(txs), name))
    return out


SIMPA_SUBSIDY = 44_000_000_000  # month 0 of the deflationary phase, which simpa's params (deflationary_phase_daa_score 0) give every block


def fixture_blocks(name):
    """the blocks of a reference DAG fixture (tests/golden/simpa_goref_*.json.gz) with their real header values.  The first one is the
    DAG's genesis: the reference never validates its body, and its payload carries the genesis subsidy, so only the isolation stage
    applies to it"""
    from golden_util import load, tx_from_json
    return [{"transactions": [tx_from_json(t) for t in b["transactions"]], "hash_merkle_root": bytes.fromhex(b["hash_merkle_root"]),
             "daa_score": b["daa_score"], "blue_score": b["blue_score"], "past_median_time": 0, "expected_subsidy": SIMPA_SUBSIDY}
            for b in load(name)["blocks"]]
