"""CPU restatement of a chain block's UTXO-state verdict (test infrastructure), on top of oracle_body.py and oracle/pyref.py.

Written from the reference's Rust, one chain block at a time, in its order:
  calculate_utxo_state             consensus/src/pipeline/virtual_processor/utxo_validation.rs:110-173 (accepted ids, mergeset_rewards)
  verify_expected_utxo_state       :182-228, checks 1 (commitment), 2 (accepted-id root), 4 (coinbase) and 5 (the chain block's txs)
  verify_coinbase_transaction      :242-258
  expected_coinbase_transaction    consensus/src/processes/coinbase.rs:97-142
The reference's panics (u64 overflow with overflow-checks on, unwrap of a payload parse) become the statuses kgv_replay_verify_chain
reports, at the point where the reference panics.  Check 3 (pruning point) is the caller's and is not restated.
"""
import oracle_body as ob
import oracle_isolation as oi
import pyref

U64 = (1 << 64) - 1
STATUS = {"Ok": 0, "BadUTXOCommitment": 1, "BadAcceptedIDMerkleRoot": 2, "BadCoinbaseTransaction": 3, "RewardOverflow": 4, "CoinbasePayloadUnparsable": 5}
RED, NON_DAA = 1, 2  # KGV_MERGED_*


class ChainPanic(Exception):
    def __init__(self, name):
        super().__init__(name)
        self.status = STATUS[name]


def _add(a, b):
    """u64 addition with the reference's overflow check"""
    if a + b > U64:
        raise ChainPanic("RewardOverflow")
    return a + b


def miner_data(payload, max_payload_len, max_spk_len):
    """deserialize_coinbase_payload(...).unwrap(): (subsidy, spk_version, script, extra data)"""
    try:
        ob.deserialize_coinbase_payload(payload, max_payload_len, max_spk_len)
    except ob.BodyError:
        raise ChainPanic("CoinbasePayloadUnparsable")
    n = payload[18]
    return int.from_bytes(payload[8:16], "little"), int.from_bytes(payload[16:18], "little"), bytes(payload[19:19 + n]), bytes(payload[19 + n:])


def expected_coinbase_transaction(rewards, blue_score, expected_subsidy, miner_payload, max_payload_len, max_spk_len):
    """rewards: [(subsidy, total_fees, spk_version, script, flags)] of the mergeset in group order (mergeset_blues order for the blues).
    Returns the expected coinbase as a tx dict; raises ChainPanic where the reference panics."""
    _, m_ver, m_script, m_extra = miner_data(miner_payload, max_payload_len, max_spk_len)  # verify_coinbase_transaction, :251
    outputs = []
    for sub, fees, ver, script, flags in rewards:  # mergeset_blues filtered by mergeset_non_daa
        if flags & (RED | NON_DAA):
            continue
        v = _add(sub, fees)
        if v > 0:
            outputs.append({"value": v, "spk_version": ver, "script": script})
    red = 0
    for sub, fees, ver, script, flags in rewards:  # mergeset_reds
        if flags & RED:
            red = _add(red, fees if flags & NON_DAA else _add(sub, fees))
    if red > 0:
        outputs.append({"value": red, "spk_version": m_ver, "script": m_script})
    # serialize_coinbase_payload: its script bound is the one the parse above already applied
    payload = ob.coinbase_payload(blue_score, expected_subsidy, m_script, m_ver, m_extra)
    return {"version": 0, "inputs": [], "outputs": outputs, "lock_time": 0, "subnetwork_id": oi.COINBASE, "gas": 0, "payload": payload, "mass": 0}


def verify_chain_block(merged, chain_txs, chain_tx_ok, header, commitment, max_payload_len, max_spk_len):
    """One chain block.  merged: its mergeset in group order, the selected parent first: [{"txs", "accepted" (bool per tx; position 0 is
    not read), "fees" (per tx), "flags" (MERGED_*)}].  chain_txs: the chain block's transactions; chain_tx_ok: one bool per non-coinbase tx
    (its verdict against the block's UTXO view).  header: the kgv_chain_header fields (bytes / ints).  commitment: the finalized running
    multiset after this mergeset.  Returns (kgv_chain_result as a dict, total_fees per merged block (None once its sum overflowed))."""
    status = 0
    ids = [pyref.tx_id(merged[0]["txs"][0])]
    rewards, block_fees = [], []
    for m in merged:
        fee = 0
        for i in range(1, len(m["txs"])):
            if m["accepted"][i]:
                ids.append(pyref.tx_id(m["txs"][i]))
                fee += m["fees"][i]
        block_fees.append(fee if fee <= U64 else None)
        if status:
            continue
        if fee > U64:  # block_fee += validated_tx.calculated_fee (:147)
            status = STATUS["RewardOverflow"]
            continue
        try:  # deserialize_coinbase_payload(&txs[0].payload).unwrap() (:163)
            if not m["txs"]:
                raise ChainPanic("CoinbasePayloadUnparsable")
            sub, ver, script, _ = miner_data(bytes(m["txs"][0]["payload"]), max_payload_len, max_spk_len)
        except ChainPanic as p:
            status = p.status
            continue
        rewards.append((sub, fee, ver, script, m["flags"]))
    root = pyref.blake2b_keyed(b"MerkleBranchHash", bytes(header["selected_parent_accepted_id_merkle_root"]) + pyref.merkle_root(ids))
    out = {"utxo_commitment": bytes(commitment), "accepted_id_merkle_root": root, "coinbase_hash": bytes(32),
           "n_invalid_txs": sum(1 for ok in chain_tx_ok if not ok), "n_txs": max(len(chain_txs) - 1, 0)}
    if not status and bytes(commitment) != bytes(header["utxo_commitment"]):
        status = STATUS["BadUTXOCommitment"]
    if not status and root != bytes(header["accepted_id_merkle_root"]):
        status = STATUS["BadAcceptedIDMerkleRoot"]
    calc_failed = any(f is None for f in block_fees) or len(rewards) < len(merged)
    if not calc_failed:  # the expected coinbase exists only when calculate_utxo_state completed
        try:
            if not chain_txs:
                raise ChainPanic("CoinbasePayloadUnparsable")
            cb = expected_coinbase_transaction(rewards, header["blue_score"], header["expected_subsidy"], bytes(chain_txs[0]["payload"]),
                                               max_payload_len, max_spk_len)
            out["coinbase_hash"] = pyref.tx_hash(cb)
            if not status and out["coinbase_hash"] != pyref.tx_hash(chain_txs[0]):
                status = STATUS["BadCoinbaseTransaction"]
        except ChainPanic as p:
            if not status:
                status = p.status
    out["status"] = status
    return out, block_fees
