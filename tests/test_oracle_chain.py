"""The chain-block restatement (oracle_chain.py) pinned against the reference's own blocks: every block of both simpa DAG fixtures, each from
its own point of view (its selected parent's UTXO state and multiset, its mergeset in consensus order), must reproduce the utxoCommitment and
acceptedIdMerkleRoot the reference wrote into its header, and the restated expected coinbase must hash to the coinbase the reference's miner
put into the block.

What the fixtures can and cannot reach: every mergeset in both is all blue (blue_score(B) - blue_score(SP) == |mergeset| is asserted), and
the only non-DAA merged block is genesis, under its children (derived from daa_score differences and asserted).  Those children pay no
blue output for it, so the non-DAA skip and the "> 0" rule are pinned here.  The red reward and a non-DAA red are pinned by reading
coinbase.rs only; the GPU tests compare them with this restatement on flags the fixtures do not carry."""
import ctypes
import os
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.join(os.path.dirname(HERE), "oracle"))
sys.path.insert(0, HERE)
import oracle_body  # noqa: E402
import oracle_chain as oc  # noqa: E402
import oracle_tx  # noqa: E402
import pyref  # noqa: E402
import pytest  # noqa: E402
from golden_util import simpa_dag_replay_plan  # noqa: E402
from rusty_kaspa_b200.txbatch import build_batch  # noqa: E402

MAX_PAYLOAD_LEN, MAX_SPK_LEN = 204, 150  # simpa runs with the mainnet values of both


class OkMuHash(ctypes.Structure):
    _fields_ = [("num", ctypes.c_uint64 * 48), ("den", ctypes.c_uint64 * 48)]


def chain_block_inputs(oracle, fixture):
    """Yields, for every non-genesis block B of the fixture in file order, the inputs of oracle_chain.verify_chain_block from B's own point of
    view, plus (B's fixture record, its selected parent's record, the mergeset hashes, the number of non-DAA merged blocks)."""
    fx, by, order, sp, ordered_mergeset, chain = simpa_dag_replay_plan(fixture)
    prm = oracle_tx.params(coinbase_maturity=fx["coinbase_maturity"], storage_mass_parameter=fx["storage_mass_parameter"])
    genesis = order[0]
    last_use = {}
    for k, h in enumerate(order):
        if sp(h) is not None:
            last_use[sp(h)] = k
    state, mh = {genesis: {}}, {}
    mh[genesis] = OkMuHash()
    oracle.ok_muhash_init(ctypes.byref(mh[genesis]))

    def validate(st, tx, pov, flags):
        ents = [st.get((i["txid"], i["index"])) for i in tx["inputs"]]
        if any(e is None for e in ents):
            return None, ents  # MissingTxOutpoints
        r = oracle_tx.validate_populated(oracle, build_batch([tx], [ents]), 0, pov, flags, prm)
        return (r if int(r["status"]) == 0 else None), ents

    for k, h in enumerate(order[1:], 1):
        b, s = by[h], sp(h)
        st = dict(state[s])
        m = OkMuHash()
        ctypes.memmove(ctypes.byref(m), ctypes.byref(mh[s]), ctypes.sizeof(m))
        pov = b["daa_score"]

        def add(txid, i, o, coinbase):
            st[(txid, i)] = {"amount": o["value"], "spk_version": o["spk_version"], "script": o["script"], "block_daa_score": pov, "is_coinbase": coinbase}
            d = pyref.utxo_element_bytes(txid, i, pov, o["value"], coinbase, o["spk_version"], o["script"])
            oracle.ok_muhash_add_element(ctypes.byref(m), d, len(d))

        cb = by[s]["txs"][0]
        cid = pyref.tx_id(cb)
        for i, o in enumerate(cb["outputs"]):
            add(cid, i, o, True)
        ms = ordered_mergeset(h)
        n_non_daa = len(ms) - (b["daa_score"] - by[s]["daa_score"])
        merged = []
        for j, mb in enumerate(ms):
            txs = by[mb]["txs"]
            acc, fees = [False] * len(txs), [0] * len(txs)
            for i in range(1, len(txs)):
                r, ents = validate(st, txs[i], pov, 1 if j == 0 else 0)  # selected parent: SkipScriptChecks
                if r is None:
                    continue
                acc[i], fees[i] = True, int(r["fee"])
                for x, e in zip(txs[i]["inputs"], ents):
                    del st[(x["txid"], x["index"])]
                    d = pyref.utxo_element_bytes(x["txid"], x["index"], e["block_daa_score"], e["amount"], e["is_coinbase"], e["spk_version"], e["script"])
                    oracle.ok_muhash_remove_element(ctypes.byref(m), d, len(d))
                tid = pyref.tx_id(txs[i])
                for i2, o in enumerate(txs[i]["outputs"]):
                    add(tid, i2, o, False)
            merged.append({"txs": txs, "accepted": acc, "fees": fees, "flags": oc.NON_DAA if (n_non_daa and mb == genesis) else 0})
        mm = OkMuHash()
        ctypes.memmove(ctypes.byref(mm), ctypes.byref(m), ctypes.sizeof(m))
        commitment = ctypes.create_string_buffer(32)
        oracle.ok_muhash_finalize(ctypes.byref(mm), commitment)
        # check 5: the chain block's own transactions against its UTXO view (Full)
        tx_ok = [validate(st, tx, pov, 0)[0] is not None for tx in b["txs"][1:]]
        header = {"utxo_commitment": bytes.fromhex(b["utxo_commitment"]), "accepted_id_merkle_root": bytes.fromhex(b["accepted_id_merkle_root"]),
                  "selected_parent_accepted_id_merkle_root": bytes.fromhex(by[s]["accepted_id_merkle_root"]), "blue_score": b["blue_score"],
                  "expected_subsidy": oracle_body.SIMPA_SUBSIDY}
        yield (merged, b["txs"], tx_ok, header, commitment.raw), (b, by[s], ms, n_non_daa)
        state[h], mh[h] = st, m
        if last_use.get(s, 0) <= k:
            del state[s], mh[s]


@pytest.mark.parametrize("fixture,n_blocks", [("simpa_goref_1060.json.gz", 265), ("simpa_goref_pruning_5000.json.gz", 5000)])
def test_every_block_reproduces_its_header_and_coinbase(oracle, fixture, n_blocks):
    n = n_non_daa_children = n_reward_outputs = 0
    for args, (b, spb, ms, n_non_daa) in chain_block_inputs(oracle, fixture):
        assert b["blue_score"] - spb["blue_score"] == len(ms), b["hash"]  # all-blue mergesets
        assert n_non_daa in (0, 1) and (n_non_daa == 1) == (ms == [ms[0]] and not spb["parents"]), b["hash"]  # genesis only
        res, fees = oc.verify_chain_block(*args, MAX_PAYLOAD_LEN, MAX_SPK_LEN)
        assert res["status"] == 0 and res["n_invalid_txs"] == 0, (b["hash"], res)
        assert res["coinbase_hash"] == pyref.tx_hash(b["txs"][0]), b["hash"]
        assert res["utxo_commitment"].hex() == b["utxo_commitment"] and res["accepted_id_merkle_root"].hex() == b["accepted_id_merkle_root"]
        if n_non_daa:
            n_non_daa_children += 1
            assert b["txs"][0]["outputs"] == []
        n_reward_outputs += len(b["txs"][0]["outputs"])
        n += 1
    assert n == n_blocks and n_non_daa_children >= 1 and n_reward_outputs > n_blocks


def test_expected_coinbase_statuses_follow_the_reference_order():
    """the panics and their positions on hand-made rewards: overflow of a blue's sum, of the red sum, a non-DAA red's fees only"""
    pay = oracle_body.coinbase_payload(7, 50, b"\x20" + bytes(32) + b"\xac", 0, b"extra")
    big = (1 << 64) - 1
    cb = oc.expected_coinbase_transaction([(3, 4, 0, b"\x51", 0), (5, 6, 0, b"\x52", oc.RED), (9, 10, 0, b"\x53", oc.RED | oc.NON_DAA)], 7, 50, pay,
                                          MAX_PAYLOAD_LEN, MAX_SPK_LEN)
    assert [o["value"] for o in cb["outputs"]] == [7, 21] and cb["outputs"][1]["script"] == b"\x20" + bytes(32) + b"\xac"
    assert cb["payload"] == pay
    for rewards in ([(big, 1, 0, b"", 0)], [(big, 0, 0, b"", oc.RED), (1, 0, 0, b"", oc.RED)], [(0, big, 0, b"", oc.RED | oc.NON_DAA), (0, 1, 0, b"", oc.RED)]):
        with pytest.raises(oc.ChainPanic) as e:
            oc.expected_coinbase_transaction(rewards, 7, 50, pay, MAX_PAYLOAD_LEN, MAX_SPK_LEN)
        assert e.value.status == oc.STATUS["RewardOverflow"]
    # a non-DAA blue's sum is never formed: no panic, no output
    assert oc.expected_coinbase_transaction([(big, 1, 0, b"", oc.NON_DAA)], 7, 50, pay, MAX_PAYLOAD_LEN, MAX_SPK_LEN)["outputs"] == []
    with pytest.raises(oc.ChainPanic) as e:
        oc.expected_coinbase_transaction([], 7, 50, pay[:18], MAX_PAYLOAD_LEN, MAX_SPK_LEN)
    assert e.value.status == oc.STATUS["CoinbasePayloadUnparsable"]
