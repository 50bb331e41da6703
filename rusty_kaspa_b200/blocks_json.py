"""Reader for the reference's gzip-JSON block dumps (SURVEY.md §8f-4): the format `simpa --output-json` writes and the
integration tests replay (testing/integration/src/common/json.rs:27-40, simpa/src/blocks_json.rs:13-39;
e.g. testing/integration/testdata/dags_for_json_tests/*/blocks.json.gz): first line = consensus params, every further
line = one block {header, transactions}.  Produces the tx dict layout used by txbatch.build_batch / replay.DagReplayer, so a
real simpa or mainnet dump can be fed to the GPU path directly."""
import gzip
import json


def _tx(t):
    spk = lambda o: (int(o["scriptPublicKey"][:4], 16), bytes.fromhex(o["scriptPublicKey"][4:]))  # u16 version (big-endian hex) || script
    return {"version": t["version"],
            "inputs": [{"txid": bytes.fromhex(i["previousOutpoint"]["transactionId"]), "index": i["previousOutpoint"]["index"],
                        "sigscript": bytes.fromhex(i["signatureScript"]), "sequence": i["sequence"], "sig_op_count": i["sigOpCount"]} for i in t["inputs"]],
            "outputs": [{"value": o["value"], "spk_version": spk(o)[0], "script": spk(o)[1]} for o in t["outputs"]],
            "lock_time": t["lockTime"], "subnetwork_id": bytes.fromhex(t["subnetworkId"]), "gas": t["gas"],
            "payload": bytes.fromhex(t["payload"]), "mass": t.get("mass", 0)}


def header_from_json(h):
    """One JSON header (simpa/src/blocks_json.rs field names) -> the header dict of headers.HeaderBatch: every field the header hash
    covers, parents_by_level expanded (one list of 32-byte hashes per level), blue_work as an int, plus its stored "hash"."""
    return {"hash": bytes.fromhex(h["hash"]), "version": h["version"],
            "parents_by_level": [[bytes.fromhex(p) for p in lvl] for lvl in h["parentsByLevel"]],
            "hash_merkle_root": bytes.fromhex(h["hashMerkleRoot"]), "accepted_id_merkle_root": bytes.fromhex(h["acceptedIdMerkleRoot"]),
            "utxo_commitment": bytes.fromhex(h["utxoCommitment"]), "timestamp": h["timestamp"], "bits": h["bits"], "nonce": h["nonce"],
            "daa_score": h["daaScore"], "blue_work": int(h["blueWork"] or "0", 16), "blue_score": h["blueScore"],
            "pruning_point": bytes.fromhex(h["pruningPoint"])}


def load_headers_json(path):
    """Returns (params dict, list of header dicts (header_from_json)) in file order, from a blocks.json(.gz) dump or a headers-only
    file of the same line format (first line params, then one {"header": ...} per line)."""
    opener = gzip.open if str(path).endswith(".gz") else open
    with opener(path, "rt") as f:
        lines = [l for l in f.read().splitlines() if l.strip()]
    return json.loads(lines[0]), [header_from_json(json.loads(l)["header"]) for l in lines[1:]]


def load_blocks_json(path):
    """Returns (params dict, list of blocks); a block = {"hash", "daa_score", "blue_score", "hash_merkle_root",
    "accepted_id_merkle_root", "utxo_commitment", "parents" (level 0), "transactions" (tx dicts)} in file (topological) order."""
    opener = gzip.open if str(path).endswith(".gz") else open
    with opener(path, "rt") as f:
        lines = [l for l in f.read().splitlines() if l.strip()]
    params = json.loads(lines[0])
    blocks = []
    for l in lines[1:]:
        b = json.loads(l)
        h = b["header"]
        blocks.append({"hash": bytes.fromhex(h["hash"]), "daa_score": h["daaScore"], "blue_score": h["blueScore"],
                       "hash_merkle_root": bytes.fromhex(h["hashMerkleRoot"]),
                       "accepted_id_merkle_root": bytes.fromhex(h["acceptedIdMerkleRoot"]), "utxo_commitment": bytes.fromhex(h["utxoCommitment"]),
                       "parents": [bytes.fromhex(p) for p in (h["parentsByLevel"][0] if h["parentsByLevel"] else [])],
                       "transactions": [_tx(t) for t in b["transactions"]]})
    return params, blocks
