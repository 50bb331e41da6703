"""The CPU restatement of the block body rules (oracle_body.py) against the reference's own data: both DAG fixtures with their real header
values, and the example block of validate_body_in_isolation_test with every mutation that test applies."""
import oracle_body as ob
import oracle_isolation as oi

MAX_BLOCK_MASS, MAX_COINBASE_PAYLOAD_LEN = 500_000, 204  # MAINNET_PARAMS; the DAG fixtures were generated with the same two values


def _accepts_every_block(name, n_blocks):
    blocks = ob.fixture_blocks(name)
    assert len(blocks) == n_blocks
    rules = oi.mainnet_rules()
    # the first block is the DAG's genesis, which the reference stores without validating its body: the isolation rules hold for it, the
    # context stage (its payload carries the genesis subsidy, not a block subsidy) is run for every other block
    verdicts = ob.ok_validate_bodies(blocks[:1], rules, MAX_BLOCK_MASS, MAX_COINBASE_PAYLOAD_LEN, isolation_only=True)
    verdicts += ob.ok_validate_bodies(blocks[1:], rules, MAX_BLOCK_MASS, MAX_COINBASE_PAYLOAD_LEN)
    for k, (verdict, masses) in enumerate(verdicts):
        assert verdict == ob.OK, (k, ob.NAME[verdict["status"]], verdict)
        txs = blocks[k]["transactions"]
        assert masses[0] == sum(oi.ok_tx_non_contextual_masses(t, rules)[0] for t in txs) and masses[2] == sum(t["mass"] for t in txs)


def test_every_block_of_the_265_block_dag_passes():
    _accepts_every_block("simpa_goref_1060.json.gz", 266)


def test_every_block_of_the_5000_block_dag_passes():
    _accepts_every_block("simpa_goref_pruning_5000.json.gz", 5001)


def test_reference_example_block_and_its_mutations():
    """validate_body_in_isolation_test (:409-460): Ok, then the eight errors the test asserts, in its order"""
    cases = ob.reference_example_blocks()
    assert [c[2] for c in cases] == ["Ok"] + list(ob.REFERENCE_MUTATIONS)
    rules = oi.mainnet_rules()
    for name, block, err in cases:
        verdict, masses = ob.ok_validate_body(block, rules, MAX_BLOCK_MASS, MAX_COINBASE_PAYLOAD_LEN, isolation_only=True)
        assert ob.NAME[verdict["status"]] == err, (name, verdict)
        assert (masses != (0, 0, 0)) == (err == "Ok")
    by = {c[0]: ob.ok_validate_body(c[1], rules, MAX_BLOCK_MASS, MAX_COINBASE_PAYLOAD_LEN, isolation_only=True)[0] for c in cases}
    assert by["MultipleCoinbases"]["index"] == 0  # txs[1] is position 0 of transactions[1..]
    assert by["TxInIsolationValidationFailed"]["index"] == 1 and by["TxInIsolationValidationFailed"]["tx_status"] == oi.STATUS["NoTxInputs"]
    assert by["ExceedsComputeMassLimit"]["index"] == 1 and by["ExceedsComputeMassLimit"]["a"] > by["ExceedsComputeMassLimit"]["b"] == MAX_BLOCK_MASS
    assert by["DuplicateTransactions"]["index"] == 5  # the pushed clone


def test_coinbase_payload_parse_order():
    """deserialize_coinbase_payload compares lengths before it reads: each error carries the reference's two numbers"""
    p = ob.coinbase_payload(7, 9, bytes(34))
    assert ob.deserialize_coinbase_payload(p, 204, 150) == (7, 9)
    for payload, max_len, max_spk, want in [(p[:18], 204, 150, (1, 18, 19)), (p + bytes(200), 204, 150, (2, len(p) + 200, 204)),
                                           (p, 204, 33, (3, 34, 33)), (p[:-1], 204, 150, (4, len(p) - 1, 19 + 34))]:
        try:
            ob.deserialize_coinbase_payload(payload, max_len, max_spk)
            assert False, want
        except ob.BodyError as e:
            assert (e.verdict["tx_status"], e.verdict["a"], e.verdict["b"]) == want


def test_context_rules_follow_the_isolation_rules():
    """validate_body_in_context on the example block: blue score, then subsidy, then the first transaction that is not final"""
    _, block, _ = ob.reference_example_blocks()[0]
    rules = oi.mainnet_rules()
    run = lambda b: ob.ok_validate_body(b, rules, MAX_BLOCK_MASS, MAX_COINBASE_PAYLOAD_LEN)[0]
    blue = int.from_bytes(block["transactions"][0]["payload"][:8], "little")
    assert ob.NAME[run(block)["status"]] == "BadCoinbasePayloadBlueScore" and run(block)["a"] == blue
    block["blue_score"] = blue
    assert run(block) == ob.OK
    assert run(dict(block, expected_subsidy=5)) == dict(ob.OK, status=ob.STATUS["WrongSubsidy"], a=5, b=0)
    block["transactions"][2]["lock_time"] = 100
    block["transactions"][2]["inputs"][0]["sequence"] = 0
    block["hash_merkle_root"] = ob.calc_hash_merkle_root(block["transactions"])
    assert run(dict(block, daa_score=101)) == ob.OK
    assert run(dict(block, daa_score=100)) == dict(ob.OK, status=ob.STATUS["TxInContextFailed"], index=2, tx_status=oi.STATUS["NotFinalized"])
