"""The CPU restatement of the isolation rules, lock-time finality and non-contextual masses (oracle_isolation.py) against the reference's own
cases, extracted into tests/golden/isolation_cases.json."""
import json
import os

import oracle_isolation as oi
from rusty_kaspa_b200.validator import TxRules

HERE = os.path.dirname(os.path.abspath(__file__))


def test_reference_isolation_cases():
    """validate_tx_in_isolation_test: every mutated transaction gives the reference's error class (and Ok where it expects Ok)"""
    cases, rules = oi.isolation_golden_cases()
    assert len(cases) == 12 and rules["max_tx_inputs"] == 10 and rules["max_tx_outputs"] == 15
    for name, tx, err in cases:
        st, idx = oi.ok_tx_isolation(tx, rules)
        assert oi.NAME[st] == err, (name, oi.NAME[st], err)
        if err in ("TooBigSignatureScript", "TooBigScriptPublicKey"):
            assert idx == 0, name  # the test mutates input / output 0


def test_reference_finality_cases():
    """check_for_lock_time_and_sequence: lock time at the context value or above fails with NotFinalized(0), below passes, u64::MAX sequences
    pass any lock time; against the DAA score and against the past median time"""
    cases = oi.finality_golden_cases()
    assert len(cases) == 8 and {c[1]["lock_time"] >= oi.LOCK_TIME_THRESHOLD for c in cases} == {False, True}
    for name, tx, err, daa, pmt in cases:
        st, idx = oi.ok_tx_finality(tx, daa, pmt)
        assert oi.NAME[st] == err and idx == 0, (name, oi.NAME[st], err)


def test_mainnet_rules_match_the_python_defaults():
    """TxRules() carries the reference's mainnet values (extracted with the fixture)"""
    g = oi.golden()
    r = TxRules()
    for k, v in oi.mainnet_rules(g).items():
        assert getattr(r, k) == v, k
    m = g["mainnet"]
    assert (m["MAX_SOMPI"], m["LOCK_TIME_THRESHOLD"], m["TRANSIENT_BYTE_TO_MASS_FACTOR"], m["TX_VERSION"]) == \
        (oi.MAX_SOMPI, oi.LOCK_TIME_THRESHOLD, oi.TRANSIENT_BYTE_TO_MASS_FACTOR, oi.TX_VERSION)


def test_golden_block_masses():
    """the transactions of validate_body_in_isolation_test's block: the coinbase has masses (0, 0); every other one passes isolation and
    its masses follow the size estimate (the block passes the reference's mainnet block mass limit of 500 000 with them)"""
    with open(os.path.join(HERE, "golden", "body_validation_block.json")) as f:
        blk = json.load(f)
    txs = [oi._tx_from_json(t) for t in blk["txs"]]
    rules = oi.mainnet_rules()
    masses = [oi.ok_tx_non_contextual_masses(t, rules) for t in txs]
    assert oi.is_coinbase(txs[0]) and masses[0] == (0, 0)
    total_compute = 0
    for t, (c, tr) in zip(txs[1:], masses[1:]):
        assert oi.ok_tx_isolation(t, rules) == (0, 0)
        size = oi.estimated_serialized_size(t)
        assert tr == 4 * size and c == size + 10 * sum(2 + len(o["script"]) for o in t["outputs"]) + 1000 * sum(i["sig_op_count"] for i in t["inputs"])
        total_compute += c
    assert 0 < total_compute <= 500_000


def test_wrapping_masses():
    """u64 wrap-around as in a release build: a mass_per_tx_byte of 2^63 times an even size wraps to 0"""
    _, rules = oi.isolation_golden_cases()
    tx = oi.isolation_golden_cases()[0][1][1]
    size = oi.estimated_serialized_size(tx)
    assert size % 2 == 0
    c, _ = oi.ok_tx_non_contextual_masses(tx, dict(rules, mass_per_tx_byte=1 << 63, mass_per_script_pub_key_byte=0, mass_per_sig_op=0))
    assert c == 0
