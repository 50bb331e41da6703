"""The CPU restatement of the standardness policy (oracle_standard.py) on the reference's own cases (tests/golden/standard_cases.json) and on
the quirks of its rule order."""
import pytest

import oracle_standard as os_

G = os_.golden()


def test_constants_match_the_reference():
    k = G["constants"]
    assert (k["MAX_STANDARD_P2SH_SIG_OPS"], k["MAXIMUM_STANDARD_SIGNATURE_SCRIPT_SIZE"], k["MAXIMUM_STANDARD_TRANSACTION_MASS"]) == (
        os_.MAX_STANDARD_P2SH_SIG_OPS, os_.MAXIMUM_STANDARD_SIGNATURE_SCRIPT_SIZE, os_.MAXIMUM_STANDARD_TRANSACTION_MASS)
    assert k["DEFAULT_MINIMUM_RELAY_TRANSACTION_FEE"] == os_.DEFAULT_MINIMUM_RELAY_TRANSACTION_FEE and k["MAX_SOMPI"] == os_.MAX_SOMPI
    assert k["DEFAULT_MINIMUM_STANDARD_TRANSACTION_VERSION"] == k["DEFAULT_MAXIMUM_STANDARD_TRANSACTION_VERSION"] == k["TX_VERSION"] == 0


def test_relay_fee_rows():
    rows = G["relay_fee"]["rows"]
    assert len(rows) == 8
    for r in rows:
        assert os_.minimum_required_transaction_relay_fee(r["size"], r["minimum_relay_transaction_fee"]) == r["want"], r["name"]


def test_dust_rows():
    rows = G["dust"]["rows"]
    assert len(rows) == 7
    for r in rows:
        assert os_.is_transaction_output_dust(r["value"], bytes.fromhex(r["script"]), r["minimum_relay_transaction_fee"]) == r["is_dust"], r["name"]


def test_isolation_cases():
    cases = G["isolation"]["cases"]
    assert [c["name"] for c in cases] == list(os_.ISOLATION_EXPECTED)
    for c in cases:
        tx = os_.tx_from_golden(c["tx"])
        st, idx, _ = os_.check_in_isolation(tx, c["compute_mass"], c["transient_mass"], os_.Policy())
        assert (st == 0) == c["is_standard"], c["name"]
        assert (os_.NAME[st], idx) == os_.ISOLATION_EXPECTED[c["name"]], c["name"]
    big = next(c for c in cases if c["name"] == "Transaction size is too large")
    assert len(os_.tx_from_golden(big["tx"])["outputs"][0]["script"]) == 100_001


P2PK = bytes([0x20]) + bytes(32) + bytes([0xac])
P2SH = bytes([0xaa, 0x20]) + bytes(32) + bytes([0x87])


def _tx(n_in):
    return {"version": 0, "inputs": [{"sigscript": b"", "sequence": 0, "sig_op_count": 1, "txid": bytes(32), "index": 0} for _ in range(n_in)],
            "outputs": []}


def test_fee_check_sits_between_input_0_and_input_1():
    p = os_.Policy()
    bad = {"spk_version": 0, "script": b"\x51"}
    good = {"spk_version": 0, "script": P2PK}
    # input 0 non-standard, fee too low: the input's verdict
    assert os_.check_in_context(_tx(2), [bad, good], 0, 1000, 0, p)[:2] == (os_.STATUS["RejectInputScriptClass"], 0)
    # input 1 non-standard, fee too low: the fee's verdict
    assert os_.check_in_context(_tx(2), [good, bad], 0, 1000, 0, p) == (os_.STATUS["RejectInsufficientFee"], 0, 1000)
    # no inputs: the fee is never checked
    assert os_.check_in_context(_tx(0), [], 0, 1000, 0, p) == (0, 0, 0)
    assert os_.check_in_context(_tx(2), [good, bad], 0, 1000, 1000, p)[:2] == (os_.STATUS["RejectInputScriptClass"], 1)
    assert os_.check_in_context(_tx(1), [good], 100_001, 1000, 0, p) == (os_.STATUS["RejectStorageMass"], 0, 100_001)
    with pytest.raises(OverflowError):
        os_.check_in_context(_tx(1), [good], 0, 2, 0, os_.Policy(minimum_relay_transaction_fee=2**63))


def test_sig_op_bound_edges():
    push = lambda d: (bytes([len(d)]) if len(d) <= 75 else bytes([0x4c, len(d)])) + d
    assert os_.sig_op_count_upper_bound_p2sh(b"") == 0
    assert os_.sig_op_count_upper_bound_p2sh(push(b"\xac" * 16)) == 16
    assert os_.sig_op_count_upper_bound_p2sh(b"\x51" + push(b"\xac" * 16)) == 16
    assert os_.sig_op_count_upper_bound_p2sh(b"\x61" + push(b"\xac" * 16)) == 0  # not push-only
    assert os_.sig_op_count_upper_bound_p2sh(push(b"\xac" * 16) + b"\x05\x01") == 0  # parse error
    assert os_.sig_op_count_upper_bound_p2sh(push(b"\xac" * 16) + b"\x51") == 0  # a small int pushes no data
    assert os_.sig_op_count_upper_bound_p2sh(push(b"\xae")) == 20  # multisig first
    assert os_.sig_op_count_upper_bound_p2sh(push(b"\x53\xae")) == 3
    assert os_.sig_op_count_upper_bound_p2sh(push(b"\x60\xae")) == 16  # the reference panics here
    assert os_.sig_op_count_upper_bound_p2sh(push(b"\x00\xae")) == 20
    assert os_.sig_op_count_upper_bound_p2sh(push(b"\xac\xac\x4d\x05")) == 2  # the redeem walk stops at its parse error
