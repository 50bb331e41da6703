"""The standardness methods of the C++ host mirror (include/kgv.hpp) driven by tests/cpp/standard_mirror_test.cpp on the reference's own cases
(tests/golden/standard_cases.json): every printed verdict is compared with the CPU restatement (oracle_standard.py), and the fused call's
output with the Python mirror's on the same batch."""
import os
import subprocess
import sys

import numpy as np
import pytest

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
sys.path.insert(0, HERE)
import oracle_standard as os_  # noqa: E402
from test_gpu_standard import P2PK, _ent, _masses, _tx  # noqa: E402

pytestmark = pytest.mark.gpu


def _dump(d, name, b):
    for part, arr in (("txs", b.txs), ("inputs", b.inputs), ("outputs", b.outputs), ("entries", b.entries), ("arena", b.arena)):
        np.ascontiguousarray(arr).tofile(os.path.join(d, "%s_%s.bin" % (name, part)))


def test_cpp_standard_methods(tmp_path, gpu_ctx):
    from rusty_kaspa_b200 import GpuUtxoSet, MempoolPolicy, TransactionValidator
    from rusty_kaspa_b200.txbatch import build_batch
    binary = str(tmp_path / "standard_mirror_test")
    subprocess.run(["g++", "-O2", "-std=c++17", "-o", binary, os.path.join(HERE, "cpp", "standard_mirror_test.cpp"), "-L" + os.path.join(ROOT, "rusty_kaspa_b200"),
                    "-l:libkgv.so", "-Wl,-rpath," + os.path.join(ROOT, "rusty_kaspa_b200")], check=True)
    g = os_.golden()
    d = str(tmp_path)
    p = os_.Policy()
    # in isolation: the reference's seven transactions with their masses
    iso = [os_.tx_from_golden(c["tx"]) for c in g["isolation"]["cases"]]
    iso_m = [(c["compute_mass"], c["transient_mass"]) for c in g["isolation"]["cases"]]
    _dump(d, "iso", build_batch(iso))
    _masses(iso_m).tofile(os.path.join(d, "iso_masses.bin"))
    # in context: the relay-fee rows, one standard input, compute mass = size, the fee one below the minimum (at the default relay fee)
    rows = g["relay_fee"]["rows"]
    ctx_m = [(r["size"], 0) for r in rows]
    ctx_fee = [os_.minimum_required_transaction_relay_fee(r["size"], p.fee) - 1 + (k % 2) for k, r in enumerate(rows)]
    _dump(d, "ctx", build_batch([_tx() for _ in rows], [[_ent()] for _ in rows]))
    _masses(ctx_m).tofile(os.path.join(d, "ctx_masses.bin"))
    np.zeros(len(rows), np.uint64).tofile(os.path.join(d, "ctx_smass.bin"))
    np.array(ctx_fee, np.uint64).tofile(os.path.join(d, "ctx_fee.bin"))
    # dust: the reference's rows as the outputs of one transaction (at the default relay fee)
    drows = g["dust"]["rows"]
    dust_tx = _tx(n_out=len(drows))
    for o, r in zip(dust_tx["outputs"], drows):
        o.update(value=r["value"], script=bytes.fromhex(r["script"]))
    _dump(d, "dust", build_batch([dust_tx]))
    # the fused call: the isolation cases (and two standard spends) with their entries supplied, against an empty UTXO set
    pol_txs = iso + [_tx(), _tx(sig=b"")]
    pol_ents = [[_ent() for _ in t["inputs"]] for t in pol_txs]
    pb = build_batch(pol_txs, pol_ents)
    _dump(d, "pol", pb)
    out = subprocess.run([binary, d, str(p.fee)], capture_output=True, text=True, timeout=300)
    assert out.returncode == 0, out.stdout + out.stderr
    lines = [l.split() for l in out.stdout.split("\n") if l]
    by = lambda tag: [[int(x) for x in l[2:]] for l in lines if l[0] == tag]
    assert lines[-1] == ["threw"]
    assert by("iso") == [list(os_.check_in_isolation(t, m[0], m[1], p)) for t, m in zip(iso, iso_m)]
    assert [os_.NAME[r[0]] for r in by("iso")] == [os_.ISOLATION_EXPECTED[c["name"]][0] for c in g["isolation"]["cases"]]
    exp_ctx = [list(os_.check_in_context(_tx(), [_ent()], 0, m[0], f, p)) + [f] for m, f in zip(ctx_m, ctx_fee)]
    assert by("ctx") == exp_ctx and {r[0] for r in exp_ctx} == {0, 42}
    assert by("dust") == [[int(os_.is_transaction_output_dust(r["value"], bytes.fromhex(r["script"]), p.fee))] for r in drows]
    # the fused method equals the Python mirror on the same batch
    tv = TransactionValidator(gpu_ctx)
    us = GpuUtxoSet(gpu_ctx, 1 << 10)
    try:
        res, mass, masses, _, _, det = tv.validate_mempool_transactions_with_policy(us, pb, 1000, 0, MempoolPolicy(p.fee), supplied=np.ones(len(pb.inputs), bool))
    finally:
        us.close()
    exp_pol = [[int(res["status"][k]), int(res["fail_input"][k]), int(det[k]), int(mass[k]), int(masses["compute_mass"][k]), int(masses["transient_mass"][k])]
               for k in range(len(pol_txs))]
    assert by("pol") == exp_pol
    assert {r[0] for r in exp_pol} >= {32, 37, 38}
