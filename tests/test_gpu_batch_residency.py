"""A transaction batch's arrays are all host pointers or all device pointers (include/kgv.h, kgv_tx_batch): a batch that mixes the two
is refused with KGV_ERR_ARG before anything is copied or launched, and the same data on one side gives the bytes of the host call."""
import ctypes

import numpy as np
import pytest

KGV_ERR_ARG = -1
FIELDS = ("txs", "inputs", "outputs", "entries", "bytes")
# which arrays sit in device memory: txs alone, and everything but txs
MIXED = [("txs",), ("inputs", "outputs", "entries", "bytes")]


def _c_batch(b, on_device, keep):
    import torch
    from rusty_kaspa_b200.verifier import _KgvTxBatch
    arrays = {"txs": b.txs, "inputs": b.inputs, "outputs": b.outputs, "entries": b.entries, "bytes": b.arena}

    def ptr(name):
        a = arrays[name]
        if a is None:
            return None
        if name in on_device:
            t = torch.from_numpy(np.ascontiguousarray(a).view(np.uint8).reshape(-1).copy()).cuda()
            keep.append(t)
            return t.data_ptr()
        return a.ctypes.data
    return _KgvTxBatch(ptr("txs"), len(b.txs), ptr("inputs"), len(b.inputs), ptr("outputs"), len(b.outputs), ptr("entries"), ptr("bytes"), len(b.arena))


def _window():
    from rusty_kaspa_b200 import simgen
    from rusty_kaspa_b200.replay import REPLAY_BLOCK_DTYPE
    g = simgen.FastDag(seed=5, n_keys=32, n_nonces=64, coinbase_maturity=3, mix=(0.5, 0.2, 0.15, 0.15), frac_invalid=0.1, coinbase_outputs=4)
    g.generate(12, 8)
    b, first, pov = g.take()
    C = g.C
    g.close()
    blocks = np.zeros(len(pov), dtype=REPLAY_BLOCK_DTYPE)
    blocks["first_tx"], blocks["n_txs"], blocks["pov_daa_score"], blocks["flags"] = first[:-1], np.diff(first), pov, 1
    return b, blocks, C


def _calls(ctx, b, blocks, C):
    """name -> fn(batch struct) -> (rc, output bytes); each call gets a fresh UTXO table where it needs one"""
    from rusty_kaspa_b200 import Params
    from rusty_kaspa_b200.replay import DagReplayer, RESULT_DTYPE
    lib = ctx._lib
    params = Params(coinbase_maturity=3, storage_mass_parameter=C)

    def tx_ids(cb):
        out = np.zeros((b.n_txs, 32), dtype=np.uint8)
        return lib.kgv_tx_ids(ctx._h, ctypes.byref(cb), out.ctypes.data), out.tobytes()

    def validate_txs(cb):
        rp = DagReplayer(ctx, params, 1 << 12)
        res = np.zeros(b.n_txs, dtype=RESULT_DTYPE)
        rc = lib.kgv_validate_txs(ctx._h, rp.us._h, ctypes.byref(cb), 10, 0, ctypes.byref(rp.tv.params), res.ctypes.data)
        rp.close()
        return rc, res.tobytes()

    def replay_window(cb):
        rp = DagReplayer(ctx, params, 1 << 12)
        res = np.zeros(b.n_txs, dtype=RESULT_DTYPE)
        acc = np.zeros(b.n_txs, dtype=np.uint8)
        rc = lib.kgv_replay_window(ctx._h, rp.us._h, ctypes.byref(cb), blocks.ctypes.data, len(blocks), ctypes.byref(rp.tv.params), res.ctypes.data,
                                   acc.ctypes.data, None)
        out = res.tobytes() + acc.tobytes() + rp.us.digest()
        rp.close()
        return rc, out
    return {"kgv_tx_ids": tx_ids, "kgv_validate_txs": validate_txs, "kgv_replay_window": replay_window}


@pytest.mark.gpu
@pytest.mark.parametrize("on_device", MIXED, ids=["txs-device", "txs-host"])
def test_mixed_batch_is_refused(on_device):
    import rusty_kaspa_b200 as rk
    b, blocks, C = _window()
    ctx = rk.GpuContext(0)
    keep = []
    for name, call in _calls(ctx, b, blocks, C).items():
        rc, _ = call(_c_batch(b, on_device, keep))
        assert rc == KGV_ERR_ARG, name
        assert "kgv_tx_batch" in ctx._lib.kgv_last_error(ctx._h).decode(), name
    ctx.close()


@pytest.mark.gpu
def test_one_sided_batch_gives_the_host_bytes():
    import rusty_kaspa_b200 as rk
    b, blocks, C = _window()
    ctx = rk.GpuContext(0)
    keep = []
    for name, call in _calls(ctx, b, blocks, C).items():
        rc_h, host = call(_c_batch(b, (), keep))
        rc_d, dev = call(_c_batch(b, FIELDS, keep))
        assert rc_h == 0 and rc_d == 0, (name, ctx._lib.kgv_last_error(ctx._h).decode())
        assert dev == host, name
    ctx.close()
