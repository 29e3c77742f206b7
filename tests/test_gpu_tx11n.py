"""GPU parity tests for the 802.11n two-stream transmit path (pytest -m gpu): CUDA modulator through the C ABI against
oracle/tx11n.cpp, the reference-shaped frames through the CUDA receive path, and the on-device loop-back TX -> RX."""
import numpy as np, pytest
import oracle_py
from sora_b200 import api

pytestmark = pytest.mark.gpu

@pytest.fixture(scope="module")
def eng():
    return api.Engine(0)

@pytest.mark.parametrize("mcs", [8, 9, 10])
def test_tx_matches_oracle_bit_exact(eng, mcs):
    rng = np.random.default_rng(mcs + 40)
    lens = [1, 2, 3, 13, 14, 37, 200, 333, 1496, 57, 1000, 2000]
    pay = [rng.integers(0, 256, L).astype(np.uint8) for L in lens]
    seeds = np.array([0xAB, 0x5B, 0x02, 0x80, 0xFE, 0x13, 0xFF, 0x6D, 0x00, 0x01, 0xAB, 0x7F], np.uint8)
    o0, o1, ns = eng.tx11n_batch(pay, mcs, seeds=seeds)
    for i, p in enumerate(pay):
        w0, w1 = oracle_py.tx11n_modulate(p, mcs, int(seeds[i]))
        assert ns[i] == len(w0), (i, ns[i], len(w0))
        for got, want, name in ((o0[i], w0, "stream 0"), (o1[i], w1, "stream 1")):
            bad = np.nonzero((got[:len(want)] != want).any(1))[0]
            assert len(bad) == 0, (mcs, lens[i], name, bad[:10], got[bad[:4]], want[bad[:4]])
            assert (got[len(want):] == 0).all()

def test_default_seed_and_lead(eng):
    p = [np.arange(100, dtype=np.uint8)]
    o0, o1, ns = eng.tx11n_batch(p, 9, lead=77)
    w0, w1 = oracle_py.tx11n_modulate(p[0], 9)
    assert ns[0] == 77 + len(w0) and (o0[0, :77] == 0).all() and (o1[0, :77] == 0).all()
    assert (o0[0, 77:ns[0]] == w0).all() and (o1[0, 77:ns[0]] == w1).all()
    with pytest.raises(RuntimeError): eng.tx11n_batch(p, 15)              # MCS 15 (rate 5/6) ends in TDropAny in the reference's graph too (fb11nmod_config.hpp:153-154)
    with pytest.raises(RuntimeError): eng.tx11n_batch(p, 8, out_stride=1000)

def test_reference_shaped_frames_through_the_receive_path(eng):
    """Frames made by the restated reference modulator, mixed through a 2x2 channel with noise: CUDA receive path == receive oracle."""
    rng = np.random.default_rng(5); slots0, slots1 = [], []
    for mcs, L in ((8, 100), (9, 700), (10, 1496), (8, 33), (10, 60), (9, 1)):
        a, b = oracle_py.tx11n_modulate(rng.integers(0, 256, L).astype(np.uint8), mcs)
        ca = a[:, 0] + 1j * a[:, 1]; cb = b[:, 0] + 1j * b[:, 1]
        r0 = ca + 0.3j * cb; r1 = -0.2 * ca + 0.9 * cb
        def pk(r):
            x = np.concatenate([np.zeros((400, 2)), np.stack([r.real, r.imag], 1), np.zeros((300, 2))]) + rng.normal(0, 30, (len(r) + 700, 2))
            return np.clip(np.round(x), -32768, 32767).astype(np.int16)
        slots0.append(pk(r0)); slots1.append(pk(r1))
    off = np.cumsum([0] + [len(s) for s in slots0[:-1]]); ln = np.array([len(s) for s in slots0])
    iq0 = np.concatenate(slots0); iq1 = np.concatenate(slots1)
    res, out = eng.rx11n_batch(iq0, iq1, off, ln)
    ores, oout = oracle_py.rx11n_batch(iq0, iq1, off, ln, out_stride=out.shape[1])
    for k in ("status", "mcs", "length", "crc32", "nsym", "detect_index", "cfo_est", "lsig_length"):
        assert (res[k] == ores[k]).all(), (k, res[k], ores[k])
    assert (res["status"] == 1).all()
    for i in range(len(res)): assert (out[i, :res["length"][i]] == oout[i, :res["length"][i]]).all()

@pytest.mark.parametrize("mcs,L,F", [(8, 300, 64), (9, 1496, 128), (10, 1496, 128)])
def test_loopback_tx_to_rx_on_device(eng, mcs, L, F):
    """Modulate on the GPU into two COMPLEX16 slots per frame and decode them with the 802.11n receive path without leaving the device."""
    import torch
    rng = np.random.default_rng(mcs)
    pay = rng.integers(0, 256, (F, L)).astype(np.uint8)
    d_pay = torch.from_numpy(pay.reshape(-1)).cuda()
    d_off = torch.arange(F, dtype=torch.int64, device="cuda") * L; d_len = torch.full((F,), L, dtype=torch.int32, device="cuda")
    slot = (api.Engine.tx11n_out_stride(L, mcs, lead=400) + 300 + 27) // 28 * 28
    d0 = torch.empty((F, slot, 2), dtype=torch.int16, device="cuda"); d1 = torch.empty_like(d0); st = torch.cuda.current_stream().cuda_stream
    eng.tx11n_raw(d_pay.data_ptr(), F * L, d_off.data_ptr(), d_len.data_ptr(), 0, F, mcs, 400, d0.data_ptr(), d1.data_ptr(), slot, 0, st)
    s_off = torch.arange(F, dtype=torch.int64, device="cuda") * slot; s_len = torch.full((F,), slot, dtype=torch.int32, device="cuda")
    d_out = torch.zeros((F, 1536), dtype=torch.uint8, device="cuda"); d_res = torch.zeros((F, 7), dtype=torch.int32, device="cuda")
    eng.rx11n_raw(d0.data_ptr(), d1.data_ptr(), F * slot, s_off.data_ptr(), s_len.data_ptr(), F, d_out.data_ptr(), 1536, d_res.data_ptr(), st)
    torch.cuda.synchronize()
    res = d_res.cpu().numpy()
    assert (res[:, 0] == 1).all() and (res[:, 1] == mcs).all() and (res[:, 2] == L + 4).all(), res[:4]
    assert (d_out.cpu().numpy()[:, :L] == pay).all()
