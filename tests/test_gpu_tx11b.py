"""GPU parity tests for the 802.11b transmit path (pytest -m gpu): CUDA modulator through the C ABI against oracle/tx11b.cpp, and the
on-device loop-back TX -> RX."""
import numpy as np, pytest, zlib
import oracle_py
from sora_b200 import api

pytestmark = pytest.mark.gpu
RATES = [1000, 2000, 5500, 11000]

@pytest.fixture(scope="module")
def eng():
    return api.Engine(0)

@pytest.mark.parametrize("rate", RATES)
def test_tx_matches_oracle_bit_exact(eng, rate):
    rng = np.random.default_rng(rate + 5)
    lens = [1, 2, 13, 37, 200, 333, 1496, 57, 1000, 4091] if rate >= 5500 else [1, 2, 13, 37, 200, 333, 57]
    pay = [rng.integers(0, 256, L).astype(np.uint8) for L in lens]
    for phase in (0, 1, 2, 3):
        out, ns, fp = eng.tx11b_batch(pay, rate, init_phase=phase, return_phase=True)
        for i, p in enumerate(pay):
            want, fin = oracle_py.tx11b_modulate(p, rate, phase, return_phase=True)
            assert ns[i] == len(want) and fp[i] == fin, (i, ns[i], len(want), fp[i], fin)
            bad = np.nonzero((out[i, :len(want)] != want).any(1))[0]
            assert len(bad) == 0, (rate, phase, lens[i], bad[:10], out[i, bad[:4]], want[bad[:4]])
            assert (out[i, len(want):] == 0).all()

def test_tx_formats_and_lead(eng):
    p = [np.full(200, 0x31, np.uint8), np.arange(90, dtype=np.uint8)]
    for lead in (0, 3, 4, 8, 12, 101):
        o8, ns = eng.tx11b_batch(p, 11000, lead=lead, sample_bits=8)
        o16, ns16 = eng.tx11b_batch(p, 11000, lead=lead, sample_bits=16)
        for i in range(2):
            want = oracle_py.tx11b_modulate(p[i], 11000)
            assert ns[i] == lead + len(want) and ns16[i] == ns[i]
            assert (o8[i, :lead] == 0).all() and (o8[i, lead:ns[i]] == want).all() and (o8[i, ns[i]:] == 0).all()
            assert (o16[i, lead:ns[i]] == want.astype(np.int16) << 8).all() and (o16[i, :lead] == 0).all() and (o16[i, ns[i]:] == 0).all()

def test_bad_arguments(eng):
    p = [np.zeros(10, np.uint8)]
    with pytest.raises(RuntimeError): eng.tx11b_batch(p, 6000, out_stride=4096)
    with pytest.raises(RuntimeError): eng.tx11b_batch(p, 11000, out_stride=1001)          # not a multiple of 8
    with pytest.raises(RuntimeError): eng.tx11b_batch(p, 11000, out_stride=64)            # too small

@pytest.mark.parametrize("rate,L,F", [(11000, 1496, 256), (5500, 700, 64), (2000, 300, 32), (1000, 100, 32)])
def test_loopback_tx_to_rx_on_device(eng, rate, L, F):
    """Modulate on the GPU into COMPLEX16 slots at 44 Msps and decode them with the 802.11b receive path without leaving the device."""
    import torch
    rng = np.random.default_rng(rate)
    pay = rng.integers(0, 256, (F, L)).astype(np.uint8)
    d_pay = torch.from_numpy(pay.reshape(-1)).cuda()
    d_off = torch.arange(F, dtype=torch.int64, device="cuda") * L; d_len = torch.full((F,), L, dtype=torch.int32, device="cuda")
    slot = (api.Engine.tx11b_out_stride(L, rate, lead=304) + 600 + 55) // 56 * 56
    d_iq = torch.empty((F, slot, 2), dtype=torch.int16, device="cuda"); d_ns = torch.zeros(F, dtype=torch.int32, device="cuda")
    st = torch.cuda.current_stream().cuda_stream
    eng.tx11b_raw(d_pay.data_ptr(), F * L, d_off.data_ptr(), d_len.data_ptr(), F, rate, 0, 304, 16, d_iq.data_ptr(), slot, d_ns.data_ptr(), st)
    s_off = torch.arange(F, dtype=torch.int64, device="cuda") * slot; s_len = torch.full((F,), slot, dtype=torch.int32, device="cuda")
    d_out = torch.zeros((F, 2048), dtype=torch.uint8, device="cuda"); d_res = torch.zeros((F, 6), dtype=torch.int32, device="cuda")
    eng.rx11b_raw(d_iq.data_ptr(), F * slot, s_off.data_ptr(), s_len.data_ptr(), F, d_out.data_ptr(), 2048, d_res.data_ptr(), st)
    torch.cuda.synchronize()
    res = d_res.cpu().numpy()
    assert (res[:, 0] == 1).all() and (res[:, 1] == rate).all() and (res[:, 2] == L + 4).all(), res[:4]
    got = d_out.cpu().numpy()
    assert (got[:, :L] == pay).all()
    # the same slots through the receive oracle: verdicts and bytes identical (two of them; the scalar oracle is slow)
    iq = d_iq[:2].cpu().numpy().reshape(-1, 2)
    ores, oout = oracle_py.rx11b_batch(iq, np.arange(2, dtype=np.uint64) * slot, np.full(2, slot, np.uint32), out_stride=2048)
    for k in ("status", "rate_kbps", "length", "crc32"):
        assert (ores[k] == res[:2, ["status", "rate_kbps", "length", "crc32"].index(k)]).all(), k
    assert (oout[:, :L] == got[:2, :L]).all()
