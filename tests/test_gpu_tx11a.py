"""GPU parity tests for the 802.11a transmit path (pytest -m gpu): CUDA modulator through the C ABI against oracle/tx11a.cpp,
and the on-device loop-back TX -> RX."""
import numpy as np, pytest, zlib
import oracle_py
from sora_b200 import api, synth

pytestmark = pytest.mark.gpu

@pytest.fixture(scope="module")
def eng():
    return api.Engine(0)

@pytest.mark.parametrize("rate", sorted(synth.RATES))
def test_tx_matches_oracle_bit_exact(eng, rate):
    rng = np.random.default_rng(rate + 1)
    lens = [1, 2, 13, 37, 200, 333, 1496, 2496, 57, 1000]
    pay = [rng.integers(0, 256, L).astype(np.uint8) for L in lens]
    seeds = np.array([0xFF, 0x5B, 0x02, 0x80, 0xFE, 0x13, 0xFF, 0x6D, 0x00, 0x01], np.uint8)      # 0x00 / 0x01: the all-zero scrambler state
    out, ns = eng.tx11a_batch(pay, rate, seeds=seeds, lead=0, sample_bits=8)
    for i, p in enumerate(pay):
        want = oracle_py.tx11a_modulate(p, rate, int(seeds[i]), tail_zeros=0)
        assert ns[i] == len(want), (i, ns[i], len(want))
        bad = np.nonzero((out[i, :len(want)] != want).any(1))[0]
        assert len(bad) == 0, (rate, lens[i], bad[:10], out[i, bad[:4]], want[bad[:4]])
        assert (out[i, len(want):] == 0).all()

def test_tx_formats_and_default_seed(eng):
    p = [np.full(200, 0x31, np.uint8)]
    o8, ns = eng.tx11a_batch(p, 24000, lead=0, sample_bits=8)
    want = oracle_py.tx11a_modulate(p[0], 24000, 0xFF, 0)
    assert (o8[0, :ns[0]] == want).all()
    o16, ns16 = eng.tx11a_batch(p, 24000, lead=100, sample_bits=16)
    assert ns16[0] == ns[0] + 100 and (o16[0, :100] == 0).all()
    assert (o16[0, 100:ns16[0]] == want.astype(np.int16) << 8).all()

def test_loopback_tx_to_rx_on_device(eng):
    """Modulate on the GPU into COMPLEX16 slots and decode them with the receive path without leaving the device."""
    import torch
    rng = np.random.default_rng(9)
    for rate, L in ((54000, 1496), (6000, 100), (36000, 700)):
        F = 64
        pay = rng.integers(0, 256, (F, L)).astype(np.uint8)
        d_pay = torch.from_numpy(pay.reshape(-1)).cuda()
        d_off = torch.arange(F, dtype=torch.int64, device="cuda") * L; d_len = torch.full((F,), L, dtype=torch.int32, device="cuda")
        slot = (api.Engine.tx11a_out_stride(L, rate, lead=400) + 400 + 27) // 28 * 28   # the default slot and 400 samples of silence
        d_iq = torch.zeros((F, slot, 2), dtype=torch.int16, device="cuda"); d_ns = torch.zeros(F, dtype=torch.int32, device="cuda")
        eng.tx11a_raw(d_pay.data_ptr(), F * L, d_off.data_ptr(), d_len.data_ptr(), 0, F, rate, 400, 16, d_iq.data_ptr(), slot, d_ns.data_ptr(), torch.cuda.current_stream().cuda_stream)
        s_off = torch.arange(F, dtype=torch.int64, device="cuda") * slot; s_len = torch.full((F,), slot, dtype=torch.int32, device="cuda")
        d_out = torch.zeros((F, 2560), dtype=torch.uint8, device="cuda"); d_res = torch.zeros((F, 7), dtype=torch.int32, device="cuda")
        eng.rx11a_raw(d_iq.data_ptr(), F * slot, s_off.data_ptr(), s_len.data_ptr(), F, d_out.data_ptr(), 2560, d_res.data_ptr(), torch.cuda.current_stream().cuda_stream)
        torch.cuda.synchronize()
        res = d_res.cpu().numpy()
        assert (res[:, 0] == 1).all() and (res[:, 1] == rate).all() and (res[:, 2] == L + 4).all(), res[:4]
        got = d_out.cpu().numpy()
        assert (got[:, :L] == pay).all()
        for i in (0, F - 1):
            assert int.from_bytes(bytes(got[i, L:L + 4]), "little") == zlib.crc32(pay[i].tobytes())

def test_full_size_roundtrip_baseline_config2(eng):
    """BASELINE config #2 at full size (65 536 frames, 54 Mbps, PSDU 1500 B, 9824-sample slots) as an encode -> decode round trip:
    the device modulator makes the slots, the receive path must return every payload with a matching FCS."""
    import torch
    F, L, rate = 65536, 1496, 54000
    g = torch.Generator(device="cuda"); g.manual_seed(1234)
    d_pay = torch.randint(0, 256, (F, L), dtype=torch.uint8, device="cuda", generator=g)
    d_off = torch.arange(F, dtype=torch.int64, device="cuda") * L; d_len = torch.full((F,), L, dtype=torch.int32, device="cuda")
    slot = 9824
    d_iq = torch.empty((F, slot, 2), dtype=torch.int16, device="cuda"); st = torch.cuda.current_stream().cuda_stream
    eng.tx11a_raw(d_pay.data_ptr(), F * L, d_off.data_ptr(), d_len.data_ptr(), 0, F, rate, 32, 16, d_iq.data_ptr(), slot, 0, st)
    s_off = torch.arange(F, dtype=torch.int64, device="cuda") * slot; s_len = torch.full((F,), slot, dtype=torch.int32, device="cuda")
    d_out = torch.zeros((F, 1500), dtype=torch.uint8, device="cuda"); d_res = torch.zeros((F, 7), dtype=torch.int32, device="cuda")
    eng.rx11a_raw(d_iq.data_ptr(), F * slot, s_off.data_ptr(), s_len.data_ptr(), F, d_out.data_ptr(), 1500, d_res.data_ptr(), st)
    torch.cuda.synchronize()
    assert bool((d_res[:, 0] == 1).all()) and bool((d_res[:, 1] == rate).all()) and bool((d_res[:, 2] == L + 4).all())
    assert bool((d_out[:, :L] == d_pay).all())
    # a checksum of checksums: the FCS words the receiver saw are the CRC-32 of the payloads (spot-checked on the host)
    fcs = d_res[:, 3].cpu().numpy().astype(np.uint32); pay = d_pay[:64].cpu().numpy()
    for i in range(64): assert fcs[i] == zlib.crc32(pay[i].tobytes())
