"""The inputs of test_gpu_zz_viterbi_persistent.py do their job (no GPU: the CPU oracle on the unique captures of scale_inputs.py).

At 65 536 tiled slots every code rate's work list must be longer than one round of k_viterbi_re's persistent CTAs, with a margin: more
than SMS x 16 x 8 decoded frames (16 CTAs per SM is what the kernel's registers would allow without its shared-memory limit, so the
margin holds if a later build fits more CTAs on an SM).  Every code rate has frames the oracle decodes (FRAME_OK) and frames it rejects
on the FCS (CRC32_FAIL), and there are PLCP failures, slots without a frame and slots cut inside the DATA field.  Without these checks a
change of the generators could quietly turn the GPU tests into clean-frame tests."""
import os
import numpy as np, pytest
import oracle_py
import scale_inputs as S

SMS = 132                                               # multiprocessors of an H100 SXM
LOOP_MIN = SMS * 16 * 8                                 # decoded frames per code rate above which a CTA takes several groups
N = 65536
DECODED = (oracle_py.E_FRAME_OK, oracle_py.E_CRC32_FAIL)

@pytest.fixture(scope="module")
def ores11a():
    u = S.uniques_11a()
    r, _ = oracle_py.rx11a_batch(u.iq, u.off, u.length, out_stride=2560, nthreads=os.cpu_count())
    return u, r

@pytest.fixture(scope="module")
def ores11n():
    u = S.uniques_11n()
    oracle_py.set_ht_mcs_limit(15)
    try:
        r, _ = oracle_py.rx11n_batch(u.iq[0], u.iq[1], u.off, u.length, nthreads=os.cpu_count())
    finally:
        oracle_py.set_ht_mcs_limit(11)
    return u, r

def _per_code_rate(u, r, code_rate_of, perm):
    """Decoded frames per code rate over the slots of `perm`, and the statuses per code rate over the uniques."""
    cr = np.array([code_rate_of.get(x, -1) for x in u.rate]); dec = np.isin(r["status"], DECODED)
    counts = {c: int((dec & (cr == c))[perm].sum()) for c in range(3)}
    statuses = {c: set(int(s) for s in r["status"][cr == c]) for c in range(3)}
    return counts, statuses

@pytest.mark.parametrize("seed", (1, 2))
def test_11a_every_code_rate_loops(ores11a, seed):
    u, r = ores11a
    _, _, perm = S.tile(u, N, seed)
    counts, statuses = _per_code_rate(u, r, S.CODE_RATE_11A, perm)
    assert all(v > LOOP_MIN for v in counts.values()), counts
    for c in range(3):
        assert {oracle_py.E_FRAME_OK, oracle_py.E_CRC32_FAIL} <= statuses[c], (c, statuses[c])
    for rate in S.CODE_RATE_11A:                         # every rate decodes somewhere
        assert any(u.rate[i] == rate and r["status"][i] == 1 for i in range(len(u.rate))), rate

def test_11a_damage_present(ores11a):
    u, r = ores11a
    kind = np.array(u.kind); st = r["status"]
    assert (st == oracle_py.E_PLCP_FAIL).sum() >= 20
    assert (st == oracle_py.E_NO_FRAME).sum() >= 40 and ((kind == "noise") | (kind == "zero")).sum() >= 40
    assert (kind == "trunc").sum() >= 30 and not np.isin(st[kind == "trunc"], DECODED).any()     # a truncated code block never reaches a verdict
    assert (kind == "payload").sum() >= 60 and (st[kind == "payload"] == oracle_py.E_CRC32_FAIL).mean() > 0.8
    assert {i % 4 for i in range(len(u.rate)) if u.rate[i]} == {0, 1, 2, 3}
    assert max(u.psdu_len) >= 1400 and min(l for l in u.psdu_len if l) <= 3
    assert u.length.max() <= S.SLOT_CAP

def test_11a_tile_mixes_every_group():
    """tile(): every unique N // U or N // U + 1 times, neighbours unrelated (a group of 8 slots is not a run of one unique), and not
    periodic."""
    u = S.uniques_11a(); U = len(u.off)
    off, ln, perm = S.tile(u, N, 1)
    c = np.bincount(perm, minlength=U); assert c.min() >= N // U and c.max() <= N // U + 1
    assert (off == u.off[perm]).all() and (ln == u.length[perm]).all()
    g = perm[:N // 8 * 8].reshape(-1, 8)
    assert (np.array([len(set(x)) for x in g]) >= 6).mean() > 0.95
    assert not (perm[U:2 * U] == perm[:U]).all()
    assert (S.tile(u, N, 1)[2] == perm).all() and not (S.tile(u, N, 2)[2] == perm).all()

def test_11n_every_code_rate_loops(ores11n):
    u, r = ores11n
    _, _, perm = S.tile(u, N, 3)
    counts, statuses = _per_code_rate(u, r, S.CODE_RATE_11N, perm)
    assert all(v > LOOP_MIN for v in counts.values()), counts
    for c in range(3):
        assert {oracle_py.E_FRAME_OK, oracle_py.E_CRC32_FAIL} <= statuses[c], (c, statuses[c])
    kind = np.array(u.kind); st = r["status"]
    assert (st == oracle_py.E_PLCP_FAIL).sum() >= 5 and (st == oracle_py.E_NO_FRAME).sum() >= 10 and (kind == "trunc").sum() >= 10
    assert max(u.psdu_len) <= 400 and set(u.rate) - {0} == set(S.CODE_RATE_11N)

def test_streams_mostly_rate_34():
    """256 captures of 3 .. 5 frames, at least 85 % of them at rate 3/4; tiled to 20 480 captures, each of the first three frames of a
    capture is a decoded rate-3/4 frame in more than LOOP_MIN captures."""
    u = S.uniques_streams()
    assert len(u.off) == 256 and all(3 <= len(x) <= 5 for x in u.rate)
    flat = [x for rs in u.rate for x in rs]
    assert np.mean([S.CODE_RATE_11A[x] == 2 for x in flat]) >= 0.85 and {S.CODE_RATE_11A[x] for x in flat} == {0, 1, 2}
    _, _, perm = S.tile(u, 20480, 4)
    dec34 = np.zeros((len(u.off), 3), bool)
    for i in range(len(u.off)):
        o = int(u.off[i]); r, _ = oracle_py.rx11a_run(u.iq[o:o + int(u.length[i])], max_frames=16, out_stride=2560)
        for j in range(min(3, len(r))):
            dec34[i, j] = r["status"][j] in DECODED and S.CODE_RATE_11A.get(int(r["rate_kbps"][j]), -1) == 2
    per_pass = dec34[perm].sum(0)
    assert (per_pass > LOOP_MIN).all(), per_pass
