"""PLCP header cases (tests/plcp_inputs.py) through the CPU oracle: on clean captures its report of every header equals the plain
restatement of the reference's parsers, in one-slot-per-frame mode and, for what a context carries between events, in continuous
captures.  This pins both the header generators in sora_b200/synth.py and the table the device is held to in test_gpu_plcp_headers.py."""
import numpy as np, pytest
import oracle_py
import plcp_inputs as P
from sora_b200 import synth


def _check_batch(std, cases, res):
    bad = []
    for c, r in zip(cases, res):
        want = {"status": P.expected_status(c), **c["expect"]}
        if want["status"] == P.E_NONE:                  # no event: the batch slot reads all zero
            want = {k: (v if k == "status" else 0) for k, v in want.items()}
        got = {k: int(r[k]) for k in want}
        if got != want:
            bad.append((c["name"], got, want))
    assert not bad, f"{std}: {len(bad)} of {len(cases)} cases differ: {bad}"

def test_oracle_headers_11a():
    cases = P.cases_11a()
    res, out = oracle_py.rx11a_batch(*P.slots_of(cases), out_stride=2560)
    _check_batch("11a", cases, res)
    for c, r, o in zip(cases, res, out):
        if r["status"] == P.E_OK:
            assert (o[:len(c["body"])] == c["body"]).all(), c["name"]

def test_oracle_headers_11b():
    cases = P.cases_11b()
    res, out = oracle_py.rx11b_batch(*P.slots_of(cases), out_stride=4096)
    _check_batch("11b", cases, res)
    for c, r, o in zip(cases, res, out):
        if r["status"] == P.E_OK:
            n = len(c["body"]) - 1                      # the sink stops one byte short of the FCS end (PHY_11b.hpp:728-739)
            assert (o[:n] == c["body"][:n]).all(), c["name"]

@pytest.mark.parametrize("mcs_limit", [11, 15])
def test_oracle_headers_11n(mcs_limit):
    cases = P.cases_11n(mcs_limit)
    iq0, off, ln = P.slots_of(cases, "iq0"); iq1, _, _ = P.slots_of(cases, "iq1")
    oracle_py.set_ht_mcs_limit(mcs_limit)
    try: res, out = oracle_py.rx11n_batch(iq0, iq1, off, ln, out_stride=1536)
    finally: oracle_py.set_ht_mcs_limit(11)
    _check_batch("11n", cases, res)
    for c, r, o in zip(cases, res, out):
        if r["status"] == P.E_OK:
            assert (o[:len(c["body"])] == c["body"]).all(), c["name"]

def test_case_matrix_reaches_every_verdict():
    """Every standard's matrix has refused and accepted headers, and every verdict the issue names is reached somewhere."""
    seen = {v for f in (P.cases_11a, P.cases_11b, P.cases_11n) for v in (c["verdict"] for c in f())}
    assert seen == {"plcp", "ok", "crc", "none", "failed"}, seen

def _events(res, keep=(P.E_OK, P.E_CRC32, P.E_PLCP)):
    """The events a header decides: decoded, CRC failure, refused (continuous 802.11b captures also report sync failures on silence)."""
    return [r for r in res if int(r["status"]) in keep]

def test_oracle_stream_11a_resets_rx_vector():
    iq, want = P.stream_11a()
    res, _ = oracle_py.rx11a_run(iq, max_frames=16)
    assert len(res) == len(want) and [{k: int(r[k]) for k in w} for r, w in zip(res, want)] == want

def test_oracle_stream_11b_carries_rx_vector():
    iq, want = P.stream_11b()
    res, _ = oracle_py.rx11b_run(iq, max_frames=32)
    assert [{k: int(r[k]) for k in w} for r, w in zip(_events(res), want)] == want and len(_events(res)) == len(want)

@pytest.mark.parametrize("mcs_limit", [11, 15])
def test_oracle_stream_11n_carries_mcs_not_lsig_length(mcs_limit):
    """Decoded MCS 9, L-SIG refused, CRC-8 failure, L-SIG refused, MCS refused, L-SIG refused, decoded: the L-SIG refusals report the
    MCS of the event before (9, 0, then the refused one) and an L-SIG length of 0 or their own."""
    iq0, iq1, want = P.stream_11n(mcs_limit)
    oracle_py.set_ht_mcs_limit(mcs_limit)
    try: res, _ = oracle_py.rx11n_run(iq0, iq1, max_frames=16)
    finally: oracle_py.set_ht_mcs_limit(11)
    assert len(res) == len(want) and [{k: int(r[k]) for k in w} for r, w in zip(res, want)] == want
    assert [w["mcs"] for w in want] == [9, 9, 0, 0, 11 if mcs_limit == 11 else 15, 11 if mcs_limit == 11 else 15, 8]
    assert want[1]["lsig_length"] == 0 and want[5]["lsig_length"] == 1502

def test_generators_default_headers():
    """With no override the generators send the headers their bodies call for: the restatement accepts each at its own rate and length."""
    for rate in synth.RATES:
        assert P.parse_11a(synth.signal_word_11a(rate, 1234)) == (True, rate, 1234, -(-(1234 * 8 + 22) // P.NDBPS11A[rate]) + 1)
    for rate in (1000, 2000, 5500, 11000):
        for L in range(100, 111):
            assert P.parse_11b(*synth.plcp_11b(L, rate), True) == (True, rate, L)
