"""The channel inputs of channel_inputs.py: the helpers do what they say, the CPU oracle stays defined on every case, and the cases tell
decoding and failing frames apart.

The oracle is built with a trapping signed-overflow check, as in test_cpu_oracle_rails.py, and every case goes through its receive
entry points in a subprocess (python channel_inputs.py <library>): the device kernels are checked against the oracle bit for bit, which
means nothing where the oracle's C++ is undefined.  The subprocess prints every case's batch status, which the counts below read."""
import collections, os, subprocess, sys
import numpy as np, pytest
import channel_inputs as CI
from test_cpu_oracle_rails import ORACLE, ROOT, _make_var

E_FRAME_OK = 0x1


def _signal(n, seed):
    rng = np.random.default_rng(seed)
    return rng.normal(size=(2, n)) + 1j * rng.normal(size=(2, n))


def test_sco_zero_and_identity_channels_are_exact():
    x = _signal(3000, 1)
    assert np.array_equal(CI.sco(x, 0, 40e6), x) and np.array_equal(CI.sco(x[0], 0, 40e6, CI.FC_11A), x[0])
    assert np.array_equal(CI.resample(x, 1.0), x)
    assert np.array_equal(CI.multipath(x, [0], [1]), x)
    assert np.array_equal(CI.multipath(x, [0], [np.eye(2)]), x)
    for d in (1, 7, 48):
        y = CI.multipath(x, [d], [1])
        assert y.shape == (2, 3000 + d) and np.array_equal(y[:, d:], x) and not y[:, :d].any()
        y = CI.multipath(x, [0, d], [np.eye(2), np.zeros((2, 2))])
        assert np.array_equal(y[:, :3000], x) and not y[:, 3000:].any()


def test_multipath_is_the_stated_sum():
    x = _signal(500, 2)
    G = [np.array([[1, 0.5j], [-0.2, 0.7]]), np.array([[0.1, 0], [0.3j, -0.4]])]
    y = CI.multipath(x, [0, 5], G)
    want = np.zeros((2, 505), complex)
    for a in range(2):
        for b in range(2):
            want[a] += np.convolve(x[b], np.r_[G[0][a, b], np.zeros(4), G[1][a, b]])
    assert np.abs(y - want).max() < 1e-12


@pytest.mark.parametrize("ratio", [1 + 40e-6, 1 - 100e-6, 1.1, 1 / 1.1])
def test_resample_against_analytic_tones(ratio):
    """Twenty complex tones within +-0.3 of the input rate, evaluated at m / ratio: the resampler within -80 dB away from the edges."""
    rng = np.random.default_rng(3)
    f = rng.uniform(-0.3, 0.3, 20) * min(1.0, ratio); a = rng.normal(size=20) + 1j * rng.normal(size=20)
    sig = lambda t: (a[None, :] * np.exp(2j * np.pi * f[None, :] * t[:, None])).sum(1)
    x = sig(np.arange(4000.0)); y = CI.resample(x, ratio)
    t = np.arange(len(y)) / ratio
    assert len(y) == int(np.floor(3999 * ratio + 1e-9)) + 1
    m = (t > 60) & (t < 3940)
    err = np.abs(y[m] - sig(t[m])).max() / np.sqrt((np.abs(x) ** 2).mean())
    assert err < 1e-4, 20 * np.log10(err)


def test_sco_drift_and_matched_carrier():
    """A frame-long drift: an impulse at input sample 20000 lands at 20000 (1 + ppm 1e-6); the matched carrier offset is -ppm fc."""
    x = np.zeros(30000, complex); x[20000] = 1.0
    for ppm in (40, -100):
        y = CI.sco(x, ppm, 40e6)
        assert abs(np.argmax(np.abs(y)) - 20000 * (1 + ppm * 1e-6)) <= 0.5
    tone = CI.sco(np.ones(4000, complex), 25, 40e6, CI.FC_11A)
    ph = np.angle(tone[2001:3000] / tone[2000:2999])
    assert np.allclose(ph, -2 * np.pi * 25e-6 * CI.FC_11A / 40e6, atol=1e-6)


@pytest.mark.parametrize("k", [10, 7, -21, -1])
def test_two_ray_null_sits_on_its_subcarrier(k):
    d, g = CI.two_ray_null(k, 3, 40e6)
    H = lambda kk: sum(gi * np.exp(-2j * np.pi * kk * CI.SUBCARRIER_HZ * di / 40e6) for di, gi in zip(d, g))
    assert abs(H(k)) < 1e-12 and min(abs(H(kk)) for kk in (k - 1, k + 1)) > 0.1
    d, g = CI.two_ray_null(k, 3, 40e6, depth_db=40)
    assert abs(20 * np.log10(abs(H(k)) / abs(g[0])) + 40) < 1e-9


def test_profiles():
    for rms in (50, 150):
        d, g = CI.exp_profile(rms, 40e6, 1)
        assert max(d) < 32 and abs(sum(abs(x) ** 2 for x in g) - 1) < 1e-12          # inside the 0.8 us guard interval at 40 Msps
    d, G = CI.mimo_near_singular(3, 9)
    H = lambda kk: sum(gi * np.exp(-2j * np.pi * kk * CI.SUBCARRIER_HZ * di / 40e6) for di, gi in zip(d, G))
    det = lambda kk: abs(np.linalg.det(H(kk)))
    assert 0 < det(9) < 0.1 and np.median([det(kk) for kk in range(-28, 29) if kk]) > 5 * det(9)


def test_cases_are_whole_blocks_and_deterministic():
    for rate in CI.RATES_11A:
        for (n, x), (n44, x44) in zip(CI.cases_11a(rate), CI.cases_11a(rate, 44)):
            assert n == n44 and x.dtype == np.int16 and len(x) % 28 == 0 and len(x44) % 28 == 0
            assert abs(len(x44) / len(x) - 1.1) < 0.02
    for mcs, _ in CI.MCS_11N:
        for n, (a, b) in CI.cases_11n(mcs):
            assert a.shape == b.shape and len(a) % 28 == 0
    for rate in CI.RATES_11B:
        for n, x in CI.cases_11b(rate):
            assert len(x) % 28 == 0
    first = CI.cases_11b(11000)
    CI.cases_11b.cache_clear()                                     # rendered again from the same seeds: the same captures
    assert all(n == m and np.array_equal(x, y) for (n, x), (m, y) in zip(first, CI.cases_11b(11000)))


@pytest.mark.parametrize("rate", CI.RATES_11A)
def test_notch_reaches_the_int16_truncation_of_the_channel_inverse(rate):
    """802.11a H^-1 = (+-1600 conj(Y)) / (|Y|^2 >> 8), truncated to int16.  On bin -15 of notch21dB_trunc16 the divisor is 1, so both
    components are multiples of 1600 modulo 2^16, and one of them is 1600 * 21 or more: it wrapped."""
    import oracle_py
    x = dict(CI.cases_11a(rate))["notch21dB_trunc16"]
    t = oracle_py.rx11a_taps(x, max_sym=120)
    assert t["res"]["status"] == E_FRAME_OK
    mult = lambda v: [k for k in range(-23, 24) if (int(v) - 1600 * k) % 65536 == 0]
    re, im = t["chan_coeffs"][64 - 15]
    assert mult(re) and mult(im) and max(abs(k) for k in mult(re) + mult(im)) >= 21, (re, im)


@pytest.fixture(scope="module")
def oracle_run(tmp_path_factory):
    so = str(tmp_path_factory.mktemp("trapv") / "libsora_oracle_trapv.so")
    cxx = os.environ.get("CXX", "g++")
    flags = [f for f in _make_var("CXXFLAGS") if not f.startswith("-W")] + ["-w", "-fsanitize=signed-integer-overflow", "-fsanitize-trap=all"]
    subprocess.run([cxx] + flags + ["-shared", "-o", so] + _make_var("SRC"), cwd=ORACLE, check=True, capture_output=True, timeout=600)
    p = subprocess.run([sys.executable, os.path.join(ROOT, "tests", "channel_inputs.py"), so], capture_output=True, text=True, timeout=600)
    return p


def test_oracle_has_no_signed_overflow_on_channel_cases(oracle_run):
    lines = oracle_run.stdout.splitlines()
    assert oracle_run.returncode == 0 and lines[-1:] == ["done"], \
        f"oracle stopped (exit {oracle_run.returncode}) after {lines[-1] if lines else '?'!r}; stderr: {oracle_run.stderr[-400:]}"


# per chain: cases, at least this many FRAME_OK, and at least one that does not decode
MIN_OK = {"11a": (68, 44), "11b": (32, 10), "11n": (24, 16)}

@pytest.mark.parametrize("chain", sorted(MIN_OK))
def test_cases_decode_and_fail(oracle_run, chain):
    st = collections.Counter(); name = None
    for line in oracle_run.stdout.splitlines():
        if line.startswith(("11a ", "11b ", "11n ")): name = line
        elif line.startswith("status ") and name.startswith(chain): st[int(line.split()[1], 16) == E_FRAME_OK] += 1
    n, k = MIN_OK[chain]
    assert st[True] + st[False] == n and st[True] >= k and st[False] >= 1, dict(st)
