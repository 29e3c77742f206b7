"""Packet error rate against SNR of the eight 802.11a rates, device-resident end to end: sb200_tx11a_batch -> sb200_channel_sim ->
sb200_rx11a_batch, all on one GPU.

    python tools/per_sweep.py [--links 4096] [--bytes 500] [--snr -2:30:2]

For every rate one frame is modulated on the device and widened to COMPLEX16 (x 200, the scale the receiver's carrier sense needs), then
every link of the call reads that one row (in_link_stride 0) through its own channel:
  awgn      one unit tap;
  exp150ns  an independent exponential power-delay profile per link (rms spread 150 ns, 32 taps at 40 Msps, one Rayleigh draw per tap:
            channel_inputs.exp_profile with the link's seed, unit power), each scaled down only as far as its tap sums need (to 65000 / 16384:
            a power gain of 0.5-0.6; a fixed 1/2 would leave many frames below the receiver's carrier-sense threshold).
The noise is set from the transmit power measured on the device: sigma^2 = P_tx g / 10^(snr / 10) / 2 per component, g the link's power
gain, and every link draws different noise (the link index is in the noise counter).  A packet
counts as received when its status is FRAME_OK and its bytes equal the PSDU.  One JSON line per (channel, rate, SNR), with the card and
its power limit."""
import argparse, json, os, subprocess, sys
import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT); sys.path.insert(0, os.path.join(ROOT, "tests"))

RATES = (6000, 9000, 12000, 18000, 24000, 36000, 48000, 54000)

def card():
    try:
        s = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=name,power.limit", "--format=csv,noheader,nounits"], capture_output=True, text=True, timeout=30).stdout
        name, pl = [v.strip() for v in s.strip().splitlines()[0].split(",")]
        return name, float(pl)
    except Exception:
        return None, None

def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--links", type=int, default=4096)
    ap.add_argument("--bytes", type=int, default=500, help="PSDU bytes (MPDU + 4 FCS)")
    ap.add_argument("--snr", default="-2:30:2", help="first:last:step in dB")
    ap.add_argument("--channels", default="awgn,exp150ns")
    a = ap.parse_args()
    import torch
    from sora_b200 import api, synth
    import channel_inputs as CI
    dev = torch.device("cuda", 0); eng = api.Engine(0); name, plim = card()
    lo, hi, st = (float(v) for v in a.snr.split(":")); snrs = np.arange(lo, hi + st / 2, st)
    nl, L = a.links, 32
    mpdu = np.random.RandomState(0x9E5).randint(0, 256, a.bytes - 4).astype(np.uint8); psdu = synth.psdu_with_fcs(mpdu)
    taps_of = {"awgn": (np.broadcast_to(api.sim_taps([0], [1.0], L), (nl, 1, 1, L, 2)), np.ones(nl))}
    tl, gl = [], []
    for l in range(nl):
        d, g = CI.exp_profile(150, CI.FS_11A, 1000 + l)
        h = np.zeros(L, np.complex128); np.add.at(h, d, g)
        s = min(1.0, 65000 / ((np.abs(h.real) + np.abs(h.imag)).sum() * 16384))
        tl.append(api.sim_taps(d, [s * v for v in g], L)); gl.append(s * s)
    taps_of["exp150ns"] = (np.stack(tl), np.array(gl))
    for ch in a.channels.split(","):
        taps, gain = taps_of[ch]; dt = torch.from_numpy(np.ascontiguousarray(taps)).to(dev)
        for rate in RATES:
            td, ns = eng.tx11a_batch([mpdu], rate)                       # host copy of the frame only to size the rows
            n = int(ns[0]); si = (400 + n + 400 + 3) // 4 * 4
            flat, offs, lens = api._payload_table([mpdu]); dout = torch.zeros((1, td.shape[1], 2), dtype=torch.int8, device=dev); nsd = np.zeros(1, np.uint32)
            eng.tx11a_raw(api._ptr(flat), flat.size, api._ptr(offs), api._ptr(lens), 0, 1, rate, 0, 8, dout.data_ptr(), td.shape[1], api._ptr(nsd))
            x = torch.zeros((1, 1, si, 2), dtype=torch.int16, device=dev); x[0, 0, 400:400 + n] = dout[0, :n].to(torch.int16) * 200
            p_tx = float((x[0, 0, 400:400 + n].to(torch.float64) ** 2).sum(-1).mean())
            y = torch.zeros((nl, 1, si, 2), dtype=torch.int16, device=dev)
            off = np.arange(nl, dtype=np.uint64) * si; ln = np.full(nl, si, np.uint32)
            res = np.zeros(nl, api.RESULT_DTYPE); out = np.zeros((nl, a.bytes + 64), np.uint8)
            for snr in snrs:
                q8 = np.rint(256 * np.sqrt(p_tx * gain / 10 ** (snr / 10) / 2)).astype(np.uint32)
                links = np.zeros(nl, api.LINK_DTYPE); links["step"] = 2 ** 32; links["noise_q8"] = q8
                eng.channel_sim_raw(x.data_ptr(), 0, si, 1, si, links, dt.data_ptr(), L, nl, 0x5EED + int(snr * 10), y.data_ptr(), si, si, 1, si)
                eng.rx11a_raw(y.data_ptr(), nl * si, api._ptr(off), api._ptr(ln), nl, api._ptr(out), out.shape[1], api._ptr(res))
                ok = (res["status"] == api.FRAME_OK) & (out[:, :len(psdu)] == psdu).all(1)
                print(json.dumps({"channel": ch, "rate_kbps": rate, "snr_db": float(snr), "links": nl, "psdu_bytes": a.bytes, "per": 1.0 - float(ok.mean()),
                                  "noise_q8_mean": float(q8.mean()), "tx_power_lsb2": p_tx, "card": name, "power_limit_w": plim}), flush=True)
    eng.close()

if __name__ == "__main__":
    main()
