#!/usr/bin/env python3
"""bench_extra.py — the BASELINE.json configurations that are not the headline line of bench.py:

  --config viterbi   config #5: standalone K=7 soft Viterbi, rates 1/2, 2/3, 3/4, independent blocks of 20 022 information
                     bits (max 11a frame, 2500 B), device-resident soft values; coded bits/s and decoded Mbit/s
  --config 11b       config #3: 802.11b 11 Mbps CCK RX chain, PSDU 1500 B, 44 Msps, one frame per slot
  --config tx11a     SURVEY.md §8(f) rank 2: the 802.11a modulator on the device, 54 Mbps / 1500 B frames into config #2's slots
  --config tx11b     SURVEY.md §8(f) rank 2: the 802.11b modulator on the device, 11 Mbps CCK / 1500 B frames at 44 Msps
  --config tx11n     the 802.11n two-stream modulator on the device, MCS 8 / 9 / 10, 1500 B frames: the input of config #4 made on the device
  --config fir37     the legacy 802.11b transmit filter (BB11BPMDSpreadFIR4SSE) on the device
  --config tx11b_legacy  the legacy 802.11b transmitter (BB11BPMDPacketGenSignal: encoder + SSE filter, fused) on the device, 11 Mbps / 1500 B
  --config tx11a_legacy  the legacy 802.11a transmitter (BB11ATxFrameMod) on the device, 54 Mbps / 1500 B, at 40 and at 44 Msps
  --config channelize  the wideband channelizer: four 802.11a channels of a 160 Msps capture, 127 taps, D = 4, device-resident
  --config channelize_bank  the filter-bank channelizer: all eight odd-stacked 20 MHz channels of a 160 Msps capture, 255 taps, D = 4,
                      timed beside sb200_channelize on the same eight channels and taps
  --config channelize_rational  the rational-rate channelizer: three 802.11b channels of a 160 Msps capture to 44 Msps, 1287 taps, U / D = 11 / 40
  --config channelize_arbitrary  the arbitrary-rate channelizer: --config channelize_rational's capture to 44 Msps through a 64-tap table,
                      timed beside sb200_channelize_rational; and a 122.88 Msps capture of the 2.4 GHz band to 44 and 40 Msps
  --config combine   the wideband combiner: four 802.11a channel rows at 40 Msps into one 160 Msps capture, 127 taps, U = 4, device-resident
  --config combine_bank  the filter-bank combiner: eight odd-stacked 40 Msps rows into one 160 Msps capture, 255 taps, U = 4,
                      timed beside sb200_combine on the same eight channels and taps
  --config combine_rational  the rational-rate combiner: three 802.11b rows at 44 Msps into one 160 Msps capture, 1761 taps, U / D = 40 / 11
  --config combine_arbitrary  the arbitrary-rate combiner: --config combine_rational's rows into 160 Msps through a 64-tap table, timed
                      beside sb200_combine_rational; and the 2.4 GHz band into a 122.88 Msps capture from 44 and 40 Msps
  --config spectrum  the spectrum meter: --config channelize's 160 Msps capture, FFT<1024> every 1024 samples, Hann, 64 frames per group,
                     device-resident; also the power meter on the same capture (blocks of 4096)
  --config sim       the radio channel simulator: --frames links of config #2's 9 824-sample slots (T = R = 1, L = 16, +20 ppm, a carrier
                     offset, noise on), and a 2x2 case (T = R = 2, L = 16), device-resident
  --config 11n       config #4: 802.11n HT-MF 2x2 RX chain at MCS 8, 9, 10, PSDU 1500 B, 2 x 40 Msps, fixed 2x2 channel

Each prints one JSON line per measurement (same timing rules as bench.py: >= 3 warm-ups, CUDA events on the launch
stream, inputs larger than L2).  Results are checked against the CPU oracle on a sample before timing.
"""
import argparse, json, os, sys, time
import numpy as np

ROOT = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, ROOT); sys.path.insert(0, os.path.join(ROOT, "tests"))

def peaks():
    try: return float(json.load(open(os.path.join(ROOT, "MEASURED_PEAKS.json")))["hbm_gbs"])
    except Exception: return 6650.0

class Ctx:
    """One process per GPU (torchrun) or a single process: device, engine, and a timing helper that follows bench.py's rules
    (>= 3 warm-ups, barrier + synchronize on both sides, CUDA events on the launch stream, max over ranks)."""
    def __init__(self):
        import torch
        from sora_b200 import api
        from bench import numa_bind, effective_cpus
        self.torch = torch
        self.world = int(os.environ.get("WORLD_SIZE", "1")); self.rank = int(os.environ.get("RANK", "0")); self.local = int(os.environ.get("LOCAL_RANK", "0"))
        torch.cuda.set_device(self.local)
        self.aff0 = os.sched_getaffinity(0); self.numa = numa_bind(self.local)
        self.dist = None
        if self.world > 1:
            import torch.distributed as dist
            dist.init_process_group("nccl", device_id=torch.device("cuda", self.local)); self.dist = dist
        self.dev = torch.device("cuda", self.local); self.st = torch.cuda.current_stream()
        self.eng = api.Engine(self.local); self.eng.set_option("slot_table_immutable", 1)
        self.e0 = torch.cuda.Event(enable_timing=True); self.e1 = torch.cuda.Event(enable_timing=True)
    def cpus(self):
        from bench import effective_cpus
        os.sched_setaffinity(0, self.aff0)
        return effective_cpus()[0]
    def timed(self, fn, n, warm=3):
        torch = self.torch
        for _ in range(warm): fn()
        torch.cuda.synchronize()
        if self.dist: self.dist.barrier()
        self.e0.record(self.st)
        for _ in range(n): fn()
        self.e1.record(self.st); torch.cuda.synchronize()
        if self.dist: self.dist.barrier()
        t = torch.tensor([self.e0.elapsed_time(self.e1)], dtype=torch.float64, device=self.dev)
        if self.dist: self.dist.all_reduce(t, op=self.dist.ReduceOp.MAX)
        return float(t.item()) / n
    def emit(self, line):
        if self.rank == 0: print(json.dumps(line), flush=True)
    def close(self):
        if self.dist: self.dist.destroy_process_group()

def bench_viterbi(args):
    import oracle_py
    from sora_b200 import api, synth
    c = Ctx(); torch = c.torch; eng, dev, st = c.eng, c.dev, c.st
    L = 2500
    for cr, rate, name in ((api.CR_12, (1, 2), "1/2"), (api.CR_23, (2, 3), "2/3"), (api.CR_34, (3, 4), "3/4")):
        nbits = 8 * L + 16 + 6; nbits += (-nbits) % 48
        U = 64
        rng = np.random.default_rng(cr)
        bits = rng.integers(0, 2, (U, nbits)).astype(np.uint8); bits[:, 8 * L + 16:] = 0
        A, B = synth.conv_encode(bits); coded = synth.puncture(A, B, rate)
        soft = np.where(coded > 0, rng.integers(5, 8, coded.shape), rng.integers(0, 3, coded.shape)).astype(np.uint8)
        flip = rng.random(coded.shape) < 0.03
        soft = np.where(flip, rng.integers(0, 8, coded.shape), soft).astype(np.uint8)
        nsoft = soft.shape[1]; stride = (nsoft + 15) // 16 * 16
        # BASELINE config #5: 1e9 coded bits in total ("strong": the same total at every GPU count), or --blocks per GPU ("weak")
        total = args.blocks * c.world if args.blocks else -(-10**9 // nsoft)
        NB = -(-total // c.world)
        sp = np.zeros((U, stride), np.uint8); sp[:, :nsoft] = soft
        d_soft = torch.from_numpy(sp).to(dev).repeat((NB + U - 1) // U, 1)[:NB].contiguous()
        d_out = torch.zeros((NB, L + 2 + 14), dtype=torch.uint8, device=dev)
        def step(): eng.viterbi_raw(d_soft.data_ptr(), stride, nsoft, NB, cr, L, d_out.data_ptr(), d_out.shape[1], stream=st.cuda_stream)
        step(); torch.cuda.synchronize()
        ref = oracle_py.viterbi_blocks(soft, cr, L)
        got = d_out[:U, :L + 2].cpu().numpy()
        assert (got == ref).all(), "GPU Viterbi differs from the oracle"
        ms = c.timed(step, args.steps)
        coded_bits = NB * c.world * nsoft
        line = {"metric": "standalone K=7 soft Viterbi throughput", "code_rate": name, "value": coded_bits / (ms * 1e-3) / 1e9, "unit": "G coded bits/s",
                "decoded_mbit_s": NB * c.world * (8 * L + 16) / (ms * 1e-3) / 1e6, "ms_per_step": ms, "blocks_per_gpu": NB, "info_bits_per_block": 8 * L + 22,
                "coded_bits_per_step": coded_bits, "n_gpus": c.world, "scaling": "weak" if args.blocks else "strong (1e9 coded bits in total, BASELINE config #5)", "dtype": "uint8 path metrics",
                "parity": "bit-exact vs oracle on %d blocks" % U}
        alg = coded_bits / c.world * (1.0 + (rate[0] / rate[1]) / 8.0)
        line["roofline"] = {"bound": "hbm", "achieved": alg / (ms * 1e-3) / 1e9, "peak": peaks(), "unit": "GB/s", "frac": alg / (ms * 1e-3) / 1e9 / peaks(), "note": "per GPU"}
        if c.rank == 0 and c.world == 1:
            ncpu = c.cpus(); rep = np.tile(soft, (max(1, 4096 // U), 1))
            t0 = time.perf_counter(); oracle_py.viterbi_blocks(rep, cr, L, nthreads=ncpu); dt = time.perf_counter() - t0
            line["cpu_baseline"] = {"value": rep.shape[0] * nsoft / dt / 1e9, "unit": "G coded bits/s", "cores": ncpu, "kind": "port", "sample": f"{rep.shape[0]} blocks"}
        c.emit(line)
        del d_soft, d_out
    c.close()

def bench_11b(args):
    import oracle_py
    from sora_b200 import api, synth
    c = Ctx(); torch = c.torch; eng, dev, st = c.eng, c.dev, c.st
    # The reference's CCK decoder is a pruned search (cck.hpp:262-769) and drops isolated symbols on some band-limited
    # waveforms even without noise; the timed set is made of slots the CPU oracle decodes FRAME_OK, so that the whole
    # chain (all 1500 bytes + CRC) is exercised.  GPU == oracle is asserted on all of them either way.
    iq, ps = synth.make_frames_11b(32, psdu_len=1500, rate_kbps=11000, snr_db=40, gain=0.15, lead=392, trail=200)
    F0, slot, _ = iq.shape
    ores0, _ = oracle_py.rx11b_batch(iq.reshape(-1, 2), np.arange(F0) * slot, np.full(F0, slot), out_stride=1504)
    keep = np.nonzero(ores0["status"] == 1)[0][:16]
    iq, ps = iq[keep], ps[keep]; U = len(keep)
    assert U >= 4, "too few decodable 11b slots"
    F0, slot, _ = iq.shape
    F = args.frames
    flat = iq.reshape(F0, -1)
    d_iq = torch.from_numpy(flat).to(dev).repeat((F + U - 1) // U, 1)[:F].contiguous()
    d_off = torch.arange(F, dtype=torch.int64, device=dev) * slot
    d_len = torch.full((F,), slot, dtype=torch.int32, device=dev)
    d_out = torch.zeros((F, 1504), dtype=torch.uint8, device=dev); d_res = torch.zeros((F, 6), dtype=torch.int32, device=dev)
    def step(): eng.rx11b_raw(d_iq.data_ptr(), F * slot, d_off.data_ptr(), d_len.data_ptr(), F, d_out.data_ptr(), 1504, d_res.data_ptr(), st.cuda_stream)
    step(); torch.cuda.synchronize()
    ores, oout = oracle_py.rx11b_batch(iq.reshape(-1, 2), np.arange(U) * slot, np.full(U, slot), out_stride=1504)
    assert (d_res[:U, 0].cpu().numpy().astype(np.uint32) == ores["status"]).all() and (ores["status"] == 1).all()
    assert (d_out[:U, :1499].cpu().numpy() == oout[:, :1499]).all() and (oout[:, :1499] == ps[:, :1499]).all()
    assert (d_res[:, 0].cpu().numpy() == 1).all()
    ms = c.timed(step, args.steps)
    alg = F * (slot * 4.0 + 1516)
    line = {"metric": "802.11b 11 Mbps CCK RX PHY Msamples/s (IQ in, bits out)", "value": c.world * F * slot / (ms * 1e-3) / 1e6, "unit": "Msamples/s", "ms_per_step": ms,
            "n_gpus": c.world, "scaling": "weak", "config": {"workload": "802.11b 11 Mbps CCK long preamble, PSDU 1500 B, 44 Msps (BASELINE config #3)", "slots_per_step_per_gpu": F, "samples_per_slot": int(slot), "unique_slots": U},
            "roofline": {"bound": "hbm", "achieved": alg / (ms * 1e-3) / 1e9, "peak": peaks(), "unit": "GB/s", "frac": alg / (ms * 1e-3) / 1e9 / peaks(), "note": "per GPU"},
            "parity": "bytes and verdicts identical to the oracle on the %d unique slots" % U}
    if c.rank == 0 and c.world == 1:
        ncpu = c.cpus(); n = 2048
        t0 = time.perf_counter(); oracle_py.rx11b_batch(iq.reshape(-1, 2), (np.arange(n) % U) * slot, np.full(n, slot), out_stride=1504, nthreads=ncpu); dt = time.perf_counter() - t0
        line["cpu_baseline"] = {"value": n * slot / dt / 1e6, "unit": "Msamples/s", "cores": ncpu, "kind": "port", "sample": f"{n} slots"}
    c.emit(line); c.close()

def bench_11n(args):
    import oracle_py
    from sora_b200 import api, synth
    c = Ctx(); torch = c.torch; eng, dev, st = c.eng, c.dev, c.st; dist = c.dist
    mcs_list = [int(m) for m in args.mcs.split(",")]
    if max(mcs_list) > 10: eng.set_option("ht_mcs_limit", 15); oracle_py.set_ht_mcs_limit(15)      # the 16-/64-QAM branches (default: refuse like PHY_11n.hpp:496-501)
    for mcs in mcs_list:
        U = 32
        iq0, iq1, ps = synth.make_frames_11n(U, psdu_len=1500, mcs=mcs, snr_db=30 if mcs <= 10 else 36, lead=400, trail=200)      # fixed 2x2 channel [[1, 0.3j], [-0.2, 0.9]]
        F0, slot, _ = iq0.shape
        F = args.frames
        d0 = torch.from_numpy(iq0.reshape(U, -1)).to(dev).repeat((F + U - 1) // U, 1)[:F].contiguous()
        d1 = torch.from_numpy(iq1.reshape(U, -1)).to(dev).repeat((F + U - 1) // U, 1)[:F].contiguous()
        d_off = torch.arange(F, dtype=torch.int64, device=dev) * slot; d_len = torch.full((F,), slot, dtype=torch.int32, device=dev)
        d_out = torch.zeros((F, 1536), dtype=torch.uint8, device=dev); d_res = torch.zeros((F, 7), dtype=torch.int32, device=dev)
        def step(): eng.rx11n_raw(d0.data_ptr(), d1.data_ptr(), F * slot, d_off.data_ptr(), d_len.data_ptr(), F, d_out.data_ptr(), 1536, d_res.data_ptr(), st.cuda_stream)
        step(); torch.cuda.synchronize()
        ores, oout = oracle_py.rx11n_batch(iq0.reshape(-1, 2), iq1.reshape(-1, 2), np.arange(U) * slot, np.full(U, slot), out_stride=1536)
        assert (ores["status"] == 1).all() and (oout[:, :1500] == ps).all()
        assert (d_res[:, 0].cpu().numpy() == 1).all() and (d_out[:U, :1500].cpu().numpy() == oout[:, :1500]).all()
        ms = c.timed(step, args.steps)
        kt = eng.last_kernel_times()
        alg = F * (slot * 8.0 + 1516)
        line = {"metric": "802.11n 2x2 RX PHY Msample-pairs/s (2 x IQ in, bits out)", "mcs": mcs, "value": c.world * F * slot / (ms * 1e-3) / 1e6, "unit": "Msample-pairs/s", "ms_per_step": ms,
                "n_gpus": c.world, "scaling": "weak", "config": {"workload": "802.11n HT-MF 2x2, 20 MHz, PSDU 1500 B, 40 Msps per antenna, AWGN 30 dB, channel [[1,0.3j],[-0.2,0.9]] (BASELINE config #4)",
                                                   "slots_per_step_per_gpu": F, "sample_pairs_per_slot": int(slot), "unique_slots": U, "numa": c.numa},
                "kernel_ms": dict(zip(("carrier_sense", "ofdm_front_end", "viterbi_descramble_crc", "pack"), kt)) if kt is not None else None,
                "roofline": {"bound": "hbm", "achieved": alg / (ms * 1e-3) / 1e9, "peak": peaks(), "unit": "GB/s", "frac": alg / (ms * 1e-3) / 1e9 / peaks(), "note": "per GPU"},
                "parity": "bytes and verdicts identical to the oracle on the %d unique slots" % U}
        if dist:
            # "frames sharded across 2/4/8 H100" (BASELINE config #4): both antenna captures of all world*F slots sit on rank 0; NCCL scatters the two
            # slabs per rank, every rank decodes its share, NCCL gathers bytes + verdicts on rank 0; everything inside the timed region
            P = 4; Fp = F // P; assert Fp * P == F
            s0 = torch.empty_like(d0); s1 = torch.empty_like(d1); v0 = s0.view(torch.int32); v1 = s1.view(torch.int32)   # NCCL has no 16-bit integer type
            r0 = d0[:U].repeat((c.world * F + U - 1) // U, 1)[: c.world * F].contiguous().view(torch.int32).view(c.world, P, Fp, -1) if c.rank == 0 else None
            r1 = d1[:U].repeat((c.world * F + U - 1) // U, 1)[: c.world * F].contiguous().view(torch.int32).view(c.world, P, Fp, -1) if c.rank == 0 else None
            oa = torch.empty((c.world, F, 1536), dtype=torch.uint8, device=dev) if c.rank == 0 else None
            ra = torch.empty((c.world, F, 7), dtype=torch.int32, device=dev) if c.rank == 0 else None
            offp = torch.arange(Fp, dtype=torch.int64, device=dev) * slot; lenp = torch.full((Fp,), slot, dtype=torch.int32, device=dev)
            def step_m():
                w = []
                for p in range(P):
                    w.append((dist.scatter(v0[p * Fp:(p + 1) * Fp], [r0[r, p] for r in range(c.world)] if c.rank == 0 else None, src=0, async_op=True),
                              dist.scatter(v1[p * Fp:(p + 1) * Fp], [r1[r, p] for r in range(c.world)] if c.rank == 0 else None, src=0, async_op=True)))
                for p in range(P):
                    w[p][0].wait(); w[p][1].wait()
                    eng.rx11n_raw(s0[p * Fp:(p + 1) * Fp].data_ptr(), s1[p * Fp:(p + 1) * Fp].data_ptr(), Fp * slot, offp.data_ptr(), lenp.data_ptr(), Fp,
                                  d_out[p * Fp:(p + 1) * Fp].data_ptr(), 1536, d_res[p * Fp:(p + 1) * Fp].data_ptr(), st.cuda_stream)
                dist.gather(d_out, [oa[r] for r in range(c.world)] if c.rank == 0 else None, dst=0)
                dist.gather(d_res, [ra[r] for r in range(c.world)] if c.rank == 0 else None, dst=0)
            msm = c.timed(step_m, max(3, min(args.steps, 5)), warm=2)
            if c.rank == 0:
                assert bool((ra[:, :, 0] == 1).all()) and (oa[c.world - 1, :U, :1500].cpu().numpy() == oout[:, :1500]).all()
                line["mgpu"] = {"value": c.world * F * slot / (msm * 1e-3) / 1e6, "unit": "Msample-pairs/s", "ms_per_step": msm, "nccl_ranks": c.world,
                                "collective": "NCCL scatter of both antenna slabs (root -> ranks) + gather of bytes and verdicts",
                                "scatter_bytes_per_step": int((c.world - 1) * F * slot * 8), "gather_bytes_per_step": int((c.world - 1) * F * (1536 + 28))}
            del s0, s1, v0, v1, r0, r1, oa, ra
        if c.rank == 0 and c.world == 1:
            ncpu = c.cpus(); n = 1024
            t0 = time.perf_counter(); oracle_py.rx11n_batch(iq0.reshape(-1, 2), iq1.reshape(-1, 2), (np.arange(n) % U) * slot, np.full(n, slot), out_stride=1536, nthreads=ncpu); dt = time.perf_counter() - t0
            line["cpu_baseline"] = {"value": n * slot / dt / 1e6, "unit": "Msample-pairs/s", "cores": ncpu, "kind": "port", "sample": f"{n} slots"}
        c.emit(line)
        del d0, d1, d_out, d_res
    c.close()

def bench_tx11a(args):
    import torch, oracle_py
    from sora_b200 import api
    eng = api.Engine(0); dev = torch.device("cuda", 0); st = torch.cuda.current_stream()
    F, L, rate = args.frames, 1496, 54000                    # PSDU 1500 B incl. FCS, as BASELINE config #2's frames
    rng = np.random.default_rng(7)
    pay = rng.integers(0, 256, (256, L)).astype(np.uint8)
    d_pay = torch.from_numpy(pay).to(dev).repeat((F + 255) // 256, 1)[:F].contiguous()
    d_off = torch.arange(F, dtype=torch.int64, device=dev) * L; d_len = torch.full((F,), L, dtype=torch.int32, device=dev)
    nsym = -(-(L + 7) * 8 // 216); slot = 32 + 640 + 160 * (1 + nsym) + 32                    # 9824 samples: config #2's slot
    d_iq = torch.zeros((F, slot, 2), dtype=torch.int16, device=dev)
    def step(): eng.tx11a_raw(d_pay.data_ptr(), F * L, d_off.data_ptr(), d_len.data_ptr(), 0, F, rate, 32, 16, d_iq.data_ptr(), slot, 0, st.cuda_stream)
    step(); torch.cuda.synchronize()
    got = d_iq[:4, 32:32 + 640 + 160 * (1 + nsym)].cpu().numpy()
    for i in range(4):
        assert (got[i] == oracle_py.tx11a_modulate(pay[i], rate, 0xFF, 0).astype(np.int16) << 8).all(), "GPU modulator differs from the oracle"
    # the receive path decodes what the transmit path made
    s_off = torch.arange(F, dtype=torch.int64, device=dev) * slot; s_len = torch.full((F,), slot, dtype=torch.int32, device=dev)
    d_out = torch.zeros((F, 1500), dtype=torch.uint8, device=dev); d_res = torch.zeros((F, 7), dtype=torch.int32, device=dev)
    eng.rx11a_raw(d_iq.data_ptr(), F * slot, s_off.data_ptr(), s_len.data_ptr(), F, d_out.data_ptr(), 1500, d_res.data_ptr(), st.cuda_stream); torch.cuda.synchronize()
    assert (d_res[:, 0] == 1).all() and (d_out[:256, :L].cpu().numpy() == pay).all()
    for _ in range(3): step()
    e0 = torch.cuda.Event(enable_timing=True); e1 = torch.cuda.Event(enable_timing=True)
    torch.cuda.synchronize(); e0.record(st)
    for _ in range(args.steps): step()
    e1.record(st); torch.cuda.synchronize()
    ms = e0.elapsed_time(e1) / args.steps
    ncpu = os.cpu_count() or 1; n = 512
    import concurrent.futures as cf
    t0 = time.perf_counter()
    with cf.ThreadPoolExecutor(ncpu) as ex: list(ex.map(lambda i: oracle_py.tx11a_modulate(pay[i % 256], rate, 0xFF, 0), range(n)))
    dt = time.perf_counter() - t0
    alg = F * (L + slot * 4.0)
    print(json.dumps({"metric": "802.11a TX PHY Msamples/s (bytes in, IQ out)", "value": F * slot / (ms * 1e-3) / 1e6, "unit": "Msamples/s", "ms_per_step": ms, "n_gpus": 1,
                      "config": {"workload": "802.11a 54 Mbps modulator, PSDU 1500 B, COMPLEX16 slots of 9824 samples at 40 Msps (the input of BASELINE config #2 made on the device)", "frames_per_step": F},
                      "roofline": {"bound": "hbm", "achieved": alg / (ms * 1e-3) / 1e9, "peak": peaks(), "unit": "GB/s", "frac": alg / (ms * 1e-3) / 1e9 / peaks()},
                      "cpu_baseline": {"value": n * slot / dt / 1e6, "unit": "Msamples/s", "cores": ncpu, "kind": "port", "sample": f"{n} frames (python threads around the C oracle)"},
                      "parity": "bit-exact vs the transmit oracle on 4 frames; every slot decodes FRAME_OK through the receive path"}))

def bench_tx11b(args):
    import torch, oracle_py
    from sora_b200 import api
    eng = api.Engine(0); dev = torch.device("cuda", 0); st = torch.cuda.current_stream()
    F, L, rate = args.frames, 1496, 11000                    # PSDU 1500 B incl. FCS at 11 Mbps CCK, as BASELINE config #3's frames
    rng = np.random.default_rng(11)
    pay = rng.integers(0, 256, (256, L)).astype(np.uint8)
    d_pay = torch.from_numpy(pay).to(dev).repeat((F + 255) // 256, 1)[:F].contiguous()
    d_off = torch.arange(F, dtype=torch.int64, device=dev) * L; d_len = torch.full((F,), L, dtype=torch.int32, device=dev)
    lead = 392; ns = ((24 * 88 + (L + 4) * 8 + 5) * 4 + 7) // 8 * 8
    slot = (lead + ns + 200 + 55) // 56 * 56                 # whole 28-sample blocks, multiple of 8
    d_iq = torch.zeros((F, slot, 2), dtype=torch.int16, device=dev)
    def step(): eng.tx11b_raw(d_pay.data_ptr(), F * L, d_off.data_ptr(), d_len.data_ptr(), F, rate, 0, lead, 16, d_iq.data_ptr(), slot, 0, st.cuda_stream)
    step(); torch.cuda.synchronize()
    got = d_iq[:4, lead:lead + ns].cpu().numpy()
    for i in range(4):
        assert (got[i] == oracle_py.tx11b_modulate(pay[i], rate).astype(np.int16) << 8).all(), "GPU modulator differs from the oracle"
    # the receive path decodes what the transmit path made
    s_off = torch.arange(F, dtype=torch.int64, device=dev) * slot; s_len = torch.full((F,), slot, dtype=torch.int32, device=dev)
    d_out = torch.zeros((F, 1504), dtype=torch.uint8, device=dev); d_res = torch.zeros((F, 6), dtype=torch.int32, device=dev)
    eng.rx11b_raw(d_iq.data_ptr(), F * slot, s_off.data_ptr(), s_len.data_ptr(), F, d_out.data_ptr(), 1504, d_res.data_ptr(), st.cuda_stream); torch.cuda.synchronize()
    ok = float((d_res[:, 0] == 1).float().mean())
    assert ok == 1.0 and (d_out[:256, :L].cpu().numpy() == pay).all(), ok
    for _ in range(3): step()
    e0 = torch.cuda.Event(enable_timing=True); e1 = torch.cuda.Event(enable_timing=True)
    torch.cuda.synchronize(); e0.record(st)
    for _ in range(args.steps): step()
    e1.record(st); torch.cuda.synchronize()
    ms = e0.elapsed_time(e1) / args.steps
    ncpu = os.cpu_count() or 1; n = 512
    import concurrent.futures as cf
    t0 = time.perf_counter()
    with cf.ThreadPoolExecutor(ncpu) as ex: list(ex.map(lambda i: oracle_py.tx11b_modulate(pay[i % 256], rate), range(n)))
    dt = time.perf_counter() - t0
    alg = F * (L + slot * 4.0)
    print(json.dumps({"metric": "802.11b TX PHY Msamples/s (bytes in, IQ out)", "value": F * slot / (ms * 1e-3) / 1e6, "unit": "Msamples/s", "ms_per_step": ms, "n_gpus": 1,
                      "config": {"workload": "802.11b 11 Mbps CCK modulator, long preamble, PSDU 1500 B, COMPLEX16 slots of %d samples at 44 Msps (the input of BASELINE config #3 made on the device)" % slot, "frames_per_step": F},
                      "roofline": {"bound": "hbm", "achieved": alg / (ms * 1e-3) / 1e9, "peak": peaks(), "unit": "GB/s", "frac": alg / (ms * 1e-3) / 1e9 / peaks()},
                      "cpu_baseline": {"value": n * slot / dt / 1e6, "unit": "Msamples/s", "cores": ncpu, "kind": "port", "sample": f"{n} frames (python threads around the C oracle)"},
                      "parity": "bit-exact vs the transmit oracle on 4 frames; every slot decodes FRAME_OK through the 802.11b receive path"}))

def bench_tx11n(args):
    import torch, oracle_py
    from sora_b200 import api
    eng = api.Engine(0); dev = torch.device("cuda", 0); st = torch.cuda.current_stream()
    F, L = args.frames, 1496
    rng = np.random.default_rng(12)
    pay = rng.integers(0, 256, (256, L)).astype(np.uint8)
    d_pay = torch.from_numpy(pay).to(dev).repeat((F + 255) // 256, 1)[:F].contiguous()
    d_off = torch.arange(F, dtype=torch.int64, device=dev) * L; d_len = torch.full((F,), L, dtype=torch.int32, device=dev)
    for mcs in (8, 9, 10):
        nd = {8: 52, 9: 104, 10: 156}[mcs]; nsym = -(-((L + 4) * 8 + 22) // nd) + 1
        lead = 400; slot = (lead + 1600 + 160 * nsym + 200 + 27) // 28 * 28
        d0 = torch.zeros((F, slot, 2), dtype=torch.int16, device=dev); d1 = torch.zeros_like(d0)
        def step(): eng.tx11n_raw(d_pay.data_ptr(), F * L, d_off.data_ptr(), d_len.data_ptr(), 0, F, mcs, lead, d0.data_ptr(), d1.data_ptr(), slot, 0, st.cuda_stream)
        step(); torch.cuda.synchronize()
        for i in range(3):
            w0, w1 = oracle_py.tx11n_modulate(pay[i], mcs)
            assert (d0[i, lead:lead + len(w0)].cpu().numpy() == w0).all() and (d1[i, lead:lead + len(w1)].cpu().numpy() == w1).all(), "GPU modulator differs from the oracle"
        s_off = torch.arange(F, dtype=torch.int64, device=dev) * slot; s_len = torch.full((F,), slot, dtype=torch.int32, device=dev)
        d_out = torch.zeros((F, 1536), dtype=torch.uint8, device=dev); d_res = torch.zeros((F, 7), dtype=torch.int32, device=dev)
        eng.rx11n_raw(d0.data_ptr(), d1.data_ptr(), F * slot, s_off.data_ptr(), s_len.data_ptr(), F, d_out.data_ptr(), 1536, d_res.data_ptr(), st.cuda_stream); torch.cuda.synchronize()
        assert bool((d_res[:, 0] == 1).all()) and (d_out[:256, :L].cpu().numpy() == pay).all()
        for _ in range(3): step()
        e0 = torch.cuda.Event(enable_timing=True); e1 = torch.cuda.Event(enable_timing=True)
        torch.cuda.synchronize(); e0.record(st)
        for _ in range(args.steps): step()
        e1.record(st); torch.cuda.synchronize()
        ms = e0.elapsed_time(e1) / args.steps
        alg = F * (L + 2 * slot * 4.0)
        print(json.dumps({"metric": "802.11n 2-stream TX PHY Msample-pairs/s (bytes in, 2 x IQ out)", "mcs": mcs, "value": F * slot / (ms * 1e-3) / 1e6, "unit": "Msample-pairs/s", "ms_per_step": ms, "n_gpus": 1,
                          "config": {"workload": "802.11n HT-MF two-stream modulator, PSDU 1500 B, two COMPLEX16 slots of %d samples at 40 Msps per frame" % slot, "frames_per_step": F},
                          "roofline": {"bound": "hbm", "achieved": alg / (ms * 1e-3) / 1e9, "peak": peaks(), "unit": "GB/s", "frac": alg / (ms * 1e-3) / 1e9 / peaks()},
                          "parity": "bit-exact vs the transmit oracle on 3 frames; every slot pair decodes FRAME_OK through the 802.11n receive path"}))
        del d0, d1

def bench_fir37(args):
    """The legacy 802.11b transmit filter (BB11BPMDSpreadFIR4SSE) on device-resident chip streams: one frame = 1500 B at 11 Mbps CCK, 4x zero-stuffed."""
    import oracle_py
    c = Ctx(); torch = c.torch; eng, dev, st = c.eng, c.dev, c.st
    F = args.frames; L = ((24 * 88 + 1504 * 8) * 4 + 64 + 7) // 8 * 8                       # chips x 4 of one frame, rounded to the filter's 8-sample blocks
    rng = np.random.default_rng(7); U = 16
    host = np.zeros((U, L, 2), np.int8); k = rng.integers(0, 4, (U, L // 4))
    host[:, ::4, 0] = np.array([127, 0, -128, 0], np.int8)[k]; host[:, ::4, 1] = np.array([0, 127, 0, -128], np.int8)[k]
    x = torch.from_numpy(host.reshape(U, -1)).to(dev).repeat((F + U - 1) // U, 1)[:F].contiguous(); y = torch.empty_like(x)
    d_off = torch.arange(F, dtype=torch.int64, device=dev) * L; d_len = torch.full((F,), L, dtype=torch.int32, device=dev)
    def step(): eng.tx11b_fir37_raw(x.data_ptr(), F * L, d_off.data_ptr(), d_len.data_ptr(), F, 0, y.data_ptr(), st.cuda_stream)
    step(); torch.cuda.synchronize()
    got = y[:U].cpu().numpy().reshape(U, L, 2)
    for i in range(U): assert (got[i] == oracle_py.fir37_legacy(host[i], 0)).all(), "filter output differs from the oracle"
    if oracle_py.ref_fir37_available(): assert (got[0] == oracle_py.ref_fir37(host[0])).all(), "filter output differs from the reference's compiled body"
    ms = c.timed(step, args.steps)
    alg = F * L * 4.0
    c.emit({"metric": "legacy 802.11b transmit filter Msamples/s (COMPLEX8 in, COMPLEX8 out)", "value": c.world * F * L / (ms * 1e-3) / 1e6, "unit": "Msamples/s", "ms_per_step": ms, "n_gpus": c.world,
            "config": {"workload": "BB11BPMDSpreadFIR4SSE, 37 taps, 44 Msps chip streams of 1500 B / 11 Mbps frames", "frames_per_step_per_gpu": F, "samples_per_frame": L},
            "roofline": {"bound": "hbm", "achieved": alg / (ms * 1e-3) / 1e9, "peak": peaks(), "unit": "GB/s", "frac": alg / (ms * 1e-3) / 1e9 / peaks(), "note": "4 B per sample: 2 read + 2 written"},
            "parity": "equal to the oracle on the %d unique frames%s" % (U, " and to the reference's compiled filter body (oracle/_ref)" if oracle_py.ref_fir37_available() else "")})
    c.close()

def bench_tx11b_legacy(args):
    """The legacy 802.11b transmitter on the device: payload bytes in, the filtered COMPLEX8 stream of BB11BPMDPacketGenSignal out
    (short preamble, 11 Mbps CCK, 1500 B MPDUs, SSE filter body fused with the spreading)."""
    import oracle_tx11b_legacy as O
    c = Ctx(); torch = c.torch; eng, dev, st = c.eng, c.dev, c.st
    F = args.frames; L = 1500; rate = 11000
    slot = (4 * (1056 + (L + 4) * 8) + 37 + 127) // 128 * 128
    rng = np.random.default_rng(11); U = 16
    host = rng.integers(0, 256, (U, L)).astype(np.uint8)
    d_pay = torch.from_numpy(host).to(dev).repeat((F + U - 1) // U, 1)[:F].contiguous()
    d_off = torch.arange(F, dtype=torch.int64, device=dev) * L; d_len = torch.full((F,), L, dtype=torch.int32, device=dev)
    d_out = torch.empty((F, slot, 2), dtype=torch.int8, device=dev); d_ns = torch.zeros(F, dtype=torch.int32, device=dev)
    def step(): eng.tx11b_legacy_raw(d_pay.data_ptr(), F * L, d_off.data_ptr(), d_len.data_ptr(), F, rate, 1, 0, 1, d_out.data_ptr(), slot, d_ns.data_ptr(), st.cuda_stream)
    step(); torch.cuda.synchronize()
    got = d_out[:U].cpu().numpy()
    for i in range(U): assert (got[i] == O.modulate(host[i], rate, True, 1)).all(), "legacy transmitter output differs from the oracle"
    ms = c.timed(step, args.steps)
    alg = F * (slot * 2.0 + L)
    c.emit({"metric": "legacy 802.11b transmitter frames/s (bytes in, filtered COMPLEX8 out)", "value": c.world * F / (ms * 1e-3), "unit": "frames/s", "ms_per_step": ms, "n_gpus": c.world,
            "msamples_per_s": c.world * F * slot / (ms * 1e-3) / 1e6,
            "config": {"workload": "BB11BPMDPacketGenSignal: short preamble, 11 Mbps CCK, 1500 B MPDU, SSE filter, 44 Msps", "frames_per_step_per_gpu": F, "samples_per_frame": slot},
            "roofline": {"bound": "hbm", "achieved": alg / (ms * 1e-3) / 1e9, "peak": peaks(), "unit": "GB/s", "frac": alg / (ms * 1e-3) / 1e9 / peaks(), "note": "2 B per output sample written + the payload read"},
            "parity": "equal to the oracle (restated encoder + filter) on the %d unique frames" % U})
    c.close()

def bench_tx11a_legacy(args):
    """The legacy 802.11a transmitter on the device: payload bytes in, the RCB-padded COMPLEX8 signal of BB11ATxFrameMod out (54 Mbps,
    1500 B MPDUs), one row per sample rate (40 and 44 Msps)."""
    import oracle_tx11a_legacy as O
    c = Ctx(); torch = c.torch; eng, dev, st = c.eng, c.dev, c.st
    F = args.frames; L = 1500; rate = 54000
    rng = np.random.default_rng(12); U = 16
    host = rng.integers(0, 256, (U, L)).astype(np.uint8)
    d_pay = torch.from_numpy(host).to(dev).repeat((F + U - 1) // U, 1)[:F].contiguous()
    d_off = torch.arange(F, dtype=torch.int64, device=dev) * L; d_len = torch.full((F,), L, dtype=torch.int32, device=dev)
    d_pre = torch.from_numpy(O.preamble().copy()).to(dev)
    for sr in (40, 44):
        slot = O.padded_samples(L + 4, rate, sr)
        d_out = torch.empty((F, slot, 2), dtype=torch.int8, device=dev); d_ns = torch.zeros(F, dtype=torch.int32, device=dev)
        def step(): eng.tx11a_legacy_raw(d_pay.data_ptr(), F * L, d_off.data_ptr(), d_len.data_ptr(), F, rate, sr, 0, d_pre.data_ptr(), d_out.data_ptr(), slot, d_ns.data_ptr(), st.cuda_stream)
        step(); torch.cuda.synchronize()
        got = d_out[:U].cpu().numpy()
        for i in range(U): assert (got[i] == O.modulate(host[i], rate, sr)).all(), "legacy 802.11a transmitter output differs from the oracle"
        ms = c.timed(step, args.steps)
        written = F * slot * 2.0
        c.emit({"metric": "legacy 802.11a transmitter frames/s at %d Msps (bytes in, COMPLEX8 out)" % sr, "value": c.world * F / (ms * 1e-3), "unit": "frames/s", "ms_per_step": ms, "n_gpus": c.world,
                "gb_per_s_written": written / (ms * 1e-3) / 1e9,
                "config": {"workload": "BB11ATxFrameMod: 54 Mbps, 1500 B MPDU, %d Msps, RCB padded" % sr, "frames_per_step_per_gpu": F, "samples_per_frame": slot},
                "roofline": {"bound": "compute", "achieved": written / (ms * 1e-3) / 1e9, "peak": peaks(), "unit": "GB/s", "frac": written / (ms * 1e-3) / 1e9 / peaks(), "note": "2 B per output sample written; the payload read is 1 B per 8 samples"},
                "parity": "equal to the oracle on the %d unique frames" % U})
    c.close()

def bench_fir(args):
    """The anti-alias FIR decimator on a device-resident capture: the one streaming (HBM-bound) stage of the path; 6 B per input sample."""
    c = Ctx(); torch = c.torch; eng, dev, st = c.eng, c.dev, c.st
    n = args.frames * 9824 * 2                                           # twice config #2's per-step sample count
    x = torch.randint(-20000, 20000, (n, 2), dtype=torch.int16, device=dev); y = torch.empty(((n + 1) // 2, 2), dtype=torch.int16, device=dev)
    def step(): eng.fir_decimate2_raw(x.data_ptr(), n, 0, 0, y.data_ptr(), st.cuda_stream)
    step(); torch.cuda.synchronize()
    import numpy as np
    xs = x[:50000].cpu().numpy().astype(np.int64); taps = np.array([-121, 0, 209, 0, -381, 0, 644, 0, -1056, 0, 1759, 0, -3278, 0, 10391, 16434, 10391, 0, -3278, 0, 1759, 0, -1056, 0, 644, 0, -381, 0, 209, 0, -121], np.int64)
    xp = np.zeros((50000 + 32, 2), np.int64); xp[15:15 + 50000] = xs; ref = np.zeros((24000, 2), np.int64)
    for k, t in enumerate(taps):
        if t: ref += t * xp[k: k + 48000: 2]
    assert (np.clip((ref + (1 << 14)) >> 15, -32768, 32767) == y[:24000].cpu().numpy()).all(), "FIR output differs from the stated arithmetic"
    ms = c.timed(step, args.steps)
    alg = n * 6.0
    c.emit({"metric": "anti-alias FIR decimator 2:1 Msamples/s (COMPLEX16 in)", "value": c.world * n / (ms * 1e-3) / 1e6, "unit": "Msamples/s", "ms_per_step": ms, "n_gpus": c.world,
            "config": {"workload": "31-tap half-band low-pass, 40 -> 20 Msps, device-resident COMPLEX16", "samples_per_step_per_gpu": n},
            "roofline": {"bound": "hbm", "achieved": alg / (ms * 1e-3) / 1e9, "peak": peaks(), "unit": "GB/s", "frac": alg / (ms * 1e-3) / 1e9 / peaks(), "note": "6 B per input sample: 4 read + 4 written per two"},
            "parity": "equal to the arithmetic of include/sora_b200.h (numpy, 64-bit) on the first 24000 outputs"})
    c.close()

def _card():
    """(name, power limit W, max SM clock MHz) of GPU 0 as nvidia-smi reports them (None where it cannot)."""
    import subprocess
    try:
        s = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader,nounits"], capture_output=True, text=True, timeout=30).stdout
        name, pl, clk = [v.strip() for v in s.strip().splitlines()[0].split(",")]
        return name, float(pl), float(clk)
    except Exception:
        return None, None, None

def bench_channelize(args):
    """The wideband channelizer on a device-resident 160 Msps capture: four 802.11a channels at -60 / -20 / +20 / +60 MHz, 127 taps, D = 4.
    Work per input sample: K (4 + 2 ntaps / D) integer multiply-adds; HBM traffic 4 B read + 4 K / D B written."""
    import wideband_inputs as W
    c = Ctx(); torch = c.torch; eng, dev, st = c.eng, c.dev, c.st
    n = args.frames * 9824 * 4; K, D = 4, 4
    taps = W.lowpass(127, 0.1); ch = [(W.phase_inc(f, 160e6), 0) for f in (-60e6, -20e6, 20e6, 60e6)]
    n_out = -(-n // D); stride = (n_out + 3) // 4 * 4
    x = torch.randint(-20000, 20000, (n, 2), dtype=torch.int16, device=dev); y = torch.empty((K, stride, 2), dtype=torch.int16, device=dev)
    def step(): eng.channelize_raw(x.data_ptr(), n, ch, D, taps, y.data_ptr(), stride, st.cuda_stream)
    step(); torch.cuda.synchronize()
    P = 20000; m = (P - len(taps)) // D                                  # outputs that a prefix of P samples determines
    assert (W.channelize(x[:P].cpu().numpy(), ch, D, taps)[:, :m] == y[:, :m].cpu().numpy()).all(), "channelizer output differs from the stated arithmetic"
    ms = c.timed(step, args.steps)
    sec = ms * 1e-3
    hbm = n * (4.0 + 4.0 * K / D); macs = n * K * (4.0 + 2.0 * len(taps) / D)
    name, plim, clk = _card(); sms = torch.cuda.get_device_properties(dev).multi_processor_count
    imad_peak = sms * 64 * clk * 1e6 if clk else None                    # int32 IMAD: 64 per SM per clock on sm_90
    f_hbm = hbm / sec / 1e9 / peaks(); f_int = (macs / sec / imad_peak) if imad_peak else None
    c.emit({"metric": "wideband channelizer input Msamples/s (COMPLEX16 in, 4 channels, D = 4)", "value": c.world * n / sec / 1e6, "unit": "Msamples/s", "ms_per_step": ms, "n_gpus": c.world,
            "config": {"workload": "160 Msps capture, 4 x 802.11a channels at -60/-20/+20/+60 MHz, 127 taps, D = 4, device-resident", "samples_per_step_per_gpu": n},
            "hbm": {"achieved": hbm / sec / 1e9, "peak": peaks(), "unit": "GB/s", "frac": f_hbm, "note": "4 B read + 4 K / D B written per input sample"},
            "int_mad": {"achieved": macs / sec / 1e9, "peak": imad_peak / 1e9 if imad_peak else None, "unit": "G multiply-adds/s", "frac": f_int,
                        "note": "K (4 + 2 ntaps / D) per input sample; peak = SMs x 64 x max SM clock"},
            "bound": None if f_int is None else ("integer" if f_int > f_hbm else "hbm"),
            "card": name, "power_limit_w": plim,
            "parity": "equal to the numpy model of the stated arithmetic on the first %d outputs of every channel" % m})
    c.close()

def bench_spectrum(args):
    """The spectrum meter on the device-resident 160 Msps capture of --config channelize: FFT<1024> every 1024 samples, Hann window, sums of
    64 frames (a 0.41 ms display line per group).  HBM traffic: 4 B read per input sample + 8 N B per group written.  Then, in the same
    process on the same capture, the power meter over blocks of 4096 (4 B read per sample)."""
    import numpy as np
    sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), "tests"))
    import spectrum_model as SM
    c = Ctx(); torch = c.torch; eng, dev, st = c.eng, c.dev, c.st
    n = args.frames * 9824 * 4; N, hop, avg = 1024, 1024, 64
    from sora_b200 import api
    w = api.spectrum_window(N, "hann"); ng = api.spectrum_frames(n, N, hop) // avg
    x = torch.randint(-20000, 20000, (n, 2), dtype=torch.int16, device=dev); y = torch.empty((ng, N), dtype=torch.int64, device=dev)
    pb = 4096; yp = torch.empty((n // pb,), dtype=torch.int32, device=dev)
    def step(): eng.spectrum_raw(x.data_ptr(), n, 1, n, N, hop, avg, w, y.data_ptr(), st.cuda_stream)
    def pstep(): eng.power_meter_raw(x.data_ptr(), n, 1, n, pb, yp.data_ptr(), st.cuda_stream)
    step(); pstep(); torch.cuda.synchronize()
    G = 4; xs = x[:G * avg * N].cpu().numpy()
    assert (SM.spectrum(xs, N, hop, avg, w)[0] == y[:G].cpu().numpy()).all(), "spectrum differs from the model of the stated arithmetic"
    assert (SM.power_meter(xs, pb)[0] == yp[:G * avg * N // pb].cpu().numpy().view(np.uint32)).all(), "power meter differs from the model"
    ms = c.timed(step, args.steps); pms = c.timed(pstep, args.steps)
    hbm = n * 4.0 + ng * N * 8.0; phbm = n * 4.0 + (n // pb) * 4.0
    name, plim, clk = _card()
    c.emit({"metric": "spectrum meter input Msamples/s (COMPLEX16 in, FFT<1024>, Hann, avg 64)", "value": c.world * n / (ms * 1e-3) / 1e6, "unit": "Msamples/s",
            "ms_per_step": ms, "n_gpus": c.world,
            "config": {"workload": "160 Msps capture, N = 1024, hop 1024, Hann, avg 64, device-resident", "samples_per_step_per_gpu": n, "groups": ng},
            "hbm": {"achieved": hbm / (ms * 1e-3) / 1e9, "peak": peaks(), "unit": "GB/s", "frac": hbm / (ms * 1e-3) / 1e9 / peaks(), "note": "4 B read per input sample + 8 N B per group"},
            "power_meter": {"block_len": pb, "ms_per_step": pms, "Msamples_per_s": n / (pms * 1e-3) / 1e6, "hbm_GBps": phbm / (pms * 1e-3) / 1e9},
            "card": name, "power_limit_w": plim, "max_sm_clock_mhz": clk,
            "parity": "equal to tests/spectrum_model.py on the first %d groups and their power-meter blocks" % G})
    c.close()

def bench_channelize_bank(args):
    """The filter-bank channelizer on the device-resident 160 Msps capture of --config channelize: all eight odd-stacked channels
    (+-10 / +-30 / +-50 / +-70 MHz), 255 taps, D = 4; and, in the same process on the same capture, sb200_channelize on the same eight
    channels and taps, the way a user would take the band apart without the bank.  Integer work per input sample: bank
    2 ntaps / D + 4 M^2 / D (branch sums and the direct M-point DFT), channelizer K (4 + 2 ntaps / D)."""
    import wideband_inputs as W, bank_model as B
    c = Ctx(); torch = c.torch; eng, dev, st = c.eng, c.dev, c.st
    n = args.frames * 9824 * 4; M, D = 8, 4
    taps = W.lowpass(255, 10e6 / 160e6); ch = B.phase_incs(M, 1)
    n_out = -(-n // D); stride = (n_out + 3) // 4 * 4
    x = torch.randint(-20000, 20000, (n, 2), dtype=torch.int16, device=dev); y = torch.empty((M, stride, 2), dtype=torch.int16, device=dev)
    P = 20000; m = (P - len(taps)) // D                                  # outputs that a prefix of P samples determines
    def bank(): eng.channelize_bank_raw(x.data_ptr(), n, M, D, taps, y.data_ptr(), stride, odd=True, stream=st.cuda_stream)
    def chan(): eng.channelize_raw(x.data_ptr(), n, ch, D, taps, y.data_ptr(), stride, st.cuda_stream)
    bank(); torch.cuda.synchronize()
    assert (B.window(x[:P].cpu().numpy(), M, D, 1, taps, 0, m) == y[:, :m].cpu().numpy()).all(), "filter-bank output differs from the stated arithmetic"
    chan(); torch.cuda.synchronize()
    assert (W.channelize(x[:P].cpu().numpy(), ch, D, taps)[:, :m] == y[:, :m].cpu().numpy()).all(), "channelizer output differs from the stated arithmetic"
    ms_bank = c.timed(bank, args.steps); ms_chan = c.timed(chan, args.steps)
    name, plim, clk = _card(); sms = torch.cuda.get_device_properties(dev).multi_processor_count
    imad_peak = sms * 64 * clk * 1e6 if clk else None                    # int32 IMAD: 64 per SM per clock on sm_90
    hbm = n * (4.0 + 4.0 * M / D)
    for what, ms, work, note in (("filter-bank channelizer (sb200_channelize_bank)", ms_bank, n * (2.0 * len(taps) / D + 4.0 * M * M / D), "2 ntaps / D + 4 M^2 / D per input sample"),
                                 ("wideband channelizer (sb200_channelize) on the same channels", ms_chan, n * M * (4.0 + 2.0 * len(taps) / D), "K (4 + 2 ntaps / D) per input sample")):
        sec = ms * 1e-3; f_int = (work / sec / imad_peak) if imad_peak else None
        c.emit({"metric": "%s input Msamples/s (COMPLEX16 in, 8 odd-stacked channels, 255 taps, D = 4)" % what, "value": c.world * n / sec / 1e6, "unit": "Msamples/s",
                "ms_per_step": ms, "n_gpus": c.world, "bank_speedup": ms_chan / ms_bank,
                "config": {"workload": "160 Msps capture, 8 x 20 MHz channels at +-10/30/50/70 MHz, 255 taps, D = 4, device-resident", "samples_per_step_per_gpu": n},
                "hbm": {"achieved": hbm / sec / 1e9, "peak": peaks(), "unit": "GB/s", "frac": hbm / sec / 1e9 / peaks(), "note": "4 B read + 4 M / D B written per input sample"},
                "int_mad": {"achieved": work / sec / 1e9, "peak": imad_peak / 1e9 if imad_peak else None, "unit": "G multiply-adds/s", "frac": f_int,
                            "note": note + "; peak = SMs x 64 x max SM clock"},
                "card": name, "power_limit_w": plim, "sm_clock_max_mhz": clk,
                "parity": "equal to the numpy model of the stated arithmetic on the first %d outputs of every channel" % m})
    c.close()

def bench_channelize_rational(args):
    """The rational-rate channelizer on a device-resident 160 Msps capture the size of --config channelize's: three 802.11b channels at
    -25 / 0 / +25 MHz brought to 44 Msps (U = 11, D = 40) through 1287 taps (117 per branch).  Work per input sample: K (4 + 2 ntaps / D)
    integer multiply-adds (each output meets one branch of ntaps / U taps, and there are U / D outputs per input); HBM traffic 4 B read +
    4 K U / D B written."""
    import wideband_inputs as W, rational_model as R
    c = Ctx(); torch = c.torch; eng, dev, st = c.eng, c.dev, c.st
    n = args.frames * 9824 * 4; K, U, D = 3, 11, 40
    taps = W.lowpass(1287, 12e6 / 1.76e9, gain=11); ch = [(W.phase_inc(f, 160e6), 0) for f in (-25e6, 0.0, 25e6)]
    n_out = -(-U * n // D); stride = (n_out + 3) // 4 * 4
    x = torch.randint(-20000, 20000, (n, 2), dtype=torch.int16, device=dev); y = torch.empty((K, stride, 2), dtype=torch.int16, device=dev)
    def step(): eng.channelize_raw(x.data_ptr(), n, ch, D, taps, y.data_ptr(), stride, st.cuda_stream, interp=U)
    step(); torch.cuda.synchronize()
    P = 20000; m = (U * P - len(taps)) // D                              # outputs that a prefix of P samples determines
    assert (R.channelize_rational(x[:P].cpu().numpy(), ch, U, D, taps)[:, :m] == y[:, :m].cpu().numpy()).all(), "channelizer output differs from the stated arithmetic"
    ms = c.timed(step, args.steps)
    sec = ms * 1e-3
    hbm = n * (4.0 + 4.0 * K * U / D); macs = n * K * (4.0 + 2.0 * len(taps) / D)
    name, plim, clk = _card(); sms = torch.cuda.get_device_properties(dev).multi_processor_count
    imad_peak = sms * 64 * clk * 1e6 if clk else None                    # int32 IMAD: 64 per SM per clock on sm_90
    f_hbm = hbm / sec / 1e9 / peaks(); f_int = (macs / sec / imad_peak) if imad_peak else None
    c.emit({"metric": "rational channelizer input Msamples/s (COMPLEX16 in, 3 channels, U / D = 11 / 40)", "value": c.world * n / sec / 1e6, "unit": "Msamples/s", "ms_per_step": ms,
            "n_gpus": c.world,
            "config": {"workload": "160 Msps capture, 3 x 802.11b channels at -25/0/+25 MHz to 44 Msps, 1287 taps, U = 11, D = 40, device-resident", "samples_per_step_per_gpu": n},
            "hbm": {"achieved": hbm / sec / 1e9, "peak": peaks(), "unit": "GB/s", "frac": f_hbm, "note": "4 B read + 4 K U / D B written per input sample"},
            "int_mad": {"achieved": macs / sec / 1e9, "peak": imad_peak / 1e9 if imad_peak else None, "unit": "G multiply-adds/s", "frac": f_int,
                        "note": "K (4 + 2 ntaps / D) per input sample; peak = SMs x 64 x max SM clock"},
            "bound": None if f_int is None else ("integer" if f_int > f_hbm else "hbm"),
            "card": name, "power_limit_w": plim, "sm_clock_max_mhz": clk,
            "parity": "equal to the numpy model of the stated arithmetic on the first %d outputs of every channel" % m})
    c.close()

def bench_channelize_arbitrary(args):
    """The arbitrary-rate channelizer on device-resident captures the size of --config channelize's, 64-tap tables.
    1. --config channelize_rational's workload: three 802.11b channels at -25 / 0 / +25 MHz of 160 Msps to 44 Msps (step 160 / 44), timed in
       the same process beside sb200_channelize_rational (U / D = 11 / 40, 1287 taps) on the same capture.  The two use different filters:
       a data point, not a like-for-like comparison.
    2. A 122.88 Msps capture of the 2.4 GHz band, which no other call brings to the receivers' rates: 802.11b at -25 and +25 MHz to 44 Msps
       and OFDM at 0 Hz to 40 Msps, two calls per step.
    Integer work per output: 2 ntaps multiply-adds per component pair, plus 4 per input sample and rotating channel (the rotation)."""
    import wideband_inputs as W, rational_model as R, arbitrary_model as A
    from sora_b200 import api
    c = Ctx(); torch = c.torch; eng, dev, st = c.eng, c.dev, c.st
    n = args.frames * 9824 * 4; P = 20000
    x = torch.randint(-20000, 20000, (n, 2), dtype=torch.int16, device=dev); xp = x[:P].cpu().numpy()
    name, plim, clk = _card(); sms = torch.cuda.get_device_properties(dev).multi_processor_count
    imad_peak = sms * 64 * clk * 1e6 if clk else None                    # int32 IMAD: 64 per SM per clock on sm_90
    def calls(fs, plan):
        """plan: [(centres, fs_out, passband, stop band)] -> (step function, [(channels, step, taps, n_out)], output buffers)"""
        out = []
        for fcs, fo, fp, fsb in plan:
            ch = [(W.phase_inc(f, fs), 0) for f in fcs]; step = api.arbitrary_step(fs, fo); taps = api.arbitrary_taps(fs, fo, 64, fp, fsb)
            n_out = A.n_inside(n, 0, step); y = torch.empty((len(ch), (n_out + 3) // 4 * 4, 2), dtype=torch.int16, device=dev)
            out.append((ch, step, taps, n_out, y))
        def step_fn():
            for ch, step, taps, n_out, y in out: eng.channelize_arbitrary_raw(x.data_ptr(), n, ch, 0, step, taps, y.data_ptr(), y.shape[1], n_out, stream=st.cuda_stream)
        step_fn(); torch.cuda.synchronize()
        for ch, step, taps, n_out, y in out:
            m = ((P - 64) << 32) // step                                 # outputs that a prefix of P samples determines
            assert (A.channelize_arbitrary(xp, ch, 0, step, taps, m) == y[:, :m].cpu().numpy()).all(), "arbitrary-rate output differs from the stated arithmetic"
        return step_fn, out
    def emit(what, ms, out, workload, extra):
        sec = ms * 1e-3; work = sum(len(ch) * (n_o * 2.0 * taps.shape[1] + 4.0 * n * any(a or b >> 20 for a, b in ch)) for ch, _, taps, n_o, _ in out)
        f_int = (work / sec / imad_peak) if imad_peak else None
        c.emit(dict({"metric": "%s input Msamples/s (COMPLEX16 in)" % what, "value": c.world * n / sec / 1e6, "unit": "Msamples/s", "ms_per_step": ms, "n_gpus": c.world,
                     "config": {"workload": workload, "samples_per_step_per_gpu": n},
                     "int_mad": {"achieved": work / sec / 1e9, "peak": imad_peak / 1e9 if imad_peak else None, "unit": "G multiply-adds/s", "frac": f_int,
                                 "note": "2 ntaps per output and channel + 4 per input sample and rotating channel; peak = SMs x 64 x max SM clock"},
                     "card": name, "power_limit_w": plim, "sm_clock_max_mhz": clk,
                     "parity": "equal to the numpy model of the stated arithmetic on the outputs a %d-sample prefix determines" % P}, **extra))
    arb160, out160 = calls(160e6, [((-25e6, 0.0, 25e6), 44e6, 9e6, 17e6)])
    U, D = 11, 40; rtaps = W.lowpass(1287, 12e6 / 1.76e9, gain=11); rch = out160[0][0]
    n_r = -(-U * n // D); yr = torch.empty((3, (n_r + 3) // 4 * 4, 2), dtype=torch.int16, device=dev)
    def rat(): eng.channelize_raw(x.data_ptr(), n, rch, D, rtaps, yr.data_ptr(), yr.shape[1], st.cuda_stream, interp=U)
    rat(); torch.cuda.synchronize()
    m = (U * P - len(rtaps)) // D
    assert (R.channelize_rational(xp, rch, U, D, rtaps)[:, :m] == yr[:, :m].cpu().numpy()).all(), "channelizer output differs from the stated arithmetic"
    ms_arb = c.timed(arb160, args.steps); ms_rat = c.timed(rat, args.steps)
    emit("arbitrary-rate channelizer (sb200_channelize_arbitrary), 160 -> 44 Msps", ms_arb, out160,
         "160 Msps capture, 3 x 802.11b channels at -25/0/+25 MHz to 44 Msps, 64-tap table, step 160 / 44, device-resident",
         {"rational_ms_per_step": ms_rat, "rational_msamples_per_s": c.world * n / (ms_rat * 1e-3) / 1e6,
          "rational_note": "sb200_channelize_rational on the same capture and channels: U / D = 11 / 40, 1287 taps (a different filter)"})
    del out160, yr
    arb122, out122 = calls(122.88e6, [((-25e6, 25e6), 44e6, 9e6, 17e6), ((0.0,), 40e6, 8.3e6, 17e6)])
    ms = c.timed(arb122, args.steps)
    emit("arbitrary-rate channelizer (sb200_channelize_arbitrary), 122.88 -> 44 and 40 Msps", ms, out122,
         "122.88 Msps capture of the 2.4 GHz band: 802.11b at -25/+25 MHz to 44 Msps and OFDM at 0 Hz to 40 Msps (two calls), 64-tap tables, device-resident", {})
    c.close()

def bench_combine(args):
    """The wideband combiner into a device-resident 160 Msps capture: four 802.11a channel rows at 40 Msps moved to -60 / -20 / +20 / +60 MHz,
    127 taps, U = 4; as many output samples as --config channelize reads.  Work per output sample: K (2 ceil(ntaps / U) + 4 + 2) integer
    multiply-adds; HBM traffic 4 B written + 4 K / U B read."""
    import wideband_inputs as W, combine_model as CM
    c = Ctx(); torch = c.torch; eng, dev, st = c.eng, c.dev, c.st
    K, U = 4, 4; n_out = args.frames * 9824 * 4; n_in = n_out // U
    taps = W.lowpass(127, 0.1, gain=U); ch = [(W.phase_inc(f, 160e6), 0, 4096) for f in (-60e6, -20e6, 20e6, 60e6)]
    x = torch.randint(-8000, 8000, (K, n_in, 2), dtype=torch.int16, device=dev); y = torch.empty((n_out, 2), dtype=torch.int16, device=dev)
    def step(): eng.combine_raw(x.data_ptr(), n_in, n_in, ch, U, taps, y.data_ptr(), st.cuda_stream)
    step(); torch.cuda.synchronize()
    P = 5000; m = U * P - len(taps)                                      # outputs that a prefix of P input samples determines
    assert (CM.combine(x[:, :P].cpu().numpy(), ch, U, taps)[:m] == y[:m].cpu().numpy()).all(), "combiner output differs from the stated arithmetic"
    ms = c.timed(step, args.steps)
    sec = ms * 1e-3
    hbm = n_out * (4.0 + 4.0 * K / U); macs = n_out * K * (2.0 * -(-len(taps) // U) + 6.0)
    name, plim, clk = _card(); sms = torch.cuda.get_device_properties(dev).multi_processor_count
    imad_peak = sms * 64 * clk * 1e6 if clk else None                    # int32 IMAD: 64 per SM per clock on sm_90
    f_hbm = hbm / sec / 1e9 / peaks(); f_int = (macs / sec / imad_peak) if imad_peak else None
    c.emit({"metric": "wideband combiner output Msamples/s (COMPLEX16 out, 4 channels, U = 4)", "value": c.world * n_out / sec / 1e6, "unit": "Msamples/s", "ms_per_step": ms, "n_gpus": c.world,
            "config": {"workload": "4 x 802.11a rows at 40 Msps -> 160 Msps capture, channels at -60/-20/+20/+60 MHz, 127 taps, U = 4, device-resident", "output_samples_per_step_per_gpu": n_out},
            "hbm": {"achieved": hbm / sec / 1e9, "peak": peaks(), "unit": "GB/s", "frac": f_hbm, "note": "4 B written + 4 K / U B read per output sample"},
            "int_mad": {"achieved": macs / sec / 1e9, "peak": imad_peak / 1e9 if imad_peak else None, "unit": "G multiply-adds/s", "frac": f_int,
                        "note": "K (2 ceil(ntaps / U) + 4 + 2) per output sample; peak = SMs x 64 x max SM clock"},
            "bound": None if f_int is None else ("integer" if f_int > f_hbm else "hbm"),
            "card": name, "power_limit_w": plim, "max_sm_clock_mhz": clk,
            "parity": "equal to the numpy model of the stated arithmetic on the first %d outputs" % m})
    c.close()

def bench_combine_bank(args):
    """The filter-bank combiner into a device-resident 160 Msps capture of --config combine's size: eight odd-stacked rows at 40 Msps
    (+-10 / +-30 / +-50 / +-70 MHz), 255 taps, U = 4; and, in the same process on the same rows, sb200_combine on the same eight channels and
    taps, the way a user would fill the grid without the bank.  Integer work per output sample: bank 2 ntaps / U + 4 M^2 / U (the branch
    filter and the direct M-point IDFT), combiner K (2 ceil(ntaps / U) + 6)."""
    import wideband_inputs as W, combine_bank_model as CB
    c = Ctx(); torch = c.torch; eng, dev, st = c.eng, c.dev, c.st
    M, U = 8, 4; n_out = args.frames * 9824 * 4; n_in = n_out // U
    taps = W.lowpass(255, 10e6 / 160e6, gain=U); ch = CB.channels(M, 1)
    x = torch.randint(-8000, 8000, (M, n_in, 2), dtype=torch.int16, device=dev); y = torch.empty((n_out, 2), dtype=torch.int16, device=dev)
    P = 5000; m = U * P - len(taps)                                      # outputs that a prefix of P input samples determines
    def bank(): eng.combine_bank_raw(x.data_ptr(), n_in, n_in, M, U, taps, y.data_ptr(), n_out, odd=True, stream=st.cuda_stream)
    def comb(): eng.combine_raw(x.data_ptr(), n_in, n_in, ch, U, taps, y.data_ptr(), st.cuda_stream)
    bank(); torch.cuda.synchronize()
    xp = x[:, :P].cpu().numpy()
    assert (CB.window(xp, M, U, 1, taps, 0, m) == y[:m].cpu().numpy()).all(), "filter-bank output differs from the stated arithmetic"
    ms_bank = c.timed(bank, args.steps); ms_comb = c.timed(comb, args.steps)
    name, plim, clk = _card(); sms = torch.cuda.get_device_properties(dev).multi_processor_count
    imad_peak = sms * 64 * clk * 1e6 if clk else None                    # int32 IMAD: 64 per SM per clock on sm_90
    hbm = n_out * (4.0 + 4.0 * M / U)
    for what, ms, work, note in (("filter-bank combiner (sb200_combine_bank)", ms_bank, n_out * (2.0 * len(taps) / U + 4.0 * M * M / U), "2 ntaps / U + 4 M^2 / U per output sample"),
                                 ("wideband combiner (sb200_combine) on the same channels", ms_comb, n_out * M * (2.0 * -(-len(taps) // U) + 6.0), "K (2 ceil(ntaps / U) + 6) per output sample")):
        sec = ms * 1e-3; f_int = (work / sec / imad_peak) if imad_peak else None
        c.emit({"metric": "%s output Gsamples/s (COMPLEX16 out, 8 odd-stacked channels, 255 taps, U = 4)" % what, "value": c.world * n_out / sec / 1e9, "unit": "Gsamples/s",
                "ms_per_step": ms, "n_gpus": c.world, "bank_speedup": ms_comb / ms_bank,
                "config": {"workload": "8 rows at 40 Msps -> 160 Msps capture, channels at +-10/30/50/70 MHz, 255 taps, U = 4, device-resident", "output_samples_per_step_per_gpu": n_out},
                "hbm": {"achieved": hbm / sec / 1e9, "peak": peaks(), "unit": "GB/s", "frac": hbm / sec / 1e9 / peaks(), "note": "4 B written + 4 M / U B read per output sample"},
                "int_mad": {"achieved": work / sec / 1e9, "peak": imad_peak / 1e9 if imad_peak else None, "unit": "G multiply-adds/s", "frac": f_int,
                            "note": note + "; peak = SMs x 64 x max SM clock"},
                "card": name, "power_limit_w": plim, "sm_clock_max_mhz": clk,
                "parity": "bank equal to the numpy model of the stated arithmetic on the first %d outputs" % m})
    c.close()

def bench_combine_rational(args):
    """The rational-rate combiner into a device-resident 160 Msps capture the size of --config combine's: three 802.11b rows at 44 Msps
    moved to -25 / 0 / +25 MHz, U / D = 40 / 11 through 1761 taps (45 per branch; --ratio U/D picks another pair, with 45 taps per branch
    of a low-pass at 0.55 of the row's Nyquist).  Work per output sample: K (2 ceil(ntaps / U) + 4 + 2) integer multiply-adds; HBM traffic
    4 B written + 4 K D / U B read."""
    import wideband_inputs as W, combine_rational_model as CR
    c = Ctx(); torch = c.torch; eng, dev, st = c.eng, c.dev, c.st
    U, D = (int(v) for v in args.ratio.split("/")); K = 3; n_out = args.frames * 9824 * 4; n_in = -(-D * n_out // U); stride = (n_in + 3) // 4 * 4
    taps = W.lowpass(1761, 12e6 / 1.76e9, gain=40) if (U, D) == (40, 11) else W.lowpass(45 * U - 1 + (U % 2), 0.275 / U, gain=U)
    ch = [(W.phase_inc(f, 160e6), 0, 4096) for f in (-25e6, 0.0, 25e6)]
    x = torch.randint(-8000, 8000, (K, stride, 2), dtype=torch.int16, device=dev); y = torch.empty((n_out, 2), dtype=torch.int16, device=dev)
    def step(): eng.combine_raw(x.data_ptr(), stride, n_in, ch, U, taps, y.data_ptr(), st.cuda_stream, decim=D, n_out=n_out)
    step(); torch.cuda.synchronize()
    m = 20000                                                            # the first outputs, from the inputs they read
    assert (CR.combine_rational_window(x[:, :D * m // U + len(taps)].cpu().numpy(), ch, U, D, taps, 0, m) == y[:m].cpu().numpy()).all(), "combiner output differs from the stated arithmetic"
    ms = c.timed(step, args.steps)
    sec = ms * 1e-3
    hbm = n_out * (4.0 + 4.0 * K * D / U); macs = n_out * K * (2.0 * -(-len(taps) // U) + 6.0)
    name, plim, clk = _card(); sms = torch.cuda.get_device_properties(dev).multi_processor_count
    imad_peak = sms * 64 * clk * 1e6 if clk else None                    # int32 IMAD: 64 per SM per clock on sm_90
    f_hbm = hbm / sec / 1e9 / peaks(); f_int = (macs / sec / imad_peak) if imad_peak else None
    c.emit({"metric": "rational combiner output Msamples/s (COMPLEX16 out, 3 channels, U / D = %d / %d)" % (U, D), "value": c.world * n_out / sec / 1e6, "unit": "Msamples/s", "ms_per_step": ms,
            "n_gpus": c.world,
            "config": {"workload": "3 x 802.11b rows at 44 Msps -> 160 Msps capture, channels at -25/0/+25 MHz, %d taps, U = %d, D = %d, device-resident" % (len(taps), U, D), "output_samples_per_step_per_gpu": n_out},
            "hbm": {"achieved": hbm / sec / 1e9, "peak": peaks(), "unit": "GB/s", "frac": f_hbm, "note": "4 B written + 4 K D / U B read per output sample"},
            "int_mad": {"achieved": macs / sec / 1e9, "peak": imad_peak / 1e9 if imad_peak else None, "unit": "G multiply-adds/s", "frac": f_int,
                        "note": "K (2 ceil(ntaps / U) + 4 + 2) per output sample; peak = SMs x 64 x max SM clock"},
            "bound": None if f_int is None else ("integer" if f_int > f_hbm else "hbm"),
            "card": name, "power_limit_w": plim, "max_sm_clock_mhz": clk,
            "parity": "equal to the numpy model of the stated arithmetic on the first %d outputs" % m})
    c.close()

def bench_combine_arbitrary(args):
    """The arbitrary-rate combiner into device-resident captures of --config combine's size, 64-tap tables (api.arbitrary_taps):
    1. Three 802.11b rows at 44 Msps moved to -25 / 0 / +25 MHz of a 160 Msps capture (step 44 / 160), timed in the same process beside
       sb200_combine_rational (U / D = 40 / 11, 1761 taps) on the same rows.  The two use different filters: a data point, not a
       like-for-like comparison.
    2. The 2.4 GHz band at 122.88 Msps, which no other call reaches from the transmitters' rates: 802.11b rows at -25 and +25 MHz from
       44 Msps, then the OFDM row at 0 Hz from 40 Msps added onto them, two calls per step.
    Work per output sample and row: 2 ntaps integer multiply-adds of the filter + 4 of the rotation + 2 of the gain; HBM traffic 4 B written
    (plus 4 B read with accumulate) per output sample + 4 B read per row sample."""
    import wideband_inputs as W, combine_arbitrary_model as CA, combine_rational_model as CR, arbitrary_model as A
    from sora_b200 import api
    c = Ctx(); torch = c.torch; eng, dev, st = c.eng, c.dev, c.st
    n_out = args.frames * 9824 * 4; P = 20000
    name, plim, clk = _card(); sms = torch.cuda.get_device_properties(dev).multi_processor_count
    imad_peak = sms * 64 * clk * 1e6 if clk else None                    # int32 IMAD: 64 per SM per clock on sm_90
    def calls(fs, plan):
        """plan: [(centres, row rate, passband)], one call each, the later ones added onto the earlier -> (step function, [(channels, step,
        taps, rows, n_in)], output)"""
        y = torch.empty((n_out, 2), dtype=torch.int16, device=dev); out = []
        for fcs, fr, fp in plan:
            ch = [(W.phase_inc(f, fs), 0, 4096) for f in fcs]; step = api.arbitrary_step(fr, fs); taps = api.arbitrary_taps(fr, fs, 64, fp)
            n_in = (n_out * step >> 32) + 64; n_in += (-n_in) % 4
            out.append((ch, step, taps, torch.randint(-8000, 8000, (len(ch), n_in, 2), dtype=torch.int16, device=dev), n_in))
        def step_fn():
            for i, (ch, step, taps, x, n_in) in enumerate(out):
                eng.combine_arbitrary_raw(x.data_ptr(), n_in, n_in, ch, 0, step, taps, y.data_ptr(), n_out, accumulate=i > 0, stream=st.cuda_stream)
        step_fn(); torch.cuda.synchronize()
        m = min(((P - 64) << 32) // step for _, step, _, _, _ in out)    # outputs that a prefix of P row samples determines
        want = None
        for ch, step, taps, x, _ in out: want = CA.combine_arbitrary_window(x[:, :P].cpu().numpy(), ch, 0, step, taps, 0, m, want)
        assert (want == y[:m].cpu().numpy()).all(), "arbitrary-rate combiner output differs from the stated arithmetic"
        return step_fn, out, m
    def emit(what, ms, out, m, workload, extra):
        sec = ms * 1e-3
        work = n_out * sum(len(ch) * (2.0 * taps.shape[1] + 6.0) for ch, _, taps, _, _ in out)
        hbm = n_out * 4.0 * (2 * len(out) - 1) + sum(4.0 * len(ch) * n_in for ch, _, _, _, n_in in out)
        f_hbm = hbm / sec / 1e9 / peaks(); f_int = (work / sec / imad_peak) if imad_peak else None
        c.emit(dict({"metric": "%s output Msamples/s (COMPLEX16 out)" % what, "value": c.world * n_out / sec / 1e6, "unit": "Msamples/s", "ms_per_step": ms, "n_gpus": c.world,
                     "config": {"workload": workload, "output_samples_per_step_per_gpu": n_out},
                     "hbm": {"achieved": hbm / sec / 1e9, "peak": peaks(), "unit": "GB/s", "frac": f_hbm,
                             "note": "per call 4 B written (+ 4 B read with accumulate) per output sample + 4 B read per row sample"},
                     "int_mad": {"achieved": work / sec / 1e9, "peak": imad_peak / 1e9 if imad_peak else None, "unit": "G multiply-adds/s", "frac": f_int,
                                 "note": "K (2 ntaps + 6) per output sample and call; peak = SMs x 64 x max SM clock"},
                     "bound": None if f_int is None else ("integer" if f_int > f_hbm else "hbm"),
                     "card": name, "power_limit_w": plim, "max_sm_clock_mhz": clk,
                     "parity": "equal to the numpy model of the stated arithmetic on the first %d outputs" % m}, **extra))
    arb160, out160, m160 = calls(160e6, [((-25e6, 0.0, 25e6), 44e6, 9e6)])
    U, D = 40, 11; rtaps = W.lowpass(1761, 12e6 / 1.76e9, gain=40); ch, _, _, x, n_in = out160[0]
    n_r = -(-D * n_out // U); yr = torch.empty((n_out, 2), dtype=torch.int16, device=dev)
    def rat(): eng.combine_raw(x.data_ptr(), n_in, n_r, ch, U, rtaps, yr.data_ptr(), st.cuda_stream, decim=D, n_out=n_out)
    rat(); torch.cuda.synchronize()
    mr = 20000
    assert (CR.combine_rational_window(x[:, :D * mr // U + len(rtaps)].cpu().numpy(), ch, U, D, rtaps, 0, mr) == yr[:mr].cpu().numpy()).all(), "combiner output differs from the stated arithmetic"
    ms_arb = c.timed(arb160, args.steps); ms_rat = c.timed(rat, args.steps)
    emit("arbitrary-rate combiner (sb200_combine_arbitrary), 44 -> 160 Msps", ms_arb, out160, m160,
         "3 x 802.11b rows at 44 Msps -> 160 Msps capture, channels at -25/0/+25 MHz, 64-tap table, step 44 / 160, device-resident",
         {"rational_ms_per_step": ms_rat, "rational_msamples_per_s": c.world * n_out / (ms_rat * 1e-3) / 1e6,
          "rational_note": "sb200_combine_rational on the same rows and channels: U / D = 40 / 11, 1761 taps (a different filter)"})
    del out160, yr, x
    arb122, out122, m122 = calls(122.88e6, [((-25e6, 25e6), 44e6, 9e6), ((0.0,), 40e6, 8.3e6)])
    ms = c.timed(arb122, args.steps)
    emit("arbitrary-rate combiner (sb200_combine_arbitrary), 44 and 40 -> 122.88 Msps", ms, out122, m122,
         "122.88 Msps capture of the 2.4 GHz band: 802.11b rows at -25/+25 MHz from 44 Msps, then OFDM at 0 Hz from 40 Msps added onto them (two calls), 64-tap tables, device-resident", {})
    c.close()

def bench_sim(args):
    """The radio channel simulator on device-resident links of config #2's slot length (9 824 samples at 40 Msps): T = R = 1 with 16 taps,
    and T = R = 2 with 16 taps per pair, every link at +20 ppm with a carrier offset and noise.  Integer work per output sample, from the
    shapes: 16 T multiply-adds of the interpolation, 4 T L of the taps, 4 of the rotation and the noise's two 64-bit products (counted as
    8), plus half a Philox4x32-10 block (20 32-bit multiplies); HBM traffic 4 T B read + 4 R B written per output sample and row."""
    import sim_model as SM
    from sora_b200 import api
    c = Ctx(); torch = c.torch; eng, dev, st = c.eng, c.dev, c.st
    name, plim, clk = _card(); sms = torch.cuda.get_device_properties(dev).multi_processor_count
    imad_peak = sms * 64 * clk * 1e6 if clk else None                    # int32 IMAD: 64 per SM per clock on sm_90
    for T, R, nl in ((1, 1, args.frames * 2), (2, 2, args.frames // 2)):
        L = 16; n = 9824; n_out = n
        x = torch.randint(-8000, 8000, (nl, T, n, 2), dtype=torch.int16, device=dev); y = torch.empty((nl, R, n_out, 2), dtype=torch.int16, device=dev)
        rng = np.random.default_rng(T)
        links = api.sim_links([(int(rng.integers(0, 2 ** 32)), api.clock_step(20), api.phase_inc(-20e-6 * 5.2e9, 40e6), int(rng.integers(0, 2 ** 32)), 2000) for _ in range(nl)])
        taps = rng.integers(-1000, 1000, (nl, R, T, L, 2)).astype(np.int16); taps[:, :, :, 0, 0] = 12000
        dl = torch.from_numpy(links.view(np.uint8).copy()).to(dev); dt = torch.from_numpy(taps).to(dev)
        def step(): eng.channel_sim_raw(x.data_ptr(), T * n, n, T, n, dl.data_ptr(), dt.data_ptr(), L, nl, 0x5EED, y.data_ptr(), R * n_out, n_out, R, n_out, st.cuda_stream)
        step(); torch.cuda.synchronize()
        pick = [0, nl - 1]
        want = SM.sim_window(x[pick].cpu().numpy(), links[pick], taps[pick], 0x5EED, 0, 3000, link_ids=pick)
        assert (y[pick, :, :3000].cpu().numpy() == want).all(), "channel simulator output differs from the stated arithmetic"
        ms = c.timed(step, args.steps); sec = ms * 1e-3
        outs = nl * R * n_out
        work = outs * (16.0 * T + 4.0 * T * L + 4 + 8 + 20 / 2)
        hbm = nl * n_out * (4.0 * T + 4.0 * R)
        f_int = (work / sec / imad_peak) if imad_peak else None; f_hbm = hbm / sec / 1e9 / peaks()
        c.emit({"metric": "channel simulator output Msamples/s (COMPLEX16, T = %d, R = %d, L = %d)" % (T, R, L), "value": c.world * outs / sec / 1e6, "unit": "Msamples/s",
                "ms_per_step": ms, "n_gpus": c.world,
                "config": {"workload": "%d links x 9824 samples at 40 Msps, +20 ppm, carrier offset, noise, device-resident" % nl, "output_samples_per_step_per_gpu": outs},
                "hbm": {"achieved": hbm / sec / 1e9, "peak": peaks(), "unit": "GB/s", "frac": f_hbm, "note": "4 T B read + 4 R B written per output sample of a row"},
                "int_ops": {"achieved": work / sec / 1e9, "peak": imad_peak / 1e9 if imad_peak else None, "unit": "G integer multiply-adds/s", "frac": f_int,
                            "note": "16 T + 4 T L + 4 + 8 + 10 per output sample and row; peak = SMs x 64 x max SM clock"},
                "card": name, "power_limit_w": plim, "max_sm_clock_mhz": clk,
                "parity": "equal to the numpy model of the stated arithmetic on the first 3000 outputs of the first and last links"})
    c.close()

if __name__ == "__main__":
    ap = argparse.ArgumentParser()
    ap.add_argument("--config", choices=["viterbi", "11b", "11n", "tx11a", "tx11b", "tx11n", "fir", "fir37", "tx11b_legacy", "tx11a_legacy", "channelize", "channelize_bank", "channelize_rational", "channelize_arbitrary", "combine", "combine_bank", "combine_rational", "combine_arbitrary", "spectrum", "sim"], required=True)
    ap.add_argument("--steps", type=int, default=5)
    ap.add_argument("--blocks", type=int, default=0, help="Viterbi code blocks per GPU (0 = BASELINE config #5: 1e9 coded bits in total over all GPUs)")
    ap.add_argument("--frames", type=int, default=32768)
    ap.add_argument("--ratio", default="40/11", help="U/D of --config combine_rational; the channel plan stays three rows at -25/0/+25 MHz of 160 Msps, and "
                    "a pair other than 40/11 takes a generic low-pass of 45 taps per branch at 0.55 of the row's Nyquist")
    ap.add_argument("--mcs", default="8,9,10", help="802.11n MCS list for --config 11n (11..14 enable the engine option ht_mcs_limit = 15)")
    a = ap.parse_args()
    {"viterbi": bench_viterbi, "11b": bench_11b, "11n": bench_11n, "tx11a": bench_tx11a, "tx11b": bench_tx11b, "tx11n": bench_tx11n, "fir": bench_fir, "fir37": bench_fir37, "tx11b_legacy": bench_tx11b_legacy, "tx11a_legacy": bench_tx11a_legacy, "channelize": bench_channelize, "channelize_bank": bench_channelize_bank, "channelize_rational": bench_channelize_rational, "channelize_arbitrary": bench_channelize_arbitrary, "combine": bench_combine, "combine_bank": bench_combine_bank, "combine_rational": bench_combine_rational, "combine_arbitrary": bench_combine_arbitrary, "spectrum": bench_spectrum, "sim": bench_sim}[a.config](a)
