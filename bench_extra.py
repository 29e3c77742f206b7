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

if __name__ == "__main__":
    ap = argparse.ArgumentParser()
    ap.add_argument("--config", choices=["viterbi", "11b", "11n", "tx11a", "tx11b", "tx11n", "fir", "fir37", "tx11b_legacy", "tx11a_legacy", "channelize"], required=True)
    ap.add_argument("--steps", type=int, default=5)
    ap.add_argument("--blocks", type=int, default=0, help="Viterbi code blocks per GPU (0 = BASELINE config #5: 1e9 coded bits in total over all GPUs)")
    ap.add_argument("--frames", type=int, default=32768)
    ap.add_argument("--mcs", default="8,9,10", help="802.11n MCS list for --config 11n (11..14 enable the engine option ht_mcs_limit = 15)")
    a = ap.parse_args()
    {"viterbi": bench_viterbi, "11b": bench_11b, "11n": bench_11n, "tx11a": bench_tx11a, "tx11b": bench_tx11b, "tx11n": bench_tx11n, "fir": bench_fir, "fir37": bench_fir37, "tx11b_legacy": bench_tx11b_legacy, "tx11a_legacy": bench_tx11a_legacy, "channelize": bench_channelize}[a.config](a)
