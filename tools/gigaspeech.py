"""Timings of GigaSpeech's Conformer-Transducer (12 layers, d_model 768, RelPosMHAXL with 8 heads of 96; proj_enc 768 -> 512,
LSTM 512, joint 512, 1024 tokens) on one GPU, on seeded weights (tests/gigaspeech_oracle.py):

* the RelPosMHAXL encoder attention kernel alone at 8 heads of 96 against 12 heads of 64, the Loquacious-large shape at the
  same d_model 768 (equal attention FLOPs and equal P traffic): B = 32 at T = 251, B = 4 and B = 32 at T = 2500, every
  other utterance at 70 % length.  Through the kernel test hooks, which synchronise after each launch: CUDA events over 50
  launches per window, 5 windows.  With the CTAs per SM each instantiation reaches (cudaOccupancyMaxActiveBlocksPerMultiprocessor);
* wav -> encoder states of 32 x 10 s (AsrEngine.encode_wav), and the beam-10 transducer search (state_beam = expand_beam
  = 2.3) on proj_enc of those states: CUDA events around whole calls after warm-up, --reps windows;
* one streaming chunk of the encoder (TransformerASR.encode_streaming, features to encoder states) followed by the greedy
  transducer search on its proj_enc output, at 1 and 32 streams for DynChunkTrainConfig (32, 4) and (16, 8), in steady
  state (the left context full): device time per chunk from CUDA events, and the host time of enqueueing it;
* --profile: a separate torch.profiler run of one 32 x 10 s encode (the attention kernel's total CUDA time from the
  trace), and the attention kernel's per-launch device time at the shapes above, without the hook's synchronisation.

Every time is printed as the median with min and max.  Prints one JSON object with the GPU name and power limit read in
the same run."""
import argparse
import ctypes
import json
import math
import os
import subprocess
import sys
import time

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))


def gpu_info():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True)
    return q.stdout.strip()


def events(fn, n, windows=5):
    """(median, min, max) over windows of the mean time (ms) of n calls of fn"""
    for _ in range(3):
        fn()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    out = []
    for _ in range(windows):
        e0.record()
        for _ in range(n):
            fn()
        e1.record()
        torch.cuda.synchronize()
        out.append(e0.elapsed_time(e1) / n)
    out.sort()
    return dict(median=out[len(out) // 2], min=out[0], max=out[-1])


def scaled(t, k):
    return {key: v * k for key, v in t.items()}


def enc_attention(dev, B, T, H, dh):
    from speechbrain_b200._lib import check, lib, ptr, stream_ptr
    d = H * dh
    qkv = torch.randn(B * T, 3 * d, device=dev).half()
    out = torch.empty(B * T, d, device=dev, dtype=torch.float16)
    u = 0.1 * torch.randn(d, device=dev)
    P = torch.randn(T, d, device=dev).half()
    lens = torch.full((B,), T, dtype=torch.int32, device=dev)
    lens[1::2] = int(0.7 * T)
    scale = ctypes.c_float(1 / math.sqrt(d))
    f = lambda: check(lib().sbk_encoder_attention_window_test(ptr(qkv), None, B, T, H, dh, ptr(lens), 1, ptr(u), ptr(u),  # noqa: E731
                                                              ptr(P), scale, 0, -1, 0, 0, 0, ptr(out), stream_ptr(dev)),
                      "encoder attention")
    return scaled(events(f, 50), 1000)


def occupancy(dh, stream_form):
    from speechbrain_b200._lib import check, lib
    n = ctypes.c_int(0)
    check(lib().sbk_encoder_attention_occupancy(dh, int(stream_form), ctypes.byref(n)), "occupancy")
    return n.value


def model(dev):
    import gigaspeech_oracle as GO
    from mirrors import build_mirror
    from speechbrain_b200.engine import AsrEngine
    cfg = GO.config()
    sd, w_enc, W = GO.weights()
    return cfg, sd, w_enc.to(dev), W, AsrEngine(cfg, sd, device=str(dev)), build_mirror(cfg, sd)


def searcher(W, beam):
    import gigaspeech_oracle as GO
    import test_gpu_transducer as GT
    from speechbrain_b200.decoders.transducer import TransducerBeamSearcher
    g, _, mods = GT.build(GO.J, GO.H, GO.V, GO.BLANK, GO.PN_SEED)
    for prefix, m in mods.items():
        m.load_state_dict({k[len(prefix) + 1:]: v for k, v in W.items() if k.startswith(prefix + ".")})
    if beam == 1:
        return g
    return TransducerBeamSearcher(list(g.decode_network_lst), g.tjoint, list(g.classifier_network), blank_id=GO.BLANK,
                                  beam_size=beam, nbest=1, state_beam=GO.STATE_BEAM, expand_beam=GO.EXPAND_BEAM)


def model_times(dev, B, reps):
    import gigaspeech_oracle as GO
    from speechbrain_b200.utils.dynamic_chunk_training import DynChunkTrainConfig
    cfg, sd, w_enc, W, eng, mirror = model(dev)
    g = torch.Generator().manual_seed(0)
    wav = torch.randn(B, 160000, generator=g).to(dev)
    lens = torch.ones(B, device=dev)
    res = {"encode_32x10s_ms": events(lambda: eng.encode_wav(wav, lens), 1, reps)}
    tn = (eng.encode_wav(wav, lens) @ w_enc.T).contiguous()
    bs = searcher(W, GO.BEAM)
    res["beam10_32x10s_ms"] = events(lambda: bs(tn), 1, reps)
    greedy = searcher(W, 1)
    tr = mirror.tr
    src_all = mirror.front_end()(wav, lens)
    src_all = src_all.reshape(B, src_all.shape[1], -1)
    for cs, lc in ((32, 4), (16, 8)):
        for n in (1, 32):
            src = src_all[:n]
            ctx = tr.make_streaming_context(DynChunkTrainConfig(cs, lc))
            n_fill = lc + 1
            for k in range(n_fill):  # steady state: the left context holds lc chunks
                tr.encode_streaming(src[:, k * cs:(k + 1) * cs].contiguous(), ctx)
            chunk = src[:, n_fill * cs:(n_fill + 1) * cs].contiguous()
            wt = w_enc.T.contiguous()
            host = []

            def step():
                t0 = time.perf_counter()
                x = tr.encode_streaming(chunk, ctx) @ wt
                greedy.device_search(x.device).greedy(x.contiguous(), 0, GO.MAX_SYMBOLS, None)
                host.append(time.perf_counter() - t0)
            t = events(step, 10, reps)
            host.sort()
            res[f"stream_chunk_{cs}_{lc}_B{n}_ms"] = t
            res[f"stream_chunk_{cs}_{lc}_B{n}_host_ms"] = dict(median=1e3 * host[len(host) // 2], min=1e3 * host[0],
                                                               max=1e3 * host[-1])
    return res


def kernel_times(dev):
    """per-launch device time (us) of the attention kernel at each shape, from a torch.profiler trace of 20 launches:
    free of the test hook's per-launch host synchronisation"""
    from torch.profiler import ProfilerActivity, profile

    from speechbrain_b200._lib import check, lib, ptr, stream_ptr
    res = {}
    for B, T in ((32, 251), (4, 2500), (32, 2500)):
        for H, dh in ((8, 96), (12, 64)):
            d = H * dh
            qkv = torch.randn(B * T, 3 * d, device=dev).half()
            out = torch.empty(B * T, d, device=dev, dtype=torch.float16)
            u = 0.1 * torch.randn(d, device=dev)
            P = torch.randn(T, d, device=dev).half()
            lens = torch.full((B,), T, dtype=torch.int32, device=dev)
            lens[1::2] = int(0.7 * T)
            f = lambda: check(lib().sbk_encoder_attention_window_test(  # noqa: E731
                ptr(qkv), None, B, T, H, dh, ptr(lens), 1, ptr(u), ptr(u), ptr(P), ctypes.c_float(1 / math.sqrt(d)), 0, -1,
                0, 0, 0, ptr(out), stream_ptr(dev)), "encoder attention")
            for _ in range(3):
                f()
            with profile(activities=[ProfilerActivity.CUDA]) as prof:
                for _ in range(20):
                    f()
            ev = sorted(getattr(e, "device_time", 0) or e.cuda_time for e in prof.events() if "encoder_attention_kernel" in e.name)
            res[f"kernel_B{B}_T{T}_H{H}_dh{dh}_us"] = dict(median=ev[len(ev) // 2], min=ev[0], max=ev[-1])
    return res


def profile_encode(dev, out_dir):
    from torch.profiler import ProfilerActivity, profile
    _, _, _, _, eng, _ = model(dev)
    wav = torch.randn(32, 160000, device=dev)
    lens = torch.ones(32, device=dev)
    eng.encode_wav(wav, lens)
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        eng.encode_wav(wav, lens)
        torch.cuda.synchronize()
    if out_dir:
        prof.export_chrome_trace(os.path.join(out_dir, "gigaspeech_encode.json"))
    att = [e for e in prof.key_averages() if "encoder_attention_kernel" in e.key]
    total = sum(e.device_time_total for e in prof.key_averages())
    return {"encoder_attention_us_per_encode": sum(e.device_time_total for e in att), "all_kernels_us_per_encode": total}


def main():
    ap = argparse.ArgumentParser(description=__doc__.split("\n")[0])
    ap.add_argument("--batch", type=int, default=32)
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--profile", action="store_true", help="only the torch.profiler run")
    ap.add_argument("--kernels-only", action="store_true", help="only the attention kernels and their occupancy")
    ap.add_argument("--out-dir", default=None, help="where --profile writes its trace")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("gigaspeech.py measures on a GPU; none found")
    dev = torch.device("cuda:0")
    res = {"gpu": gpu_info()}
    if args.profile:
        res.update(profile_encode(dev, args.out_dir))
        res.update(kernel_times(dev))
    else:
        res["ctas_per_sm"] = {"dh96": occupancy(96, False), "dh96_stream": occupancy(96, True), "dh64": occupancy(64, False),
                              "dh64_stream": occupancy(64, True)}
        for B, T in ((32, 251), (4, 2500), (32, 2500)):
            for H, dh in ((8, 96), (12, 64)):
                res[f"enc_attention_relpos_B{B}_T{T}_H{H}_dh{dh}_us"] = enc_attention(dev, B, T, H, dh)
        if not args.kernels_only:
            res.update(model_times(dev, args.batch, args.reps))
    print(json.dumps(res))


if __name__ == "__main__":
    main()
