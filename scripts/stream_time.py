"""Streaming vocoding of 64 live sessions (the 64 seeded utterance lengths of scripts/ragged_time.py, uniform in [86, 861]
mel frames), every session pushing n frames per step (the last push carries END), served three ways on the same weights:
  stream  one Generator.stream step per push (mg_gen_stream_step: cached left context per kernel boundary)
  halo    one forward_ragged per step over windows with an 8-frame halo either side (what GeneratorHost.stream does for one
          session, batched): a chunk is emitted once the 8 frames after it have arrived
  whole   one ragged forward of the whole utterances (the floor: no streaming at all)
The packed mel of every step is built before the timed passes.  Per arm and n: total device time of the schedule (CUDA
events, no synchronisation inside), and per-step latency from call to audio ready (host clock around step + synchronise),
median and p95; arms alternated REPS times.  Then one session at n in {4, 8, 16}: step latency.  Every arm's audio is
compared with the whole forward (stream: torch.equal).  --profile: a separate torch.profiler run of the stream at each n that
splits device time between the window-assembly copies and the chain kernels; the bytes those copies move come from
mg_gen_stream_dry_step on the same schedule.  Writes a JSON record with the card's name, power limit and clock cap."""
import argparse
import ctypes
import json
import subprocess
import sys
import time

import numpy as np
import torch

sys.path.insert(0, ".")
from melgan_multi_b200 import engine, models, synth

B, LO, HI, SEED, REPS, HALO = 64, 86, 861, 2024, 3, 8
PUSH = (4, 8, 16, 32)


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True).stdout.strip().splitlines()
    return q[torch.cuda.current_device()] if q else "unknown"


def stream_schedule(mel, lens, n):
    """Per step: (packed mel [S, 80, n], frames, flags) for sessions pushing n frames per step."""
    S = len(lens)
    steps = []
    for s in range((max(lens) + n - 1) // n):
        m = torch.zeros((S, 80, n), device="cuda")
        frames, flags = [], []
        for i, L in enumerate(lens):
            a, b = min(L, s * n), min(L, (s + 1) * n)
            m[i, :, :b - a] = mel[i, :, a:b]
            frames.append(b - a)
            flags.append(engine.STREAM_END if a < L and b == L else 0)
        steps.append((m, frames, flags))
    return steps


def halo_schedule(mel, lens, n):
    """Per step: (mel windows [B', 80, T'], window lengths, [(session, crop start, crop end, out frame lo, hi)])."""
    S = len(lens)
    done = [0] * S
    steps = []
    for s in range((max(lens) + n - 1) // n):
        wins = []
        for i, L in enumerate(lens):
            have = min(L, (s + 1) * n)
            hi = L if have == L else max(done[i], have - HALO)
            if hi <= done[i]:
                continue
            lo = done[i]
            a, b = max(0, lo - HALO), min(L, hi + HALO)
            wins.append((i, a, b, lo, hi))
            done[i] = hi
        if not wins:
            steps.append(None)
            continue
        Tm = max(b - a for _, a, b, _, _ in wins)
        m = torch.zeros((len(wins), 80, Tm), device="cuda")
        for j, (i, a, b, _, _) in enumerate(wins):
            m[j, :, :b - a] = mel[i, :, a:b]
        steps.append((m, [b - a for _, a, b, _, _ in wins], wins))
    return steps


def run_stream(gen, steps, S, n, keep=False):
    st = gen.stream(S, n)
    outs = [[] for _ in range(S)] if keep else None
    for m, frames, flags in steps:
        audio, counts = st.step_packed(m, frames, flags)
        if keep:
            for i, c in enumerate(counts):
                outs[i].append(audio[i, :c])
    return st, outs


def run_halo(gen, steps, S, keep=False):
    dev = gen._ensure_packed()
    outs = [[] for _ in range(S)] if keep else None
    for step in steps:
        if step is None:
            continue
        m, lens, wins = step
        y = dev.forward_ragged(m, lens)
        if keep:
            for j, (i, a, _b, lo, hi) in enumerate(wins):
                outs[i].append(y[j, 0, 256 * (lo - a):256 * (hi - a)])
    return outs


def timed(fn):
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    fn()
    b.record()
    torch.cuda.synchronize()
    return a.elapsed_time(b)


def step_latencies_stream(gen, steps, S, n):
    st = gen.stream(S, n)
    ms = []
    for m, frames, flags in steps:
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        st.step_packed(m, frames, flags)
        torch.cuda.synchronize()
        ms.append(1e3 * (time.perf_counter() - t0))
    st.check_status()
    return ms


def step_latencies_halo(gen, steps):
    dev = gen._ensure_packed()
    ms = []
    for step in steps:
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        if step is not None:
            dev.forward_ragged(step[0], step[1])
        torch.cuda.synchronize()
        ms.append(1e3 * (time.perf_counter() - t0))
    return ms


def stats(v):
    return {"median_ms": float(np.median(v)), "p95_ms": float(np.percentile(v, 95)), "n": len(v)}


def dry_bytes(lens, n):
    """Bytes the window-assembly and audio copies move over the whole schedule, and the frames it pushes."""
    L = engine.lib()
    S = len(lens)
    h = ctypes.c_void_p()
    assert L.mg_gen_stream_create(ctypes.byref(h), S, n, 0, ctypes.c_void_p(1 << 20), L.mg_gen_stream_state_bytes(S, n)) == 0
    total = 0
    try:
        for s in range((max(lens) + n - 1) // n):
            frames = [max(0, min(Lk, (s + 1) * n) - min(Lk, s * n)) for Lk in lens]
            flags = [engine.STREAM_END if min(Lk, s * n) < Lk <= (s + 1) * n else 0 for Lk in lens]
            cnt, nb = (ctypes.c_int * S)(), ctypes.c_longlong()
            engine.check(L.mg_gen_stream_dry_step(h, (ctypes.c_int * S)(*frames), (ctypes.c_int * S)(*flags), S, cnt, None,
                                                  ctypes.byref(nb)))
            total += nb.value
    finally:
        L.mg_gen_stream_destroy(h)
    return total


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default="profiles/h100_stream.json")
    ap.add_argument("--profile", action="store_true", help="torch.profiler split of the stream's device time instead")
    args = ap.parse_args()
    g = models.Generator()
    g.load_state_dict({k: torch.from_numpy(v) for k, v in synth.generator_state(1234).items()})
    g = g.cuda().eval()
    lens = [int(v) for v in np.random.default_rng(SEED).integers(LO, HI + 1, B)]
    T = max(lens)
    mel = torch.zeros(B, 80, T, device="cuda")
    for i, L in enumerate(lens):
        mel[i, :, :L] = torch.from_numpy(synth.mel_input(1, L, SEED + i)[0])
    rec = {"card": card(), "workload": {"sessions": B, "frames": sum(lens), "lengths_uniform_in": [LO, HI], "seed": SEED,
                                        "audio_seconds": sum(lens) * 256 / 22050.0}}
    with torch.no_grad():
        whole = g.generate(mel, lens)
        ref = [whole[i, 0, :256 * L] for i, L in enumerate(lens)]
        if args.profile:
            from torch.profiler import ProfilerActivity, profile
            prof_rec = {}
            for n in PUSH:
                steps = stream_schedule(mel, lens, n)
                run_stream(g, steps, B, n)
                torch.cuda.synchronize()
                with profile(activities=[ProfilerActivity.CUDA]) as prof:
                    run_stream(g, steps, B, n)
                    torch.cuda.synchronize()
                per = {}
                for e in prof.key_averages():
                    t = getattr(e, "device_time_total", None) or getattr(e, "cuda_time_total", 0)
                    if t:
                        per[e.key] = per.get(e.key, 0.0) + t / 1e3
                copy = sum(v for k, v in per.items() if "stream_window_kernel" in k)
                chain = sum(v for k, v in per.items() if "stream_window_kernel" not in k and "Memset" not in k and "Memcpy" not in k
                            and "fill" not in k.lower() and "copy" not in k.lower())
                nbytes = dry_bytes(lens, n)
                prof_rec[str(n)] = {"window_copy_ms": copy, "chain_kernels_ms": chain, "copy_share": copy / (copy + chain),
                                    "copy_bytes": nbytes, "copy_bytes_per_frame": nbytes / sum(lens),
                                    "copy_GB_per_s": nbytes / (copy * 1e-3) / 1e9 if copy else None,
                                    "kernels_ms": dict(sorted(per.items(), key=lambda kv: -kv[1])[:16])}
            rec["profile"] = prof_rec
        else:
            sched = {n: (stream_schedule(mel, lens, n), halo_schedule(mel, lens, n)) for n in PUSH}
            # audio identity, and a warm-up of every shape
            ident = {}
            for n, (ss, hs) in sched.items():
                st, so = run_stream(g, ss, B, n, keep=True)
                ho = run_halo(g, hs, B, keep=True)
                torch.cuda.synchronize()
                st.check_status()
                s_eq = all(torch.equal(torch.cat(so[i]), ref[i]) for i in range(B))
                h_dev = max(float((torch.cat(ho[i]) - ref[i]).abs().max()) for i in range(B))
                ident[str(n)] = {"stream_bit_identical": s_eq, "halo_max_abs_dev": h_dev}
            rec["identity"] = ident
            tot = {a: {str(n): [] for n in PUSH} for a in ("stream", "halo", "whole")}
            lat = {a: {str(n): [] for n in PUSH} for a in ("stream", "halo")}
            for _ in range(REPS):
                for n, (ss, hs) in sched.items():
                    tot["stream"][str(n)].append(timed(lambda: run_stream(g, ss, B, n)))
                    tot["halo"][str(n)].append(timed(lambda: run_halo(g, hs, B)))
                    tot["whole"][str(n)].append(timed(lambda: g.generate(mel, lens)))
                    lat["stream"][str(n)] += step_latencies_stream(g, ss, B, n)
                    lat["halo"][str(n)] += step_latencies_halo(g, hs)
            rec["total_ms"] = {a: {n: {"median": float(np.median(v)), "min": min(v), "max": max(v), "runs": v} for n, v in d.items()}
                               for a, d in tot.items()}
            rec["step_latency"] = {a: {n: stats(v) for n, v in d.items()} for a, d in lat.items()}
            one = {}
            L1 = max(lens)
            m1 = mel[lens.index(L1):lens.index(L1) + 1]
            ref1 = g.generate(m1[:, :, :L1].contiguous())[0, 0]
            for n in (4, 8, 16):
                ss = stream_schedule(m1, [L1], n)
                _, so = run_stream(g, ss, 1, n, keep=True)
                assert torch.equal(torch.cat(so[0]), ref1)
                v = []
                for _ in range(REPS):
                    v += step_latencies_stream(g, ss, 1, n)
                one[str(n)] = stats(v)
            rec["one_session_step_latency"] = one
    print(json.dumps(rec, indent=1))
    with open(args.out, "w") as f:
        json.dump(rec, f, indent=1)


if __name__ == "__main__":
    main()
