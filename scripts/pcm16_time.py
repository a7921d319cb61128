"""16-bit PCM output against converting fp32 audio after the call, on the same weights and inputs:
  config2   B = 64, T = 32: generate() then a correct torch conversion, against generate(dtype=torch.int16)
  ragged    the 64-utterance workload of scripts/ragged_time.py (lengths uniform in [86, 861] frames), the same two arms
  host      GeneratorHost.forward (float, then the same conversion in numpy) against forward(dtype=np.int16), end to end:
            host clock around each call, which copies in, runs, copies out and synchronises; pinned output buffers
  stream    64 sessions pushing 8 frames per step for 32 steps (END on the last): float steps with one conversion per
            returned slot, against int16 steps; host clock around the whole run, ended by a synchronise
A "correct conversion" is where(isnan(a), 0, clamp(round(32768 a), -32768, 32767)).to(int16) (round: half to even).  Every
pair of arms is checked to give identical int16 audio.  Arms alternate; each reports the median of REPS runs and the
min / max.  Writes a JSON record with the card's name and power limit (default profiles/h100_pcm16.json)."""
import argparse
import json
import subprocess
import sys
import time

import numpy as np
import torch

sys.path.insert(0, ".")
from melgan_multi_b200 import engine, models, synth

B_RAG, LO, HI, SEED, REPS = 64, 86, 861, 2024, 5
S_STREAM, PUSH, STEPS = 64, 8, 32


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True).stdout.strip().splitlines()
    return q[torch.cuda.current_device()] if q else "unknown"


def to_pcm16(a):
    return torch.where(torch.isnan(a), 0.0, torch.clamp(torch.round(a * 32768.0), -32768.0, 32767.0)).to(torch.int16)


def to_pcm16_np(a):
    s = np.clip(np.rint(a * np.float32(32768.0)), -32768, 32767)
    s[np.isnan(a)] = 0
    return s.astype(np.int16)


def stats(v):
    return {"median": float(np.median(v)), "min": float(np.min(v)), "max": float(np.max(v)), "runs": [float(x) for x in v]}


def device_ms(f):
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    out = f()
    b.record()
    b.synchronize()
    return a.elapsed_time(b), out


def host_ms(f):
    torch.cuda.synchronize()
    t = time.perf_counter()
    out = f()
    torch.cuda.synchronize()
    return 1e3 * (time.perf_counter() - t), out


def alternate(arms, timer):
    """{name: stats} over REPS alternated runs (after one warm-up each); asserts the arms' outputs are identical."""
    outs = {k: f() for k, f in arms.items()}
    torch.cuda.synchronize()
    ms = {k: [] for k in arms}
    for _ in range(REPS):
        for k, f in arms.items():
            t, outs[k] = timer(f)
            ms[k].append(t)
    ref = None
    for k, o in outs.items():
        o = o.cpu().numpy() if torch.is_tensor(o) else (np.concatenate([x.cpu().numpy() for x in o], axis=None)
                                                          if isinstance(o, list) else o)
        assert ref is None or np.array_equal(o, ref), k
        ref = o
    return {k: stats(v) for k, v in ms.items()}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default="profiles/h100_pcm16.json")
    args = ap.parse_args()
    state = synth.generator_state(1234)
    g = models.Generator()
    g.load_state_dict({k: torch.from_numpy(v) for k, v in state.items()})
    g = g.cuda().eval()
    rec = {"card": card(), "reps": REPS, "note": "median / min / max in ms over alternated runs"}

    with torch.no_grad():
        mel2 = torch.from_numpy(synth.mel_input(64, 32, 7)).cuda()
        rec["config2_device_ms"] = alternate({"float_then_convert": lambda: to_pcm16(g.generate(mel2)),
                                              "int16": lambda: g.generate(mel2, dtype=torch.int16)}, device_ms)
        lens = [int(v) for v in np.random.default_rng(SEED).integers(LO, HI + 1, B_RAG)]
        T = max(lens)
        mel = torch.zeros(B_RAG, 80, T, device="cuda")
        for i, L in enumerate(lens):
            mel[i, :, :L] = torch.from_numpy(synth.mel_input(1, L, SEED + i)[0])
        rec["ragged_device_ms"] = alternate({"float_then_convert": lambda: to_pcm16(g.generate(mel, lens)),
                                             "int16": lambda: g.generate(mel, lens, dtype=torch.int16)}, device_ms)
        rec["ragged_audio_bytes"] = {"float": 4 * B_RAG * 256 * T, "int16": 2 * B_RAG * 256 * T}

    eng = engine.GeneratorHost(B_RAG, T)
    try:
        eng.load_state(state)
        host = {}
        for name, m, ln in (("config2", mel2.cpu().numpy(), None), ("ragged", mel.cpu().numpy(), lens)):
            B_, _, T_ = m.shape
            f_out = torch.empty((B_, 1, 256 * T_), dtype=torch.float32).pin_memory().numpy()
            i_out = torch.empty((B_, 1, 256 * T_), dtype=torch.int16).pin_memory().numpy()
            if ln is None:
                arms = {"float_then_convert": lambda: to_pcm16_np(eng.forward(m, out=f_out)),
                        "int16": lambda: eng.forward(m, out=i_out, dtype=np.int16).copy()}
            else:
                arms = {"float_then_convert": lambda: to_pcm16_np(eng.forward_ragged(m, ln, out=f_out)),
                        "int16": lambda: eng.forward_ragged(m, ln, out=i_out, dtype=np.int16).copy()}
            host[name] = alternate(arms, host_ms)
        rec["host_engine_ms"] = host
    finally:
        eng.close()

    with torch.no_grad():
        smel = torch.from_numpy(synth.mel_input(S_STREAM, PUSH * STEPS, 99)).cuda()

        def run(dtype):
            st = g.stream(S_STREAM, PUSH, dtype=dtype)
            pieces = [[] for _ in range(S_STREAM)]
            for k in range(STEPS):
                chunks = [smel[i, :, k * PUSH:(k + 1) * PUSH] for i in range(S_STREAM)]
                outs = st.step(chunks, end=[k == STEPS - 1] * S_STREAM)
                for i, o in enumerate(outs):
                    pieces[i].append(to_pcm16(o) if dtype == torch.float32 else o)
            st.check_status()
            st.close()
            return [torch.cat(p, dim=1) for p in pieces]
        rec["stream_64x8_ms"] = alternate({"float_then_convert": lambda: run(torch.float32),
                                           "int16": lambda: run(torch.int16)}, host_ms)
        rec["stream_shape"] = {"sessions": S_STREAM, "push_frames": PUSH, "steps": STEPS}
    print(json.dumps(rec, indent=1))
    with open(args.out, "w") as f:
        json.dump(rec, f, indent=1)


if __name__ == "__main__":
    main()
