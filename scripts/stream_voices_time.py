"""Streaming 16 voices x 4 live sessions (the 64 seeded utterance lengths of scripts/ragged_time.py, uniform in [86, 861]
mel frames; session i belongs to voice i // 4, each voice a Generator of its own seed), every session pushing n frames per
step (the last push carries END), served four ways:
  voices    one models.stream_voices handle of 64 sessions (mg_gen_stream_step_voices: one step for every voice)
  handles   16 one-voice handles (Generator.stream, 4 sessions each), stepped one after another on one stream
  streams   the same 16 handles spread round-robin over 4 CUDA streams, joined back after each step
  floor     one voice with 64 sessions (Generator.stream): what the voices arm would cost with no voice change at all
The packed mel of every step is built before the timed passes.  Per arm and n in {4, 8, 16}: total device time of the
schedule (CUDA events around it, no synchronisation inside), and per-step latency from call to audio ready (host clock
around one step of every session + synchronise), median and p95; the arms alternated REPS times.  Every arm's audio is
checked against the whole-utterance forward of its voice (torch.equal).  Writes a JSON record with the card's name,
power limit and clock cap (default profiles/h100_stream_voices.json)."""
import argparse
import json
import subprocess
import sys
import time

import numpy as np
import torch

sys.path.insert(0, ".")
from melgan_multi_b200 import engine, models, synth

V, PER, LO, HI, SEED, REPS, NSTREAMS = 16, 4, 86, 861, 2024, 3, 4
PUSH = (4, 8, 16)
ARMS = ("voices", "handles", "streams", "floor")


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True).stdout.strip().splitlines()
    return q[torch.cuda.current_device()] if q else "unknown"


def schedule(mel, lens, n):
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


class Arm:
    """Fresh handles for one pass of one arm; step(k) runs step k of the schedule for every session."""

    def __init__(self, kind, gens, steps, n, streams):
        self.kind, self.steps, self.streams = kind, steps, streams
        B = V * PER
        if kind == "voices":
            self.handles = [models.stream_voices(gens, B, n)]
            self.voice = [i // PER for i in range(B)]
        elif kind == "floor":
            self.handles = [gens[0].stream(B, n)]
        else:
            self.handles = [g.stream(PER, n) for g in gens]
        self.outs = [[] for _ in range(B)]

    def step(self, k, keep=False):
        m, frames, flags = self.steps[k]
        if self.kind in ("voices", "floor"):
            audio, counts = self.handles[0].step_packed(m, frames, flags, voice=self.voice if self.kind == "voices" else None)
            parts = [(0, audio, counts)]
        elif self.kind == "handles":
            parts = []
            for v, h in enumerate(self.handles):
                sl = slice(v * PER, (v + 1) * PER)
                audio, counts = h.step_packed(m[sl], frames[sl], flags[sl])
                parts.append((v * PER, audio, counts))
        else:
            cur = torch.cuda.current_stream()
            for s in self.streams:
                s.wait_stream(cur)
            parts = []
            for v, h in enumerate(self.handles):
                sl = slice(v * PER, (v + 1) * PER)
                with torch.cuda.stream(self.streams[v % NSTREAMS]):
                    audio, counts = h.step_packed(m[sl], frames[sl], flags[sl])
                    audio.record_stream(cur)
                parts.append((v * PER, audio, counts))
            for s in self.streams:
                cur.wait_stream(s)
        if keep:
            for i0, audio, counts in parts:
                for j, c in enumerate(counts):
                    self.outs[i0 + j].append(audio[j, :c])

    def run(self, keep=False):
        for k in range(len(self.steps)):
            self.step(k, keep)

    def check_status(self):
        for h in self.handles:
            h.check_status()


def stats(v):
    return {"median_ms": float(np.median(v)), "p95_ms": float(np.percentile(v, 95)), "n": len(v)}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default="profiles/h100_stream_voices.json")
    args = ap.parse_args()
    gens = []
    for v in range(V):
        g = models.Generator()
        g.load_state_dict({k: torch.from_numpy(a) for k, a in synth.generator_state(1000 + v).items()})
        gens.append(g.cuda().eval())
    B = V * PER
    lens = [int(v) for v in np.random.default_rng(SEED).integers(LO, HI + 1, B)]
    T = max(lens)
    mel = torch.zeros(B, 80, T, device="cuda")
    for i, L in enumerate(lens):
        mel[i, :, :L] = torch.from_numpy(synth.mel_input(1, L, SEED + i)[0])
    streams = [torch.cuda.Stream() for _ in range(NSTREAMS)]
    rec = {"card": card(),
           "workload": {"voices": V, "sessions_per_voice": PER, "frames": sum(lens), "lengths_uniform_in": [LO, HI],
                        "seed": SEED, "voice_seeds": [1000, 1000 + V - 1], "audio_seconds": sum(lens) * 256 / 22050.0,
                        "push_frames": list(PUSH), "streams_arm_streams": NSTREAMS, "passes": REPS}}
    with torch.no_grad():
        voice = [i // PER for i in range(B)]
        ref = models.generate_voices(gens, mel, voice, lens)
        ref_floor = gens[0].generate(mel, lens)
        sched = {n: schedule(mel, lens, n) for n in PUSH}
        ident = {}
        for n, steps in sched.items():  # audio identity, and a warm-up of every shape
            ident[str(n)] = {}
            for kind in ARMS:
                arm = Arm(kind, gens, steps, n, streams)
                arm.run(keep=True)
                torch.cuda.synchronize()
                arm.check_status()
                want = ref_floor if kind == "floor" else ref
                ident[str(n)][kind] = all(torch.equal(torch.cat(arm.outs[i]), want[i, 0, :256 * L]) for i, L in enumerate(lens))
        rec["bit_identical"] = ident
        tot = {a: {str(n): [] for n in PUSH} for a in ARMS}
        lat = {a: {str(n): [] for n in PUSH} for a in ARMS}
        for _ in range(REPS):
            for n, steps in sched.items():
                for kind in ARMS:
                    arm = Arm(kind, gens, steps, n, streams)
                    torch.cuda.synchronize()
                    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                    a.record()
                    arm.run()
                    b.record()
                    torch.cuda.synchronize()
                    tot[kind][str(n)].append(a.elapsed_time(b))
                for kind in ARMS:
                    arm = Arm(kind, gens, steps, n, streams)
                    for k in range(len(steps)):
                        torch.cuda.synchronize()
                        t0 = time.perf_counter()
                        arm.step(k)
                        torch.cuda.synchronize()
                        lat[kind][str(n)].append(1e3 * (time.perf_counter() - t0))
                    arm.check_status()
        rec["steps"] = {str(n): len(s) for n, s in sched.items()}
        rec["total_ms"] = {a: {n: {"median": float(np.median(v)), "min": min(v), "max": max(v), "runs": v} for n, v in d.items()}
                           for a, d in tot.items()}
        rec["step_latency"] = {a: {n: stats(v) for n, v in d.items()} for a, d in lat.items()}
        rec["voices_total_vs"] = {n: {a: rec["total_ms"][a][n]["median"] / rec["total_ms"]["voices"][n]["median"]
                                      for a in ARMS if a != "voices"} for n in map(str, PUSH)}
    print(json.dumps(rec, indent=1))
    with open(args.out, "w") as f:
        json.dump(rec, f, indent=1)
    assert all(all(d.values()) for d in rec["bit_identical"].values()), rec["bit_identical"]


if __name__ == "__main__":
    main()
