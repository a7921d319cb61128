"""Vocoding 16 voices x 4 utterances (the seeded lengths of scripts/ragged_time.py: 64 utterances uniform in [86, 861] mel
frames, 1 to 10 s at 22.05 kHz; utterance i belongs to voice i // 4) three ways, each voice a Generator of its own seed:
  voices   one models.generate_voices(generators, mel [64, 80, T_max], voice, lengths) call
  serial   16 calls of generators[v].generate(mel_v, lengths_v), one after another on one stream
  streams  the same 16 calls spread round-robin over 4 CUDA streams (each voice's module keeps one workspace per stream)
at fp32 and at bf16.  Device time per pass (CUDA events on the caller's stream around the whole pass, the side streams
joined back into it), median of REPS passes with the six arms alternated, min / max for the spread.  Every arm's audio
must be bit-identical to the serial arm's at the same precision.  Writes a JSON record with the card's name and power
limit (default profiles/h100_voices.json)."""
import argparse
import json
import subprocess
import sys

import numpy as np
import torch

sys.path.insert(0, ".")
from melgan_multi_b200 import models, synth

V, PER, LO, HI, SEED, REPS, NSTREAMS = 16, 4, 86, 861, 2024, 5, 4


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True).stdout.strip().splitlines()
    return q[torch.cuda.current_device()] if q else "unknown"


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default="profiles/h100_voices.json")
    args = ap.parse_args()
    gens = []
    for v in range(V):
        g = models.Generator()
        g.load_state_dict({k: torch.from_numpy(a) for k, a in synth.generator_state(1000 + v).items()})
        gens.append(g.cuda().eval())
    B = V * PER
    lens = [int(v) for v in np.random.default_rng(SEED).integers(LO, HI + 1, B)]
    voice = [i // PER for i in range(B)]
    T = max(lens)
    mel = torch.zeros(B, 80, T, device="cuda")
    for i, L in enumerate(lens):
        mel[i, :, :L] = torch.from_numpy(synth.mel_input(1, L, SEED + i)[0])
    parts = [(mel[v * PER:(v + 1) * PER, :, :max(lens[v * PER:(v + 1) * PER])].contiguous(), lens[v * PER:(v + 1) * PER])
             for v in range(V)]
    streams = [torch.cuda.Stream() for _ in range(NSTREAMS)]

    def one_call(prec):
        return lambda: models.generate_voices(gens, mel, voice, lens, precision=prec)

    def serial(prec):
        return lambda: [gens[v].generate(x, l, precision=prec) for v, (x, l) in enumerate(parts)]

    def spread(prec):
        def run():
            cur = torch.cuda.current_stream()
            out = []
            for s in streams:
                s.wait_stream(cur)
            for v, (x, l) in enumerate(parts):
                with torch.cuda.stream(streams[v % NSTREAMS]):
                    y = gens[v].generate(x, l, precision=prec)
                    y.record_stream(cur)
                    out.append(y)
            for s in streams:
                cur.wait_stream(s)
            return out
        return run

    arms = {}
    for prec in ("fp32", "bf16"):
        arms["voices_" + prec], arms["serial_" + prec], arms["streams_" + prec] = one_call(prec), serial(prec), spread(prec)
    with torch.no_grad():
        for f in arms.values():  # warm every shape, workspace and stream
            f()
        torch.cuda.synchronize()
        ms = {k: [] for k in arms}
        for _ in range(REPS):
            for k, f in arms.items():
                a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                a.record()
                f()
                b.record()
                torch.cuda.synchronize()
                ms[k].append(a.elapsed_time(b))
        identical = {}
        for prec in ("fp32", "bf16"):
            ref = arms["serial_" + prec]()
            one = arms["voices_" + prec]()
            spr = arms["streams_" + prec]()
            torch.cuda.synchronize()
            ok_one = all(torch.equal(one[v * PER + j, :, :256 * L], ref[v][j, :, :256 * L])
                         for v in range(V) for j, L in enumerate(parts[v][1]))
            ok_spr = all(torch.equal(a, b) for a, b in zip(spr, ref))
            identical[prec] = {"voices_vs_serial": ok_one, "streams_vs_serial": ok_spr}
        gens[0]._dev.check_status(B, T)
    stat = {k: {"median_ms": float(np.median(v)), "min_ms": float(min(v)), "max_ms": float(max(v)), "runs_ms": v}
            for k, v in ms.items()}
    rec = {
        "card": card(),
        "workload": {"voices": V, "utterances_per_voice": PER, "frames": sum(lens), "T_max": T,
                     "lengths_uniform_in": [LO, HI], "seed": SEED, "voice_seeds": [1000, 1000 + V - 1],
                     "audio_seconds": sum(lens) * 256 / 22050.0, "streams_arm_streams": NSTREAMS, "passes": REPS},
        "timing": stat,
        "speedup_voices_vs": {prec: {other: stat["%s_%s" % (other, prec)]["median_ms"] / stat["voices_" + prec]["median_ms"]
                                     for other in ("serial", "streams")} for prec in ("fp32", "bf16")},
        "bit_identical": identical,
    }
    print(json.dumps(rec, indent=1))
    with open(args.out, "w") as f:
        json.dump(rec, f, indent=1)
    assert all(all(d.values()) for d in identical.values()), identical


if __name__ == "__main__":
    main()
