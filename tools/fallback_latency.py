"""Chunk latency when some streams climb the temperature-fallback ladder (run on an H100).

large-v3 (random-init weights), max_streams=32, beam 5, best_of 5.  Every cycle, each of the 32 streams submits one
chunk at its own uniformly drawn time inside the arrival period to the product's scheduler, RoundScheduler(step_tokens=16),
as bench.py's streaming phase does.  A chosen fraction of the streams is forced through the whole ladder 0.0 ... 1.0
(log_prob_threshold=0.0: no window's average log-probability reaches it); the rest decode with temperature=[0.0].
Reports p50 / p90 / max chunk latency (submit -> segments) of the beam-only streams and of all streams, the number of
one-shot sampling ``generate`` calls, and the card's name and power limit.  One JSON line on stdout.

    python tools/fallback_latency.py [--fallback-frac 0.25] [--cycles 3] [--period-ms 3000] [--root DIR]

--root imports the package from another checkout (built in place), so two builds can be compared in one session."""
import argparse
import json
import os
import random
import subprocess
import sys
import time


def card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                             text=True, timeout=30).stdout.strip().splitlines()[0]
        name, limit = (s.strip() for s in out.split(","))
        return {"gpu": name, "power_limit": limit}
    except Exception as ex:     # the numbers are still reported; the card is then unknown
        return {"gpu": None, "power_limit": None, "card_error": str(ex)}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--root", default=os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
    ap.add_argument("--model", default="large-v3")
    ap.add_argument("--streams", type=int, default=32)
    ap.add_argument("--fallback-frac", type=float, default=0.25)
    ap.add_argument("--cycles", type=int, default=3, help="measured cycles (one more warm-up cycle runs first)")
    ap.add_argument("--period-ms", type=float, default=3000.0, help="arrival period: every stream submits one chunk per period")
    ap.add_argument("--step-tokens", type=int, default=16)
    ap.add_argument("--out", default=None, help="also write the JSON line to this file")
    args = ap.parse_args()
    sys.path.insert(0, os.path.abspath(args.root))

    import torch
    if not torch.cuda.is_available():
        raise SystemExit("fallback_latency.py: no CUDA device")
    from whisperlive_b200 import synth
    from whisperlive_b200.config import dims_for
    from whisperlive_b200.engine import B200Whisper
    from whisperlive_b200.feature_extractor import FeatureExtractor
    from whisperlive_b200.scheduler import BatchRequest, RoundScheduler
    from whisperlive_b200.tokenizer import build_synthetic_tokenizer
    from whisperlive_b200.transcriber import B200WhisperModel
    from whisperlive_b200.weights import random_init

    dims = dims_for(args.model)
    n = args.streams
    eng = B200Whisper(dims, random_init(dims, seed=0), max_streams=n, max_beam=5, enc_slots=2 * n + 2)
    model = B200WhisperModel(args.model, engine=eng, hf_tokenizer=build_synthetic_tokenizer(dims.vocab),
                             feature_extractor=FeatureExtractor(eng, dims.n_mels))
    sampling_calls = [0]
    generate = eng.generate

    def counted(*a, **kw):
        if kw.get("beam_size", 5) == 1 and kw.get("sampling_topk", 1) != 1 and kw.get("sampling_temperature", 0) > 0:
            sampling_calls[0] += 1
        return generate(*a, **kw)
    eng.generate = counted

    durs = synth.chunk_durations(n, 5.0, 30.0, seed=1234)
    waves = [synth.speech_like(d, seed=1234 + i) for i, d in enumerate(durs)]
    n_fb = int(round(args.fallback_frac * n))
    fallback = set(random.Random(99).sample(range(n), n_fb))
    common = dict(beam_size=5, best_of=5, compression_ratio_threshold=None, no_speech_threshold=None,
                  suppress_tokens=[-1, eng.eot], suppress_blank=False, condition_on_previous_text=False,
                  language="en" if dims.multilingual else None, _single_window=True)
    kws = [dict(common, max_new_tokens=int(3.2 * d) + 8,
                **(dict(temperature=[0.0, 0.2, 0.4, 0.6, 0.8, 1.0], log_prob_threshold=0.0) if i in fallback
                   else dict(temperature=[0.0], log_prob_threshold=None)))
           for i, d in enumerate(durs)]

    class Req(BatchRequest):
        def kwargs(self_):
            return self_.kw

    period = args.period_ms / 1000.0
    rng = random.Random(4321)
    sch = RoundScheduler(model, max_batch_size=n, step_tokens=args.step_tokens)
    sch.start()
    lat = {"beam": [], "all": []}
    t0 = time.perf_counter()
    try:
        for cyc in range(args.cycles + 1):          # cycle 0 warms up (graph captures, first launches)
            if cyc == 1:
                sampling_calls[0] = 0
            t_start = time.monotonic()
            batch = []
            for off, i in sorted((rng.uniform(0.0, period), i) for i in range(n)):
                dt = t_start + off - time.monotonic()
                if dt > 0:
                    time.sleep(dt)
                r = Req(audio=waves[i])
                r.kw, r.stream = kws[i], i
                sch.submit(r)
                batch.append(r)
            for r in batch:
                if not r.future.wait(600):
                    raise RuntimeError("a chunk was not answered within 600 s")
                if r.error is not None:
                    raise r.error
            left = t_start + period - time.monotonic()
            if left > 0:
                time.sleep(left)
            if cyc > 0:
                for r in batch:
                    ms = 1000.0 * (r.finished_at - r.submitted_at)
                    lat["all"].append(ms)
                    if r.stream not in fallback:
                        lat["beam"].append(ms)
    finally:
        sch.stop()

    def stats(v):
        v = sorted(v)
        if not v:
            return None
        q = lambda f: round(v[min(len(v) - 1, int(f * len(v)))], 1)
        return {"p50_ms": q(0.5), "p90_ms": q(0.9), "max_ms": round(v[-1], 1), "chunks": len(v)}
    line = {"tool": "fallback_latency", "root": os.path.abspath(args.root), "model": args.model, "streams": n,
            "fallback_streams": n_fb, "cycles": args.cycles, "arrival_period_ms": args.period_ms,
            "scheduler": f"RoundScheduler(step_tokens={args.step_tokens})", "beam_only": stats(lat["beam"]),
            "all": stats(lat["all"]), "one_shot_sampling_generate_calls": sampling_calls[0],
            "wall_s": round(time.perf_counter() - t0, 1), **card()}
    print(json.dumps(line), flush=True)
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "a") as f:
            f.write(json.dumps(line) + "\n")


if __name__ == "__main__":
    main()
