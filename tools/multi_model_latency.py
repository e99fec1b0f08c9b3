"""Chunk latency of two models served side by side on one GPU (run on an H100).

Two models (default large-v3 and small.en, random-init weights, synthetic tokenizer) are resident in one process, each
with its own engine context and its own RoundScheduler(step_tokens=16) -- what the backend plugin's model registry runs
with ``single_model=False``.  Each model gets partial_latency.py's staggered workload: N streams (default 16), chunks
U[5, 30] s, offered load 0.6 of that model's own batch throughput (one transcribe_batch over its N chunks after a
warm-up), every chunk submitted at its own uniformly drawn time inside the arrival period.

A round runs three cycles in rotating order, all replaying the same arrival times:
  * the first model alone (the second resident and idle), * the second model alone, * both at once.
One warm-up round first.  Reported per model: submit -> final p50 / p90 alone and with both models decoding, plus the
card's name and power limit.  One JSON line on stdout.

    python tools/multi_model_latency.py [--models large-v3,small.en] [--streams 16] [--cycles 2] [--out FILE]"""
import argparse
import json
import math
import os
import random
import sys
import threading
import time

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from tools.fallback_latency import card   # noqa: E402


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--models", default="large-v3,small.en")
    ap.add_argument("--streams", type=int, default=16)
    ap.add_argument("--beam", type=int, default=4)
    ap.add_argument("--load", type=float, default=0.6)
    ap.add_argument("--cycles", type=int, default=2, help="measured rounds of the three configurations (after one warm-up)")
    ap.add_argument("--step-tokens", type=int, default=16)
    ap.add_argument("--out", default=None, help="also write the JSON line to this file")
    args = ap.parse_args()

    import torch
    if not torch.cuda.is_available():
        raise SystemExit("multi_model_latency.py: no CUDA device")
    from whisperlive_b200 import synth
    from whisperlive_b200.config import dims_for
    from whisperlive_b200.engine import B200Whisper
    from whisperlive_b200.feature_extractor import FeatureExtractor
    from whisperlive_b200.scheduler import BatchRequest, RoundScheduler
    from whisperlive_b200.tokenizer import build_synthetic_tokenizer
    from whisperlive_b200.transcriber import B200WhisperModel
    from whisperlive_b200.weights import random_init

    class Req(BatchRequest):
        def kwargs(self_):
            return self_.kw

    n = args.streams
    names = [m.strip() for m in args.models.split(",") if m.strip()]
    if len(names) != 2:
        raise SystemExit("--models takes two model names")
    served = []
    for k, name in enumerate(names):
        dims = dims_for(name)
        eng = B200Whisper(dims, random_init(dims, seed=k), max_streams=n, max_beam=max(args.beam, 1), enc_slots=2 * n + 2)
        model = B200WhisperModel(name, engine=eng, hf_tokenizer=build_synthetic_tokenizer(dims.vocab),
                                 feature_extractor=FeatureExtractor(eng, dims.n_mels))
        durs = synth.chunk_durations(n, 5.0, 30.0, seed=1234 + 100 * k)
        waves = [synth.speech_like(d, seed=1234 + 100 * k + i) for i, d in enumerate(durs)]
        n_sot = 3 if dims.multilingual else 1
        tokens_for = lambda d: int(math.ceil(3.2 * d)) + 8   # bench.py's decode length per chunk
        kws = [dict(beam_size=args.beam, temperature=[0.0], log_prob_threshold=None, compression_ratio_threshold=None,
                    no_speech_threshold=None, suppress_tokens=[-1, eng.eot], suppress_blank=False,
                    max_new_tokens=2 * tokens_for(d) - n_sot, language="en" if dims.multilingual else None,
                    condition_on_previous_text=False, _single_window=True) for d in durs]
        model.transcribe_batch(waves, kws)
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        model.transcribe_batch(waves, kws)
        torch.cuda.synchronize()
        batch_s = time.perf_counter() - t0
        sch = RoundScheduler(model, max_batch_size=n, step_tokens=args.step_tokens)
        served.append(dict(name=name, model=model, waves=waves, kws=kws, batch_s=batch_s, period=batch_s / args.load,
                           sch=sch, device_bytes=eng.device_bytes))

    def drive(s, arrivals, out):
        """submit s's chunks at their arrival offsets, wait for all, keep the latencies"""
        t_start = time.monotonic()
        batch = []
        for off, i in arrivals:
            dt = t_start + off - time.monotonic()
            if dt > 0:
                time.sleep(dt)
            r = Req(audio=s["waves"][i])
            r.kw = s["kws"][i]
            s["sch"].submit(r)
            batch.append(r)
        for r in batch:
            if not r.future.wait(600):
                raise RuntimeError("a chunk was not answered within 600 s")
            if r.error is not None:
                raise r.error
        left = t_start + s["period"] - time.monotonic()
        if left > 0:
            time.sleep(left)
        out.extend(1000.0 * (r.finished_at - r.submitted_at) for r in batch)

    lat = {(k, mode): [] for k in range(2) for mode in ("alone", "both")}
    rng = random.Random(4321)
    configs = [("alone", [0]), ("alone", [1]), ("both", [0, 1])]
    t_all = time.perf_counter()
    for s in served:
        s["sch"].start()
    try:
        for rnd in range(args.cycles + 1):
            arrivals = [sorted((rng.uniform(0.0, s["period"]), i) for i in range(n)) for s in served]
            order = configs[rnd % 3:] + configs[:rnd % 3]
            for mode, which in order:
                sink = {k: [] for k in which}
                threads = [threading.Thread(target=drive, args=(served[k], arrivals[k], sink[k])) for k in which]
                for t in threads:
                    t.start()
                for t in threads:
                    t.join()
                if rnd > 0:
                    for k in which:
                        lat[(k, mode)] += sink[k]
    finally:
        for s in served:
            s["sch"].stop()

    def stats(v):
        v = sorted(v)
        if not v:
            return None
        q = lambda f: round(v[min(len(v) - 1, int(f * len(v)))], 1)
        return {"p50_ms": q(0.5), "p90_ms": q(0.9), "n": len(v)}
    line = {"tool": "multi_model_latency", "streams_per_model": n, "beam": args.beam, "offered_load": args.load,
            "cycles": args.cycles, "scheduler": f"RoundScheduler(step_tokens={args.step_tokens}) per model",
            "models": [{"model": s["name"], "batch_step_ms": round(1000.0 * s["batch_s"], 1),
                        "arrival_period_ms": round(1000.0 * s["period"], 1), "device_bytes": s["device_bytes"],
                        "submit_to_final_alone": stats(lat[(k, "alone")]),
                        "submit_to_final_both": stats(lat[(k, "both")])} for k, s in enumerate(served)],
            "wall_s": round(time.perf_counter() - t_all, 1), **card()}
    print(json.dumps(line), flush=True)
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "a") as f:
            f.write(json.dumps(line) + "\n")


if __name__ == "__main__":
    main()
