"""Interim-text latency of the decode session (run on an H100).

The staggered-arrival workload of bench.py's streaming phase: large-v3 (random-init weights), 32 streams, beam 4,
chunks U[5, 30] s, offered load 0.6 of the batch throughput, every chunk submitted at its own uniformly drawn time
inside the arrival period to RoundScheduler(step_tokens=16).  The batch throughput is measured first, the way bench.py
does: one transcribe_batch over all 32 chunks after a warm-up.

Cycles come in pairs, one with ``want_partials`` on and one with it off, in alternating order; both cycles of a pair
replay the same arrival times, so the two modes run the same workload (one warm-up pair first).  Reported:
  * with partials on: submit -> first interim (the first published ``partial``) and submit -> final, p50 / p90;
  * the mean scheduler round (step_round plus, when some request wants partials, the batched ``partials`` call) with
    and without peeking, and the mean ``partials`` call alone;
  * the card's name and power limit.  One JSON line on stdout.

    python tools/partial_latency.py [--cycles 2] [--load 0.6] [--out FILE]"""
import argparse
import json
import math
import os
import random
import sys
import time

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from tools.fallback_latency import card   # noqa: E402


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--model", default="large-v3")
    ap.add_argument("--streams", type=int, default=32)
    ap.add_argument("--beam", type=int, default=4)
    ap.add_argument("--load", type=float, default=0.6)
    ap.add_argument("--cycles", type=int, default=3, help="measured cycles per mode (after one warm-up pair)")
    ap.add_argument("--step-tokens", type=int, default=16)
    ap.add_argument("--out", default=None, help="also write the JSON line to this file")
    args = ap.parse_args()

    import torch
    if not torch.cuda.is_available():
        raise SystemExit("partial_latency.py: no CUDA device")
    from whisperlive_b200 import synth
    from whisperlive_b200.config import dims_for
    from whisperlive_b200.engine import B200Whisper
    from whisperlive_b200.feature_extractor import FeatureExtractor
    from whisperlive_b200.scheduler import BatchRequest, RoundScheduler
    from whisperlive_b200.tokenizer import build_synthetic_tokenizer
    from whisperlive_b200.transcriber import B200WhisperModel, TranscribeSession
    from whisperlive_b200.weights import random_init

    dims = dims_for(args.model)
    n = args.streams
    eng = B200Whisper(dims, random_init(dims, seed=0), max_streams=n, max_beam=max(args.beam, 1), enc_slots=2 * n + 2)
    model = B200WhisperModel(args.model, engine=eng, hf_tokenizer=build_synthetic_tokenizer(dims.vocab),
                             feature_extractor=FeatureExtractor(eng, dims.n_mels))
    durs = synth.chunk_durations(n, 5.0, 30.0, seed=1234)
    waves = [synth.speech_like(d, seed=1234 + i) for i, d in enumerate(durs)]
    n_sot = 3 if dims.multilingual else 1
    tokens_for = lambda d: int(math.ceil(3.2 * d)) + 8   # bench.py's decode length per chunk
    kws = [dict(beam_size=args.beam, temperature=[0.0], log_prob_threshold=None, compression_ratio_threshold=None,
                no_speech_threshold=None, suppress_tokens=[-1, eng.eot], suppress_blank=False,
                max_new_tokens=2 * tokens_for(d) - n_sot, language="en" if dims.multilingual else None,
                condition_on_previous_text=False, _single_window=True) for d in durs]

    # batch throughput -> arrival period (bench.py: period = batch step time / load)
    model.transcribe_batch(waves, kws)
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    model.transcribe_batch(waves, kws)
    torch.cuda.synchronize()
    batch_s = time.perf_counter() - t0
    period = batch_s / args.load

    rounds = {"on": [], "off": []}
    peeks = []
    mode = {"now": "off", "timing": False}
    step_round = TranscribeSession.step_round

    def timed_round(self, max_steps=16):
        t = time.perf_counter()
        step_round(self, max_steps)
        mode["t_round"] = time.perf_counter() - t
    TranscribeSession.step_round = timed_round

    class Sched(RoundScheduler):
        def _publish_partials(self, session, in_flight):
            t = time.perf_counter()
            super()._publish_partials(session, in_flight)
            dt = time.perf_counter() - t
            if mode["timing"] and "t_round" in mode:
                rounds[mode["now"]].append(mode.pop("t_round") + dt)
                if mode["now"] == "on":
                    peeks.append(dt)

    class Req(BatchRequest):
        def kwargs(self_):
            return self_.kw

    rng = random.Random(4321)
    sch = Sched(model, max_batch_size=n, step_tokens=args.step_tokens)
    sch.start()
    lat = {"first_interim": [], "final_on": [], "final_off": []}
    t_all = time.perf_counter()
    try:
        # one arrival draw per pair, used by both of its cycles: the two modes see the same workload (pair 0 warms up)
        plan = []
        for p in range(args.cycles + 1):
            arrivals = sorted((rng.uniform(0.0, period), i) for i in range(n))
            plan += [(m, arrivals, p > 0) for m in (("on", "off") if p % 2 == 0 else ("off", "on"))]
        for m, arrivals, timed in plan:
            mode["now"], mode["timing"] = m, timed
            t_start = time.monotonic()
            batch = []
            for off, i in arrivals:
                dt = t_start + off - time.monotonic()
                if dt > 0:
                    time.sleep(dt)
                r = Req(audio=waves[i], want_partials=(m == "on"))
                r.kw, r.t_interim = kws[i], None
                pub = r.partial.publish

                def rec(segs, r=r, pub=pub):
                    ok = pub(segs)
                    if ok and r.t_interim is None:
                        r.t_interim = time.monotonic()
                    return ok
                r.partial.publish = rec
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
            if timed:
                for r in batch:
                    lat["final_" + m].append(1000.0 * (r.finished_at - r.submitted_at))
                    if m == "on" and r.t_interim is not None:
                        lat["first_interim"].append(1000.0 * (r.t_interim - r.submitted_at))
    finally:
        sch.stop()
        TranscribeSession.step_round = step_round

    def stats(v):
        v = sorted(v)
        if not v:
            return None
        q = lambda f: round(v[min(len(v) - 1, int(f * len(v)))], 1)
        return {"p50_ms": q(0.5), "p90_ms": q(0.9), "n": len(v)}
    mean = lambda v: round(1000.0 * sum(v) / len(v), 3) if v else None
    line = {"tool": "partial_latency", "model": args.model, "streams": n, "beam": args.beam, "offered_load": args.load,
            "arrival_period_ms": round(1000.0 * period, 1), "batch_step_ms": round(1000.0 * batch_s, 1),
            "cycles_per_mode": args.cycles, "scheduler": f"RoundScheduler(step_tokens={args.step_tokens})",
            "partials_on": {"submit_to_first_interim": stats(lat["first_interim"]), "submit_to_final": stats(lat["final_on"]),
                            "chunks_with_interim": len(lat["first_interim"])},
            "partials_off": {"submit_to_final": stats(lat["final_off"])},
            "mean_round_ms": {"peeking": mean(rounds["on"]), "not_peeking": mean(rounds["off"]),
                              "rounds": [len(rounds["on"]), len(rounds["off"])]},
            "mean_partials_call_ms": mean(peeks), "wall_s": round(time.perf_counter() - t_all, 1), **card()}
    print(json.dumps(line), flush=True)
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "a") as f:
            f.write(json.dumps(line) + "\n")


if __name__ == "__main__":
    main()
