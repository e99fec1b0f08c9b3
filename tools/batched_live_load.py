"""Live-stream latency beside a batched long file (``BatchedInferencePipeline``), on one GPU.

Three cases over one engine context and one ``RoundScheduler`` (step-level rounds, as the backend runs it):

  (a) ``--streams`` live streams alone, in bench.py's streaming pattern: every stream's chunk arrives at its own
      uniformly drawn time inside a period sized so the offered load is ``--load`` x the batch throughput;
  (b) the same live streams plus one ``--file-seconds`` file through ``BatchedInferencePipeline(model,
      scheduler=...)``: its speech chunks are streams of the running decode loop (at most ``max_share`` of the
      indices, live requests first), joining it with their own logits rules;
  (c) the same live streams plus the same file through the one-shot ``BatchedInferencePipeline(model)`` beside the
      scheduler: one encode / generate call per group of ``--batch-size`` chunks.  One engine context runs one call at
      a time, so the scheduler's rounds wait while a group is decoded.

The file is ``--file-seconds`` of synthetic speech cut into 30 s chunks by ``clip_timestamps`` (no VAD model is
needed); its decode options are the pipeline's defaults at beam ``--file-beam`` (default: ``--beam``).  A file beam
narrower than the live streams' joins their decode loop with that width; each case reports how many times the decode
session was opened, which counts the drains a waiting chunk needs.  ``--equal-width-only`` restores the admission
rule before per-stream widths (a chunk joins with rules only at the session's own width), so one build gives both
arms of a before / after comparison.  Live cycles continue until the file has finished (at least
``--cycles``).  Reports the live p50 / p90 chunk latency of each case, the file's audio-s/s in (b) and (c), and the
card's name, power limit and SM clocks (maximum, and current at setup and after the last case), read in the same run.  Random weights and the synthetic tokenizer; needs a CUDA device.

    python tools/batched_live_load.py --model large-v3 --streams 16 --file-seconds 600 --batch-size 16
    python tools/batched_live_load.py --model large-v3 --streams 16 --file-seconds 600 --beam 5 --file-beam 1
"""
import argparse
import json
import os
import random
import sys
import threading
import time

ROOT = os.path.abspath(os.path.join(os.path.dirname(__file__), ".."))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))

from rest_load import _SerialSessions, card, live_cycles  # noqa: E402


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--model", default="large-v3")
    ap.add_argument("--streams", type=int, default=16, help="live streams")
    ap.add_argument("--load", type=float, default=0.6, help="offered live load as a fraction of the batch throughput")
    ap.add_argument("--file-seconds", type=float, default=600.0)
    ap.add_argument("--batch-size", type=int, default=16, help="the file's batch_size (one-shot: chunks per call)")
    ap.add_argument("--max-share", type=float, default=0.5, help="case (b): share of the decode indices the file may hold")
    ap.add_argument("--beam", type=int, default=5, help="beam of the live chunks")
    ap.add_argument("--file-beam", type=int, default=None, help="beam of the file (default: --beam)")
    ap.add_argument("--equal-width-only", action="store_true",
                    help="a chunk joins the open decode session with rules only at the session's own beam width (the "
                         "admission rule before per-stream widths): the 'before' arm of a comparison in one build")
    ap.add_argument("--cycles", type=int, default=3, help="live cycles per case, at least (more while the file runs)")
    ap.add_argument("--cases", default="abc")
    ap.add_argument("--out", default=None, help="also write the JSON result here")
    args = ap.parse_args()
    file_beam = args.beam if args.file_beam is None else args.file_beam

    import torch
    if not torch.cuda.is_available():
        raise SystemExit("batched_live_load.py needs a CUDA device")
    from bench import make_streams, tokens_for
    from whisperlive_b200 import synth
    from whisperlive_b200.config import dims_for
    from whisperlive_b200.engine import B200Whisper
    from whisperlive_b200.feature_extractor import FeatureExtractor
    from whisperlive_b200.scheduler import RoundScheduler
    from whisperlive_b200.tokenizer import build_synthetic_tokenizer
    from whisperlive_b200 import transcriber
    from whisperlive_b200.transcriber import B200WhisperModel, BatchedInferencePipeline
    from whisperlive_b200.weights import random_init

    if args.equal_width_only:
        fits = transcriber._rules_fit
        transcriber._rules_fit = lambda ds, skw: fits(ds, skw) and int(skw.get("beam_size", 5)) == int(ds.beam_size)
    dims = dims_for(args.model)
    n = args.streams
    cap = n + args.batch_size                   # the live streams and a whole one-shot group fit the decode capacity
    eng = B200Whisper(dims, random_init(dims, seed=0), max_streams=cap, max_beam=max(args.beam, file_beam, 5),
                      enc_slots=2 * cap + 2)
    model = B200WhisperModel(args.model, engine=eng, hf_tokenizer=build_synthetic_tokenizer(dims.vocab),
                             feature_extractor=FeatureExtractor(eng, dims.n_mels))
    durs, waves = make_streams(n)
    n_sot = 3 if dims.multilingual else 1
    kws = [dict(beam_size=args.beam, temperature=[0.0], log_prob_threshold=None, compression_ratio_threshold=None,
                no_speech_threshold=None, max_new_tokens=2 * tokens_for(d) - n_sot,
                language="en" if dims.multilingual else None, condition_on_previous_text=False, _single_window=True)
           for d in durs]
    sr = 16000
    audio = synth.speech_like(args.file_seconds, seed=777)
    n_chunks = int(args.file_seconds // 30)
    clips = [{"start": 30 * sr * i, "end": min(len(audio), 30 * sr * (i + 1))} for i in range(n_chunks)]
    file_kw = dict(language="en", vad_filter=False, clip_timestamps=clips, batch_size=args.batch_size, beam_size=file_beam)
    opens = [0]
    open_session = eng.open_decode_session

    def counted_open(*a, **k):
        opens[0] += 1
        return open_session(*a, **k)
    eng.open_decode_session = counted_open

    model.transcribe_batch(waves, kws)                       # warm-up, then the batch step the load is sized on
    t0 = time.perf_counter()
    model.transcribe_batch(waves, kws)
    batch_step = time.perf_counter() - t0
    period = batch_step / max(args.load, 1e-3)

    result = {"card": card(), "model": args.model, "live_streams": n, "offered_load": args.load,
              "arrival_period_ms": round(1000.0 * period, 1), "file_seconds": args.file_seconds, "file_chunks": n_chunks,
              "batch_size": args.batch_size, "max_share": args.max_share,
              "live_beam": args.beam, "file_beam": file_beam, "equal_width_only": args.equal_width_only, "decode_capacity": cap, "cases": {}}
    print("setup", json.dumps(result), flush=True)
    lock = threading.Lock()
    for case in args.cases:
        served = _SerialSessions(model, lock) if case == "c" else model
        sch = RoundScheduler(served, max_batch_size=cap, step_tokens=16)
        sch.start()
        up = {}
        opens_before = opens[0]
        try:
            live_cycles(sch, waves, kws, period, 1, lambda: True, random.Random(1))     # warm-up cycle
            thread = None
            if case != "a":
                def run_file(case=case, sch=sch):
                    t = time.perf_counter()
                    if case == "b":
                        pipe = BatchedInferencePipeline(model, scheduler=sch, max_share=args.max_share)
                        segments, _info = pipe.transcribe(audio, **file_kw)
                        up["segments"] = len(list(segments))
                    else:
                        # the one-shot pipeline decodes group by group as the generator is consumed: each group's calls
                        # hold the engine, as they would in a process that shares one context with the scheduler
                        pipe = BatchedInferencePipeline(model)
                        with lock:
                            segments, _info = pipe.transcribe(audio, **file_kw)
                        it, k = iter(segments), 0
                        while True:
                            with lock:
                                s = next(it, None)
                            if s is None:
                                break
                            k += 1
                        up["segments"] = k
                    up["chunk_steps"] = [x for g in pipe.group_steps for x in g]
                    up["seconds"] = time.perf_counter() - t
                thread = threading.Thread(target=run_file, daemon=True)
                thread.start()
            live = live_cycles(sch, waves, kws, period, args.cycles,
                               (lambda: not thread.is_alive()) if thread else (lambda: True), random.Random(4321))
            if thread is not None:
                thread.join()
                if "seconds" not in up:
                    raise RuntimeError(f"case {case}: the file failed")
                live["file_audio_s_per_s"] = round(args.file_seconds / up["seconds"], 1)
                live["file_segments"] = up["segments"]
                live["file_mean_chunk_steps"] = round(sum(up["chunk_steps"]) / max(1, len(up["chunk_steps"])), 1)
            live["admitted_mid_flight"] = sch.admitted_mid_flight
            live["rule_admissions"] = sch.rule_admissions
            live["session_opens"] = opens[0] - opens_before
        finally:
            sch.stop()
        result["cases"][case] = live
        print(case, json.dumps(live), flush=True)
    result["card_after"] = card()                 # the clock right after the last case
    line = json.dumps(result)
    print(line)
    if args.out:
        with open(args.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
