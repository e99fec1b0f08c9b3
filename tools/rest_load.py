"""Live-stream latency beside a REST upload, on one GPU.

Three cases over one engine context and one ``RoundScheduler`` (step-level rounds, as the backend runs it):

  (a) ``--streams`` live streams alone, in bench.py's streaming pattern: every stream's chunk arrives at its own
      uniformly drawn time inside a period sized so the offered load is ``--load`` x the batch throughput;
  (b) the same live streams plus one ``--upload-seconds`` upload through ``rest.ScheduledWhisperModel`` -- the model work
      of ``POST /v1/audio/transcriptions`` once ``rest.install`` has run: one scheduler request, decoded inside the
      running loop (the route's HTTP shell adds the response formatting only, and is not run here);
  (c) the same live streams plus the same upload through ``B200WhisperModel.transcribe`` called beside the scheduler,
      the one-shot call a per-request model makes.  One engine context runs one call at a time, so the scheduler's
      rounds wait while the call runs.

Live cycles continue until the upload has finished (at least ``--cycles``).  Reports the live p50 / p90 chunk latency
of each case, the upload's audio-s/s in (b) and (c), and the card's name and power limit, read in the same run.
Random weights and the synthetic tokenizer (no checkpoint is needed); needs a CUDA device.

    python tools/rest_load.py --model large-v3 --streams 16 --upload-seconds 600
"""
import argparse
import json
import os
import random
import subprocess
import sys
import threading
import time

ROOT = os.path.abspath(os.path.join(os.path.dirname(__file__), ".."))
sys.path.insert(0, ROOT)


def card():
    """The card's name, power limit, maximum SM clock and the SM clock at the moment of the call."""
    import torch
    name = torch.cuda.get_device_name(0)
    keys = ("power_limit", "sm_clock_max", "sm_clock")
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=power.limit,clocks.max.sm,clocks.sm", "--format=csv,noheader",
                              "-i", "0"], capture_output=True, text=True, timeout=30).stdout.strip()
        vals = [v.strip() for v in out.split(",")]
        if len(vals) != len(keys):
            raise ValueError(out)
    except Exception as e:          # the figures are reported as unknown rather than guessed
        vals = [f"unknown ({e})"] * len(keys)
    return {"name": name, **dict(zip(keys, vals))}


class _Req:
    """A live chunk with bench.py's options (one window, bounded decode)."""

    def __new__(cls, audio, kw):
        from whisperlive_b200.scheduler import BatchRequest

        class Req(BatchRequest):
            def kwargs(self_):
                return dict(kw)
        return Req(audio=audio)


class _SerialSessions:
    """``open_session`` of a model whose step rounds hold ``lock``: case (c)'s one-shot call and the scheduler's rounds
    take turns on the one engine context."""

    def __init__(self, model, lock):
        self.model, self.lock = model, lock

    def __getattr__(self, name):
        return getattr(self.model, name)

    def open_session(self):
        session, lock = self.model.open_session(), self.lock
        for name in ("add_streams", "step_round"):          # the two session calls that reach the engine here
            call = getattr(session, name)

            def locked(*a, _call=call, **k):
                with lock:
                    return _call(*a, **k)
            setattr(session, name, locked)
        return session


def live_cycles(sch, waves, kws, period, min_cycles, upload_done, rng):
    lat = []
    cyc = 0
    while cyc < min_cycles or not upload_done():
        t_start = time.monotonic()
        offs = sorted((rng.uniform(0.0, period), i) for i in range(len(waves)))
        batch = []
        for off, i in offs:
            dt = t_start + off - time.monotonic()
            if dt > 0:
                time.sleep(dt)
            r = _Req(waves[i], kws[i])
            sch.submit(r)
            batch.append(r)
        for r in batch:
            if not r.future.wait(600):
                raise RuntimeError("a live chunk was not answered within 600 s")
            if r.error is not None:
                raise r.error
        left = t_start + period - time.monotonic()
        if left > 0:
            time.sleep(left)
        lat += [1000.0 * (r.finished_at - r.submitted_at) for r in batch]
        cyc += 1
    lat.sort()
    q = lambda f: lat[min(len(lat) - 1, int(f * len(lat)))]
    return {"p50_chunk_latency_ms": round(q(0.5), 1), "p90_chunk_latency_ms": round(q(0.9), 1), "chunks": len(lat),
            "cycles": cyc}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--model", default="large-v3")
    ap.add_argument("--streams", type=int, default=16, help="live streams")
    ap.add_argument("--load", type=float, default=0.6, help="offered live load as a fraction of the batch throughput")
    ap.add_argument("--upload-seconds", type=float, default=600.0)
    ap.add_argument("--beam", type=int, default=5, help="beam of the live chunks (5: the route's default, so they share its loop)")
    ap.add_argument("--cycles", type=int, default=3, help="live cycles per case, at least (more while the upload runs)")
    ap.add_argument("--out", default=None, help="also write the JSON result here")
    args = ap.parse_args()

    import torch
    if not torch.cuda.is_available():
        raise SystemExit("rest_load.py needs a CUDA device")
    from bench import make_streams, tokens_for
    from whisperlive_b200 import synth
    from whisperlive_b200.config import dims_for
    from whisperlive_b200.engine import B200Whisper
    from whisperlive_b200.feature_extractor import FeatureExtractor
    from whisperlive_b200.rest import ScheduledWhisperModel
    from whisperlive_b200.scheduler import RoundScheduler
    from whisperlive_b200.tokenizer import build_synthetic_tokenizer
    from whisperlive_b200.transcriber import B200WhisperModel
    from whisperlive_b200.weights import random_init

    dims = dims_for(args.model)
    n = args.streams
    eng = B200Whisper(dims, random_init(dims, seed=0), max_streams=n + 1, max_beam=max(args.beam, 5),
                      enc_slots=2 * (n + 1) + 2)
    model = B200WhisperModel(args.model, engine=eng, hf_tokenizer=build_synthetic_tokenizer(dims.vocab),
                             feature_extractor=FeatureExtractor(eng, dims.n_mels))
    durs, waves = make_streams(n)
    n_sot = 3 if dims.multilingual else 1
    # the decode-session options (beam, suppression) stay at the defaults the route's upload uses, as a live
    # connection's do: streams with other options would wait for the loop to drain instead of sharing it
    kws = [dict(beam_size=args.beam, temperature=[0.0], log_prob_threshold=None, compression_ratio_threshold=None,
                no_speech_threshold=None, max_new_tokens=2 * tokens_for(d) - n_sot,
                language="en" if dims.multilingual else None, condition_on_previous_text=False, _single_window=True)
           for d in durs]
    upload = synth.speech_like(args.upload_seconds, seed=777)

    model.transcribe_batch(waves, kws)                       # warm-up, then the batch step the load is sized on
    t0 = time.perf_counter()
    model.transcribe_batch(waves, kws)
    batch_step = time.perf_counter() - t0
    period = batch_step / max(args.load, 1e-3)

    result = {"card": card(), "model": args.model, "live_streams": n, "offered_load": args.load,
              "arrival_period_ms": round(1000.0 * period, 1), "upload_seconds": args.upload_seconds, "cases": {}}
    lock = threading.Lock()
    for case in ("a", "b", "c"):
        served = _SerialSessions(model, lock) if case == "c" else model
        sch = RoundScheduler(served, max_batch_size=n + 1, step_tokens=16)
        sch.start()
        up = {}
        try:
            live_cycles(sch, waves, kws, period, 1, lambda: True, random.Random(1))     # warm-up cycle
            thread = None
            if case != "a":
                def run_upload(case=case, sch=sch):
                    t = time.perf_counter()
                    if case == "b":
                        segments, _info = ScheduledWhisperModel(args.model, scheduler=sch).transcribe(upload)
                        up["segments"] = len(list(segments))
                    else:
                        with lock:
                            segments, _info = model.transcribe(upload, temperature=0.0, vad_filter=False)
                        up["segments"] = len(list(segments))
                    up["seconds"] = time.perf_counter() - t
                thread = threading.Thread(target=run_upload, daemon=True)
                thread.start()
            live = live_cycles(sch, waves, kws, period, args.cycles,
                               (lambda: not thread.is_alive()) if thread else (lambda: True), random.Random(4321))
            if thread is not None:
                thread.join()
                if "seconds" not in up:
                    raise RuntimeError(f"case {case}: the upload failed")
                live["upload_audio_s_per_s"] = round(args.upload_seconds / up["seconds"], 1)
                live["upload_segments"] = up["segments"]
            live["admitted_mid_flight"] = sch.admitted_mid_flight
        finally:
            sch.stop()
        result["cases"][case] = live
        print(case, json.dumps(live), flush=True)
    line = json.dumps(result)
    print(line)
    if args.out:
        with open(args.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
