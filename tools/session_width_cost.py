"""Token-step cost of the rows a narrow stream leaves inactive in a wider decode session.

``--chunks`` greedy (beam 1) streams -- large-v3-shaped random weights, 30 s of synthetic speech each, EOT suppressed so
every stream runs every step -- decode in two decode sessions of the same capacity:

  beam-5 session: each stream joins with its own width 1 (``rules=[{"beam_size": 1}]``) and leaves 4 of its 5 rows
                  inactive; the decode GEMMs still carry all 5 rows per index;
  beam-1 session: the same streams at the session's own width, one row per index.

Each run is ``--steps`` token steps (``break_on_finish`` off); the step time is the run's device time
(``last_device_ms(2)``, CUDA events around the graph launch) over the steps it ran.  The two sessions alternate
``--repeats`` times after a warm-up of each.  Reads the card's name, power limit and SM clocks (maximum, and current
right after the timed runs) in the same run.

    python tools/session_width_cost.py --model large-v3 --chunks 16 --steps 64
"""
import argparse
import json
import os
import statistics
import sys

import numpy as np

ROOT = os.path.abspath(os.path.join(os.path.dirname(__file__), ".."))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))

from rest_load import card  # noqa: E402


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--model", default="large-v3")
    ap.add_argument("--chunks", type=int, default=16)
    ap.add_argument("--steps", type=int, default=64)
    ap.add_argument("--repeats", type=int, default=5)
    ap.add_argument("--out", default=None, help="also write the JSON result here")
    args = ap.parse_args()

    import torch
    if not torch.cuda.is_available():
        raise SystemExit("session_width_cost.py needs a CUDA device")
    from whisperlive_b200 import synth
    from whisperlive_b200.config import dims_for
    from whisperlive_b200.engine import B200Whisper
    from whisperlive_b200.weights import random_init

    dims = dims_for(args.model)
    n = args.chunks
    eng = B200Whisper(dims, random_init(dims, seed=0), max_streams=n, max_beam=5, enc_slots=n + 2)
    waves = [synth.speech_like(30.0, seed=777 + i) for i in range(n)]
    enc = eng.encode(np.stack([f[:, :3000] for f in eng.mel(waves)]))
    views = [enc.select([i]) for i in range(n)]
    sot = [eng.sot] if not dims.multilingual else [eng.sot, eng.sot + 1, eng.sot + 1 + dims.num_languages + 1]
    opts = dict(suppress_tokens=[eng.eot], suppress_blank=False)
    steps = min(args.steps, 440)

    def step_ms(session_beam):
        sess = eng.open_decode_session(capacity=n, beam_size=session_beam, num_hypotheses=1, **opts)
        rules = [dict(opts, beam_size=1)] * n if session_beam != 1 else None
        sess.admit(views, [sot] * n, [448] * n, rules=rules)
        sess.run(max_steps=steps, break_on_finish=False)
        ran = sess.last_steps
        ms = eng.last_device_ms(2)
        sess.close()
        assert ran == steps, (session_beam, ran)
        return ms / ran

    step_ms(5), step_ms(1)                         # warm-up: graph capture of each session shape
    t5, t1 = [], []
    for _ in range(args.repeats):
        t5.append(step_ms(5))
        t1.append(step_ms(1))
    result = {"card": card(), "model": args.model, "streams": n, "steps_per_run": steps, "repeats": args.repeats,
              "beam5_session_ms_per_step": [round(x, 3) for x in t5], "beam1_session_ms_per_step": [round(x, 3) for x in t1],
              "median_ratio": round(statistics.median(t5) / statistics.median(t1), 3)}
    line = json.dumps(result)
    print(line)
    if args.out:
        with open(args.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
