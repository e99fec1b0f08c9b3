"""Model load time: ``B200Whisper.from_model(dir)`` to ready for large-v3-shaped random weights written in each
checkpoint layout, through the typed upload (bytes as stored, converted on the device) and through the fp32 upload of
the same reader (``weights.load_model_dir`` -> fp32 dict -> ``wl_load_tensor``) in the same call.  Each load runs in a
fresh process started by a parent that never holds the weights, so its peak host RSS (mapped file pages included) is
its own; the files were just written, so they are read from the page cache (warm).  Bytes to the device are the
payload handed to the library.  One run per figure.  Reads the card's name and power limit.
    python tools/load_time.py --layouts safetensors:float16 safetensors-sharded:bfloat16 bin:float32 ct2:int8_float16"""
import argparse
import json
import os
import shutil
import subprocess
import sys
import tempfile
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def _peak_rss() -> int:
    """This process's peak resident set.  ru_maxrss survives fork and exec, so the parent that starts the loads never
    holds the weights itself: a separate process writes each checkpoint."""
    import resource
    return resource.getrusage(resource.RUSAGE_SELF).ru_maxrss * 1024


def write(path: str, spec: str, model: str) -> None:
    from tests.checkpoint_layouts import write_ct2, write_hf
    from whisperlive_b200.config import dims_for
    from whisperlive_b200.weights import random_init
    fmt, dtype = spec.split(":")
    w = random_init(dims_for(model), seed=0)
    write_ct2(w, path, dtype) if fmt == "ct2" else write_hf(w, path, fmt, dtype, n_shards=4)
    with open(os.path.join(path, "config.json"), "w") as f:
        json.dump({}, f)


def one(path: str, mode: str, model: str) -> dict:
    """Load ``path`` once with ``mode`` (typed | fp32) and report the figures (runs in its own process)."""
    import torch
    from whisperlive_b200 import weights as W
    from whisperlive_b200.engine import B200Whisper
    t0 = time.perf_counter()
    if mode == "typed":
        eng = B200Whisper.from_model(path, max_streams=8, max_beam=5)
    else:
        w = W.load_model_dir(path)
        eng = B200Whisper(W.infer_dims(w, model), w, max_streams=8, max_beam=5)
    torch.cuda.synchronize()
    dt = time.perf_counter() - t0
    rss = _peak_rss()
    if mode == "typed":   # counted after the figures above: the count is not part of the load
        sent = sum(a.nbytes + (0 if s is None else s.nbytes) for _, a, s in W.open_checkpoint(path).tensors())
    else:
        sent = sum(v.numel() * 4 for v in w.values())
    return {"seconds": round(dt, 2), "peak_rss_gb": round(rss / 1e9, 2), "bytes_to_device_gb": round(sent / 1e9, 2),
            "device_bytes_gb": round(eng.device_bytes / 1e9, 2)}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--model", default="large-v3")
    ap.add_argument("--layouts", nargs="+",
                    default=["safetensors:float16", "safetensors-sharded:bfloat16", "bin:float32", "ct2:int8_float16"])
    ap.add_argument("--one", nargs=2, metavar=("DIR", "MODE"))
    ap.add_argument("--write", nargs=2, metavar=("DIR", "LAYOUT"))
    ap.add_argument("--dir", default=None, help="where the checkpoints are written (default: a temporary directory)")
    a = ap.parse_args()
    if a.one:
        print(json.dumps(one(a.one[0], a.one[1], a.model)), flush=True)
        return
    if a.write:
        write(a.write[0], a.write[1], a.model)
        return
    card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                          text=True).stdout.strip().splitlines()
    print(f"card: {card[0] if card else 'unknown'}", flush=True)
    base = tempfile.mkdtemp(dir=a.dir)
    try:
        for spec in a.layouts:
            p = os.path.join(base, spec.replace(":", "-"))
            t0 = time.perf_counter()
            subprocess.run([sys.executable, os.path.abspath(__file__), "--model", a.model, "--write", p, spec], check=True)
            size = sum(os.path.getsize(os.path.join(p, f)) for f in os.listdir(p))
            print(f"{spec}: written {size / 1e9:.2f} GB in {time.perf_counter() - t0:.1f} s", flush=True)
            for mode in ("typed", "fp32"):
                r = subprocess.run([sys.executable, os.path.abspath(__file__), "--model", a.model, "--one", p, mode],
                                   capture_output=True, text=True)
                if r.returncode != 0:
                    print(f"{spec} {mode}: failed\n{r.stderr[-2000:]}", flush=True)
                    continue
                print(json.dumps({"layout": spec, "path": mode, **json.loads(r.stdout.strip().splitlines()[-1])}),
                      flush=True)
            shutil.rmtree(p)
    finally:
        shutil.rmtree(base, ignore_errors=True)


if __name__ == "__main__":
    main()
