"""Time of wl_mt_translate (device translation) at the SMaLL-100 shape on random weights: 1 / 8 / 32 segments of 16 and
48 source tokens, beam 5, max_length 64.  Prints one line per shape: the host time of the whole call (upload, encoder,
the captured token loop, download; the call ends in a device synchronise), the decoder positions of the longest output
and the call time per such position.  With random weights a segment seldom ends on EOS, so most calls run to max_length.
When transformers is importable, it also times Hugging Face fp32 ``generate`` one segment at a time on the same card
(the reference's library call, not the reference server).  The card name and power limit are read in the same run.

    python tools/translate_time.py [--iters 5] [--out translate_time.json]"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

sys.path.insert(0, os.path.abspath(os.path.join(os.path.dirname(__file__), "..")))

from whisperlive_b200 import translation as T  # noqa: E402


def card() -> str:
    try:
        return subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                              capture_output=True, text=True, timeout=30).stdout.strip().splitlines()[0]
    except Exception as e:
        return f"unknown ({e})"


def hf_generate_ms(cfg, ck, gen, srcs, iters):
    try:
        import torch
        from transformers import M2M100Config, M2M100ForConditionalGeneration
    except Exception as e:
        return f"not measured (transformers unavailable: {e.__class__.__name__})"
    hc = M2M100Config(vocab_size=cfg.vocab, d_model=cfg.d_model, encoder_layers=cfg.enc_layers, decoder_layers=cfg.dec_layers,
                      encoder_attention_heads=cfg.n_heads, decoder_attention_heads=cfg.n_heads, encoder_ffn_dim=cfg.ffn,
                      decoder_ffn_dim=cfg.ffn, max_position_embeddings=cfg.max_positions, scale_embedding=cfg.scale_embedding)
    m = M2M100ForConditionalGeneration(hc).eval()
    sd = {k: torch.from_numpy(v) for k, v in ck.items()}
    m.load_state_dict(sd, strict=False)
    m.tie_weights()
    m = m.cuda()
    kw = dict(num_beams=gen.num_beams, max_length=gen.max_length, early_stopping=gen.early_stopping, length_penalty=gen.length_penalty,
              decoder_start_token_id=gen.decoder_start_token_id, eos_token_id=gen.eos_token_id, pad_token_id=gen.pad_token_id)
    times = []
    with torch.no_grad():
        for _ in range(iters + 1):
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            for s in srcs:
                m.generate(input_ids=torch.tensor([s], device="cuda"), **kw)
            torch.cuda.synchronize()
            times.append((time.perf_counter() - t0) * 1e3)
    return float(np.median(times[1:]))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=5)
    ap.add_argument("--out", default="")
    ap.add_argument("--hf", action="store_true", help="also time Hugging Face generate (one segment at a time)")
    a = ap.parse_args()
    cfg = T.MtConfig(**T.SMALL100_SHAPE)
    ck = T.random_checkpoint(cfg, seed=0)
    gen = T.GenSettings(num_beams=5, max_length=64)
    tr = T.DeviceTranslator(cfg, gen, ck, capacity=32, max_src_tokens=32 * 48)
    print("card:", card())
    print("device bytes:", tr.device_bytes())
    print(f"{'B':>3} {'src':>4} {'call ms':>9} {'positions':>9} {'ms/position':>11}")
    rows = []
    rng = np.random.default_rng(1)
    for n in (16, 48):
        for B in (1, 8, 32):
            srcs = [[128020] + rng.integers(3, 128000, n - 2).tolist() + [2] for _ in range(B)]
            tr.translate_ids(srcs)
            times = []
            for _ in range(a.iters):
                t0 = time.perf_counter()
                ids, _ = tr.translate_ids(srcs)
                times.append((time.perf_counter() - t0) * 1e3)
            ms = float(np.median(times))
            pos = max(len(x) for x in ids)
            rows.append(dict(B=B, src_tokens=n, call_ms=ms, positions=pos, ms_per_position=ms / max(pos, 1)))
            print(f"{B:>3} {n:>4} {ms:>9.2f} {pos:>9d} {ms / max(pos, 1):>11.3f}")
    hf = None
    if a.hf:
        srcs = [[128020] + rng.integers(3, 128000, 14).tolist() + [2] for _ in range(8)]
        hf = hf_generate_ms(cfg, ck, gen, srcs, 2)
        print("Hugging Face fp32 generate, 8 segments of 16 tokens one at a time (ms):", hf)
    tr.close()
    if a.out:
        os.makedirs(os.path.dirname(a.out) or ".", exist_ok=True)
        with open(a.out, "w") as fh:
            json.dump(dict(card=card(), rows=rows, hf_generate_8x16_ms=hf), fh, indent=1)


if __name__ == "__main__":
    main()
