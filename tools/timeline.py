#!/usr/bin/env python
"""Per-kernel cost INSIDE the replayed decode-step graph, from the WLB200_TIMELINE dump (csrc/common.cuh).

    WLB200_TIMELINE=/tmp/tl.bin python tools/profile_step.py ...   (timeline build, on the GPU)
    python tools/timeline.py /tmp/tl.bin

Every kernel stamps %globaltimer when block 0 starts (what=0) and right after its dependency wait (what=1).
interval(k) = ready(k+1) - ready(k) is kernel k's dependent work + its boundary; entry->ready is how long the
kernel was resident ahead of its data (PDL overlap)."""
import sys
from collections import defaultdict

import numpy as np

NAMES = {1: "decoder_embed", 2: "layernorm_update", 3: "gemm split-K", 4: "self_attn", 5: "cross_attn", 6: "cross_combine",
         7: "gelu_cast", 8: "search_rows", 9: "search_streams", 10: "gemm vocab", 11: "dstep"}


def main(path):
    raw = np.fromfile(path, dtype=np.uint64)
    t = (raw >> np.uint64(8)).astype(np.int64)
    kid = ((raw >> np.uint64(2)) & np.uint64(63)).astype(int)
    what = (raw & np.uint64(3)).astype(int)
    order = np.argsort(t, kind="stable")
    t, kid, what = t[order], kid[order], what[order]
    ready = [(tt, k) for tt, k, w in zip(t, kid, what) if w == 1]
    print(f"{len(raw)} stamps, {len(ready)} kernels, span {(t[-1] - t[0]) / 1e3:.1f} us")
    # split GEMM kinds by their position in the layer sequence (the kernel after it tells which one it was)
    iv = defaultdict(list)
    for i in range(len(ready) - 1):
        (t0, k0), (t1, k1) = ready[i], ready[i + 1]
        name = NAMES.get(k0, str(k0))
        if k0 == 3:
            name += {4: " qkv", 5: " q_cross", 7: " fc1", 8: " vocab"}.get(k1, " out/fc2 (->LN)")
        iv[name].append((t1 - t0) / 1e3)
    tot = sum(sum(v) for v in iv.values())
    print(f"{'kernel':32s} {'n':>7s} {'mean us':>9s} {'p50':>8s} {'p90':>8s} {'share':>7s}")
    for name, v in sorted(iv.items(), key=lambda kv: -sum(kv[1])):
        a = np.asarray(v)
        print(f"{name:32s} {len(a):7d} {a.mean():9.2f} {np.median(a):8.2f} {np.percentile(a, 90):8.2f} {100 * a.sum() / tot:6.1f}%")
    # resident-ahead time: entry -> ready of the same kernel
    ent = {}
    ahead = defaultdict(list)
    for tt, k, w in zip(t, kid, what):
        if w == 0:
            ent[k] = tt
        elif k in ent:
            ahead[NAMES.get(k, str(k))].append((tt - ent.pop(k)) / 1e3)
    print("\nentry -> ready (resident ahead of its dependency):")
    try:
        for name, v in ahead.items():
            print(f"  {name:28s} mean {np.mean(v):6.2f} us")
    except BrokenPipeError:
        pass


if __name__ == "__main__":
    main(sys.argv[1])
