"""Records pyannote's own wespeaker-voxceleb-resnet34-LM on a machine that has pyannote.audio and the checkpoint, so
the protocol whisperlive_b200/speaker.py recalls can be checked (tests/test_spk_capture.py):

  * the checkpoint's tensor table (name, shape, dtype): the names the reader expects;
  * the fbank after CMN of fixed jfk slices, taken from pyannote's own feature path (input scaling, fbank options, CMN);
  * per-stage activation max / RMS of the real weights (whether fp16 activations are safe with them);
  * the embeddings of the same slices from pyannote's ``Inference(window="whole")``, as SpeakerDiarizer calls it.

Writes tests/golden/wespeaker_capture.npz and .json.  Run from the repository root:
    WLB200_SPK_MODEL=<pytorch_model.bin> python tests/golden/capture_wespeaker.py"""
import json
import os
import sys

import numpy as np

ROOT = os.path.abspath(os.path.join(os.path.dirname(__file__), "..", ".."))
sys.path.insert(0, ROOT)

SLICES = [(0.0, 2.5), (2.5, 4.2), (4.2, 7.0), (7.0, 11.0), (0.0, 0.3)]   # seconds of the jfk fixture


def inputs():
    jfk = np.load(os.path.join(ROOT, "tests", "golden", "jfk_16k_i16.npy")).astype(np.float32) / 32768.0
    return {f"jfk_{a:.1f}_{b:.1f}": jfk[int(a * 16000):int(b * 16000)] for a, b in SLICES}


def main():
    import torch
    from pyannote.audio import Inference, Model

    name = os.environ.get("WLB200_SPK_MODEL") or "pyannote/wespeaker-voxceleb-resnet34-LM"
    model = Model.from_pretrained(name)
    model.eval()
    inference = Inference(model, window="whole", device=torch.device("cpu"))
    state = model.state_dict()
    meta = {"model": name, "tensors": {k: [list(v.shape), str(v.dtype)] for k, v in state.items()}, "stages": {}}
    out = {}
    resnet = model.resnet
    for key, wave in inputs().items():
        w = torch.from_numpy(wave)[None, None]
        with torch.no_grad():
            feats = model.compute_fbank(w)                    # [1, T, 80] after scaling, fbank and CMN
            out["fbank_cmn_" + key] = feats[0].numpy()
            x = feats.permute(0, 2, 1).unsqueeze(1)
            h = torch.relu(resnet.bn1(resnet.conv1(x)))
            stats = [h]
            for layer in (resnet.layer1, resnet.layer2, resnet.layer3, resnet.layer4):
                h = layer(h)
                stats.append(h)
            meta["stages"][key] = [[float(s.abs().max()), float(s.pow(2).mean().sqrt())] for s in stats]
            out["embedding_" + key] = np.asarray(inference({"waveform": w[0], "sample_rate": 16000}), np.float32)
    np.savez_compressed(os.path.join(ROOT, "tests", "golden", "wespeaker_capture.npz"), **out)
    with open(os.path.join(ROOT, "tests", "golden", "wespeaker_capture.json"), "w") as f:
        json.dump(meta, f, indent=1)


if __name__ == "__main__":
    main()
