"""Generate tests/golden/batched_reference.json by EXECUTING the reference's vendored ``BatchedInferencePipeline``
(whisper_live/transcriber/transcriber_faster_whisper.py:113-571) over the CPU oracle engine, with the stubs of
make_golden_transcribe.py (ctranslate2 -> oracle.engine.OracleWhisper, the faster_whisper modules, and the
deterministic VAD detector of tests/stub_vad.py on both sides).

``faster_whisper.vad.collect_chunks`` is the faster-whisper 1.2.0 restatement in whisperlive_b200/vad.py.  The vendored
class does not run against that version as it stands, so this script applies the two adaptations faster-whisper 1.2.0
itself makes, and nothing else -- see ``ADAPTATIONS`` below.  What is pinned is therefore "the vendored code + two
adaptations", not a capture of upstream faster-whisper.

    python tests/golden/make_golden_batched.py
"""
import copy
import dataclasses
import json
import os
import sys

import torch

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.abspath(os.path.join(HERE, "..", ".."))
sys.path.insert(0, ROOT)

from oracle.engine import OracleWhisper  # noqa: E402
from tests.golden.make_golden_transcribe import install_stubs, make_audio, reference_model, seg_to_json  # noqa: E402
from whisperlive_b200 import vad as wvad  # noqa: E402
from whisperlive_b200.config import dims_for  # noqa: E402
from whisperlive_b200.weights import random_init  # noqa: E402

# about 75 s: speech runs of 8-14 s between pauses of 1.5-3 s -> at least 3 chunks of at most 30 s after collect_chunks
GAPPED_75 = ("gapped", (11.0, 2.0, 13.0, 2.5, 9.0, 3.0, 12.0, 1.5, 10.0, 2.0, 8.0), 11)
GAPPED_40 = ("gapped", (9.0, 2.0, 12.0, 3.0, 14.0), 21)
FAST = dict(max_new_tokens=24)       # random weights rarely emit EOT early: bound the decode so the oracle runs in seconds

SCENARIOS = {
    "vad_groups_of_two": dict(model="micro.en", seed=0, audio=GAPPED_75, kw=dict(batch_size=2, **FAST)),
    "batch_larger_than_chunks": dict(model="micro.en", seed=1, audio=GAPPED_40, kw=dict(batch_size=16, **FAST)),
    "clip_timestamps": dict(model="micro.en", seed=2, audio=("speech", 50.0, 31),
                            kw=dict(clip_timestamps=[{"start": 16000, "end": 16000 * 12}, {"start": 16000 * 14, "end": 16000 * 30},
                                                     {"start": 16000 * 33, "end": 16000 * 49}], batch_size=2, **FAST)),
    "short_no_vad": dict(model="micro.en", seed=3, audio=("speech", 21.0, 41), kw=dict(vad_filter=False, **FAST)),
    "words_across_groups": dict(model="micro.en", seed=1, audio=GAPPED_75,
                                kw=dict(word_timestamps=True, batch_size=2, **FAST)),
    "multilingual_detect": dict(model="micro", seed=1, audio=GAPPED_75,
                                kw=dict(multilingual=True, language=None, language_detection_segments=2, batch_size=3,
                                        **FAST)),
    "multilingual_words": dict(model="micro", seed=4, audio=GAPPED_40,
                               kw=dict(multilingual=True, word_timestamps=True, batch_size=2, **FAST)),
    "prompt_hotwords": dict(model="micro.en", seed=0, audio=GAPPED_40,
                            kw=dict(initial_prompt="hello there", hotwords="foo bar", **FAST)),
    "with_timestamps": dict(model="micro.en", seed=2, audio=GAPPED_75,
                            kw=dict(without_timestamps=False, batch_size=4, max_new_tokens=40)),
    "max_new_tokens": dict(model="micro.en", seed=5, audio=GAPPED_40, kw=dict(max_new_tokens=6, beam_size=2)),
    "vad_dict_parameters": dict(model="micro.en", seed=0, audio=GAPPED_40,
                                kw=dict(vad_parameters={"min_silence_duration_ms": 1000, "max_speech_duration_s": 5}, **FAST)),
    "all_silence": dict(model="micro.en", seed=0, audio=("silence", 40.0, 0), kw=dict()),
    "long_no_vad_raises": dict(model="micro.en", seed=0, audio=("speech", 31.0, 51), kw=dict(vad_filter=False)),
    "prompt_too_long_raises": dict(model="micro.en", seed=0, audio=("speech", 8.0, 52), kw=dict(vad_filter=False,
                                                                                                 max_new_tokens=447)),
}


# ------------------------------------------------------------------------------------------------ ADAPTATIONS
# The only two changes to the vendored code, both as faster-whisper 1.2.0 makes them:
#   1. collect_chunks is called with max_duration=chunk_length, and the chunk metadata it returns (offset / duration on
#      the speech-only axis) is given the keys the vendored forward() reads: start_time = offset,
#      end_time = offset + duration;
#   2. restore_speech_timestamps (reference :1792) maps the yielded segments back to the original time axis.
_CHUNK_LENGTH = [None]


def adapted_collect_chunks(audio, chunks):
    audio_chunks, metadata = wvad.collect_chunks(audio, chunks, max_duration=_CHUNK_LENGTH[0])
    for md in metadata:
        md["start_time"], md["end_time"] = md["offset"], md["offset"] + md["duration"]
    return audio_chunks, metadata


def run_adapted(ref, pipeline, audio, kw):
    _CHUNK_LENGTH[0] = kw.get("chunk_length") or pipeline.model.feature_extractor.chunk_length
    segments, info = pipeline.transcribe(audio, **kw)
    # the reference's restore_speech_timestamps maps in place and returns its argument: it is given the list
    segments = ref.restore_speech_timestamps(list(segments), info.transcription_options.clip_timestamps,
                                             pipeline.model.feature_extractor.sampling_rate)
    return segments, info
# ------------------------------------------------------------------------------------------------------------------


def _plain(x):
    return json.loads(json.dumps(x, default=lambda o: dataclasses.asdict(o) if dataclasses.is_dataclass(o) else list(o)))


def info_to_json(info):
    return dict(language=info.language, language_probability=float(info.language_probability),
                duration=float(info.duration), duration_after_vad=float(info.duration_after_vad),
                all_language_probs=None if info.all_language_probs is None
                else [[k, float(p)] for k, p in info.all_language_probs],
                transcription_options=_plain(dataclasses.asdict(info.transcription_options)),
                vad_options=None if info.vad_options is None else _plain(dataclasses.asdict(info.vad_options)))


def main():
    torch.set_num_threads(8)
    install_stubs()
    sys.path.insert(0, "/root/reference")
    from whisper_live.transcriber import transcriber_faster_whisper as ref
    ref.collect_chunks = adapted_collect_chunks

    out = {}
    for name, sc in SCENARIOS.items():
        dims = dims_for(sc["model"])
        model = reference_model(ref, OracleWhisper(random_init(dims, seed=sc["seed"]), dims), dims)
        pipeline = ref.BatchedInferencePipeline(model)
        try:
            segments, info = run_adapted(ref, pipeline, make_audio(sc["audio"]), copy.deepcopy(sc["kw"]))
            segments = list(segments)
        except (RuntimeError, ValueError) as e:
            out[name] = dict(raises=type(e).__name__, message=str(e))
            print(name, "raises", type(e).__name__)
            continue
        out[name] = dict(segments=[seg_to_json(s) for s in segments], info=info_to_json(info))
        print(name, info.language, len(segments), [(s.id, s.seek, s.start, s.end, len(s.tokens)) for s in segments][:6])
    with open(os.path.join(HERE, "batched_reference.json"), "w") as f:
        json.dump(out, f, indent=1)


if __name__ == "__main__":
    main()
