"""Consumes tests/golden/ct2_convert_capture.json -- what CTranslate2's TransformersConverter wrote for a seeded micro
Whisper at float16 / int8_float16 / int8 / bfloat16, recorded by tests/golden/capture_ct2_convert.py -- whenever it is
present.  It cannot be produced without ctranslate2, so until it is committed these tests SKIP with that reason and
the recalled rules (int8 dequantization, the converter's config.json keys) stay unpinned."""
import json
import os

import numpy as np
import pytest

HERE = os.path.dirname(os.path.abspath(__file__))
FIXTURE = os.path.join(HERE, "golden", "ct2_convert_capture.json")
needs_capture = pytest.mark.skipif(not os.path.exists(FIXTURE), reason=(
    "no TransformersConverter capture committed: run tests/golden/capture_ct2_convert.py on a machine with ctranslate2 "
    "and transformers (the int8 dequantization and converter metadata rules stay unpinned until then)"))


def _load():
    with open(FIXTURE) as f:
        return json.load(f)


@needs_capture
def test_converted_variable_tables_are_read():
    """Every name the loader maps exists with the dtype the quantization implies; int8 weights carry one scale per row."""
    from whisperlive_b200 import ct2_format
    for q, conv in _load()["conversions"].items():
        shapes = {k: tuple(v["shape"]) for k, v in conv["variables"].items()}
        ct2_format.ct2_plan(shapes, conv["aliases"])
        # the spec's head counts, which the loader checks against d_model
        assert set(conv["num_heads"]) == {"encoder", "decoder"}, q
        for name, v in conv["variables"].items():
            if v["dtype_id"] == 1:
                assert name + "_scale" in shapes, (q, name)
                assert int(np.prod(shapes[name + "_scale"])) == shapes[name][0], (q, name)


@needs_capture
def test_converter_metadata_matches_the_recalled_rule():
    for q, conv in _load()["conversions"].items():
        cfg = conv["config"]
        assert [list(h) for h in cfg["alignment_heads"]] == [[1, 0], [1, 1]], q
        assert cfg["suppress_ids"] == [1, 2, 7] and cfg["suppress_ids_begin"] == [220, 50257], q
        assert cfg["lang_ids"] == [50259, 50261, 50265], q


@needs_capture
def test_int8_rows_follow_the_quantization_rule():
    for q, conv in _load()["conversions"].items():
        for name, r in conv["rows"].items():
            if "scale" in r:
                rows = np.asarray(r["rows"])
                assert np.all(np.abs(rows) <= 127) and np.all(rows == np.rint(rows)), (q, name)
                assert np.all(np.abs(rows).max(axis=tuple(range(1, rows.ndim))) == 127), (q, name)


@needs_capture
def test_a_generation_config_is_read_alone():
    """model_metadata takes the keys from generation_config.json alone when it exists: a key it lacks is not taken
    from config.json (the heads fall back to the converter's default, the upper half of the layers, all heads)."""
    from whisperlive_b200.config import dims_for
    cfg = _load()["partial_generation_config"]
    assert cfg["suppress_ids"] == [1, 2, 7]
    assert not cfg.get("suppress_ids_begin")
    assert [tuple(h) for h in cfg["alignment_heads"]] == dims_for("micro").default_alignment_heads()
