"""Whisper model dimensions (SURVEY.md §8: head_dim 64 everywhere, FFN = 4d,
encoder positions 1500, decoder positions 448)."""
from __future__ import annotations

from dataclasses import dataclass, field
from typing import List, Optional, Tuple


@dataclass
class WhisperDims:
    name: str
    d_model: int
    n_heads: int
    enc_layers: int
    dec_layers: int
    n_mels: int
    vocab: int
    n_audio_ctx: int = 1500
    n_text_ctx: int = 448
    # (layer, head) pairs whose cross-attention is used for word alignment
    # (CT2 config.json "alignment_heads"); None -> all heads of the upper half of the layers,
    # which is what the CT2 converter falls back to when the HF generation_config has none.
    alignment_heads: Optional[List[Tuple[int, int]]] = None

    @property
    def multilingual(self) -> bool:
        return self.vocab >= 51865

    @property
    def num_languages(self) -> int:
        return self.vocab - 51765 - int(self.multilingual)

    @property
    def head_dim(self) -> int:
        return 64

    @property
    def d_ff(self) -> int:
        return 4 * self.d_model

    def default_alignment_heads(self) -> List[Tuple[int, int]]:
        if self.alignment_heads is not None:
            return list(self.alignment_heads)
        return [(l, h) for l in range(self.dec_layers // 2, self.dec_layers) for h in range(self.n_heads)]


_TABLE = {
    # name: (d_model, heads, enc layers, dec layers, mels, vocab)
    "micro.en": (128, 2, 2, 2, 80, 51864),   # test-only shape, not a released checkpoint
    "micro": (128, 2, 2, 2, 80, 51865),      # test-only multilingual shape
    "tiny.en": (384, 6, 4, 4, 80, 51864),
    "tiny": (384, 6, 4, 4, 80, 51865),
    "base.en": (512, 8, 6, 6, 80, 51864),
    "base": (512, 8, 6, 6, 80, 51865),
    "small.en": (768, 12, 12, 12, 80, 51864),
    "small": (768, 12, 12, 12, 80, 51865),
    "medium.en": (1024, 16, 24, 24, 80, 51864),
    "medium": (1024, 16, 24, 24, 80, 51865),
    "large-v2": (1280, 20, 32, 32, 80, 51865),
    "large-v3": (1280, 20, 32, 32, 128, 51866),
    "large-v3-turbo": (1280, 20, 32, 4, 128, 51866),
    "turbo": (1280, 20, 32, 4, 128, 51866),
    # distilled checkpoints: the teacher's encoder, two decoder layers
    "distil-small.en": (768, 12, 12, 2, 80, 51864),
    "distil-medium.en": (1024, 16, 24, 2, 80, 51864),
    "distil-large-v2": (1280, 20, 32, 2, 80, 51865),
    "distil-large-v3": (1280, 20, 32, 2, 128, 51866),
}


def dims_for(name: str) -> WhisperDims:
    if name not in _TABLE:
        raise KeyError(f"unknown Whisper size {name!r}; known: {sorted(_TABLE)}")
    d, h, le, ld, m, v = _TABLE[name]
    return WhisperDims(name, d, h, le, ld, m, v)


def model_names() -> list:
    return sorted(_TABLE)
