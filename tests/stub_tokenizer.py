"""A whitespace tokenizer with the call interface of transformers' CLIPTokenizer that the pipeline and load_new_concept use
(__call__ with padding="max_length" / truncation / return_tensors="pt", add_tokens, convert_tokens_to_ids, __len__,
model_max_length).  Words map to ids by a hash, so tests need no vocabulary file; SD's BOS 49406 / EOS 49407 are kept and
padding repeats EOS as SD's tokenizer does."""
from __future__ import annotations

import zlib
from types import SimpleNamespace

import torch

BOS, EOS = 49406, 49407


class StubTokenizer:
    def __init__(self, base_vocab: int = 49408, model_max_length: int = 77):
        self.base_vocab, self.model_max_length = base_vocab, model_max_length
        self.added = {}

    def __len__(self):
        return self.base_vocab + len(self.added)

    def add_tokens(self, names):
        n = 0
        for t in names:
            if t not in self.added:
                self.added[t] = len(self)
                n += 1
        return n

    def convert_tokens_to_ids(self, t):
        return self.added[t] if t in self.added else zlib.crc32(t.encode()) % (min(self.base_vocab, BOS))

    def encode(self, text):
        return [self.convert_tokens_to_ids(w) for w in text.split()]

    def __call__(self, texts, padding="max_length", max_length=None, truncation=True, return_tensors="pt"):
        assert padding == "max_length" and return_tensors == "pt"
        texts = [texts] if isinstance(texts, str) else texts
        L = max_length or self.model_max_length
        rows = []
        for t in texts:
            ids = [BOS] + self.encode(t)
            ids = ids[:L - 1] if truncation else ids
            ids = ids + [EOS] * (L - len(ids))
            rows.append(ids)
        return SimpleNamespace(input_ids=torch.tensor(rows, dtype=torch.long))
