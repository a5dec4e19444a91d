"""A small deterministic tokenizer with the interface the controller construction and the pipeline use: `encode` (BOS +
ids + EOS, like CLIPTokenizer.encode), `decode` of single ids, `__call__` with padding="max_length" / truncation /
return_tensors="pt", `add_tokens`, `convert_tokens_to_ids`, `__len__` and `model_max_length`.

Words are split on whitespace; a word longer than four characters becomes several tokens of at most four characters
("walking" -> "walk", "ing"), so the multi-token paths of the word lookup and of the sequence alignment are exercised the way
CLIP's BPE exercises them.  Added tokens (ED-LoRA concept tokens) stay whole.  Ids come from a hash of the piece, so they do
not depend on the order of calls; SD's BOS 49406 / EOS 49407 are kept and padding repeats EOS as SD's tokenizer does.  Used
by the controller fixture generator and by the tests, so both see the same tokens."""
from __future__ import annotations

import zlib
from types import SimpleNamespace

import torch

BOS, EOS = 49406, 49407
PIECE = 4


class ChunkTokenizer:
    def __init__(self, base_vocab: int = 49408, model_max_length: int = 77):
        self.base_vocab, self.model_max_length = base_vocab, model_max_length
        self.added = {}
        self._pieces = {BOS: "<|startoftext|>", EOS: "<|endoftext|>"}

    def __len__(self):
        return self.base_vocab + len(self.added)

    def add_tokens(self, names):
        n = 0
        for t in names:
            if t not in self.added:
                self.added[t] = len(self)
                self._pieces[self.added[t]] = t
                n += 1
        return n

    def convert_tokens_to_ids(self, t):
        if t in self.added:
            return self.added[t]
        i = zlib.crc32(t.encode()) % BOS
        self._pieces.setdefault(i, t)
        return i

    def tokenize(self, text):
        out = []
        for w in text.split():
            out += [w] if (w in self.added or len(w) <= PIECE) else [w[k:k + PIECE] for k in range(0, len(w), PIECE)]
        return out

    def encode(self, text):
        return [BOS] + [self.convert_tokens_to_ids(p) for p in self.tokenize(text)] + [EOS]

    def decode(self, ids):
        return " ".join(self._pieces[int(i)] for i in ids)

    def __call__(self, texts, padding="max_length", max_length=None, truncation=True, return_tensors="pt"):
        assert padding == "max_length" and return_tensors == "pt"
        texts = [texts] if isinstance(texts, str) else texts
        L = max_length or self.model_max_length
        rows = []
        for t in texts:
            ids = self.encode(t)
            if truncation and len(ids) > L:
                ids = ids[:L - 1] + [EOS]
            rows.append(ids + [EOS] * (L - len(ids)))
        return SimpleNamespace(input_ids=torch.tensor(rows, dtype=torch.long))
