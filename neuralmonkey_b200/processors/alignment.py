"""Word alignments in text form as matrices (reference: neuralmonkey/processors/alignment.py:29-61)."""
import re
from typing import List

import numpy as np

_PAIR_SEPARATOR = re.compile(r"[-:]")


class WordAlignmentPreprocessor:
    """Map the tokens of one alignment line to a [target_len, source_len] matrix.

    A token is `s-t` or `s:t` (the separators are interchangeable), optionally followed by `/weight`; s indexes the
    source sentence, t the target sentence, and the weight defaults to 1.  Indices are zero-based unless
    `zero_based=False`.  Pairs outside the matrix are skipped; a later token for the same cell overwrites an
    earlier one.  With `normalize`, each row is divided by its sum; rows that sum to zero stay zero.  The
    preprocessing runs on the host, once per dataset."""

    # pylint: disable=too-few-public-methods
    def __init__(self, source_len: int, target_len: int, dtype=np.float32, normalize: bool = True,
                 zero_based: bool = True) -> None:
        self._source_len = source_len
        self._target_len = target_len
        self._dtype = dtype
        self._normalize = normalize
        self._offset = 0 if zero_based else 1

    def __call__(self, sentence: List[str]) -> np.ndarray:
        matrix = np.zeros((self._target_len, self._source_len), self._dtype)
        for token in sentence:
            pair, _, weight = token.partition("/")
            src, tgt = (int(index) - self._offset for index in _PAIR_SEPARATOR.split(pair))
            if src < self._source_len and tgt < self._target_len:
                matrix[tgt, src] = float(weight) if weight else 1.
        if self._normalize:
            sums = matrix.sum(axis=1, keepdims=True)
            matrix = np.divide(matrix, sums, out=np.zeros_like(matrix), where=sums != 0)
        return matrix
