"""fp64 restatement of the reference's index-based sentence rewards (trainers/self_critical_objective.py:124-231):
the numbers `nm_sentence_ngram_reward` must reproduce.  n-grams are tuples in a Counter, decremented on every match,
as the reference does with str(ndarray) keys.  Where the reference's GLEU divides 0 by 0 (its assert fails) the
score is 0.0, the value the kernel defines there."""
from collections import Counter
from itertools import takewhile

import numpy as np

END = 2


def _ngrams(row, n):
    windows = [tuple(int(x) for x in row[i:i + n]) for i in range(len(row) - n + 1)]
    return list(takewhile(lambda g: g[-1] != END, windows))


def count_matching_ngrams(ref, hyp, n):
    ref_grams = _ngrams(ref, n)
    counts = Counter(ref_grams)
    matched = total = 0
    for gram in _ngrams(hyp, n):
        if counts[gram] > 0:
            matched += 1
            counts[gram] -= 1
        total += 1
    return matched, total, len(ref_grams)


def sentence_bleu(references: np.ndarray, hypotheses: np.ndarray) -> np.ndarray:
    scores = []
    for ref, hyp in zip(np.transpose(references), np.transpose(hypotheses)):
        matched, totals = [], []
        for n in range(1, 5):
            m, t, _ = count_matching_ngrams(ref, hyp, n)
            if n > 1:
                m, t = m + 1, t + 1
            matched.append(m)
            totals.append(t)
        if totals[0] == 0:
            scores.append(0.0)
            continue
        precision = (np.prod(matched) / np.prod(totals)) ** .25
        ref_len = sum(1 for _ in takewhile(lambda i: i != END, ref))
        scores.append(min(1.0, np.exp(1 - ref_len / totals[0])) * precision)
    return np.array(scores, dtype=np.float32)


def sentence_gleu(references: np.ndarray, hypotheses: np.ndarray) -> np.ndarray:
    scores = []
    for ref, hyp in zip(np.transpose(references), np.transpose(hypotheses)):
        counts = [count_matching_ngrams(ref, hyp, n) for n in range(1, 5)]
        m, h, r = (sum(c[i] for c in counts) for i in range(3))
        scores.append(0.0 if h == 0 or r == 0 else min(m / h, m / r))
    return np.array(scores, dtype=np.float32)
