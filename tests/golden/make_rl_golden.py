"""Golden vectors from the reference's own reward code: `sentence_bleu` / `sentence_gleu` of
`neuralmonkey/trainers/self_critical_objective.py` (imported over the numpy TensorFlow stand-in of tf_numpy_shim.py)
and `GLEUEvaluator` of `neuralmonkey/evaluators/gleu.py`, run on random and edge-case batches.

Each case is a pair of time-major int64 arrays references [T_r, B] / hypotheses [T_h, B].  Where the reference's
GLEU asserts (a 0/0 precision or recall) the row is scored on its own: the failing sentence gets 0.0, the value
`nm_sentence_ngram_reward` defines there, and `<case>_gleu_undefined` lists it.

    python tests/golden/make_rl_golden.py   ->  tests/golden/rl_golden.npz
"""
import os
import sys
import warnings

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
import tf_numpy_shim as shim  # noqa: E402
from make_host_golden import install_stubs  # noqa: E402

END, PAD = 2, 0


def _cases():
    rng = np.random.RandomState(29)
    cases = {}
    # random batches over a small vocabulary (many matches), with </s> and <pad> tails
    for tag, (t_r, t_h, bsz, vocab) in {"small": (12, 12, 64, 8), "ragged": (15, 9, 48, 6),
                                        "long": (200, 200, 8, 12), "large_ids": (40, 50, 32, 32000)}.items():
        refs = rng.randint(4, vocab + 4, size=(t_r, bsz)).astype(np.int64)
        hyps = rng.randint(4, vocab + 4, size=(t_h, bsz)).astype(np.int64)
        if tag == "large_ids":          # hypotheses share many tokens with their references
            hyps[:min(t_r, t_h)] = np.where(rng.rand(min(t_r, t_h), bsz) < 0.6, refs[:min(t_r, t_h)],
                                            hyps[:min(t_r, t_h)])
        for arr in (refs, hyps):
            for b in range(bsz):
                if rng.rand() < 0.85:               # most rows end with </s> then <pad>; the others are truncated
                    end = rng.randint(0, arr.shape[0])
                    arr[end, b] = END
                    arr[end + 1:, b] = PAD
        cases[tag] = (refs, hyps)
    # hand-made rows, one quirk each (columns of one batch, padded to a common length with <pad>)
    rows = [
        ([5, 6, 7, 8, 2, 0], [5, 6, 7, 8, 2, 0]),          # identical
        ([5, 6, 7, 8, 9, 10], [5, 6, 7, 8, 2, 0]),         # reference truncated at max_output_len: no </s>
        ([5, 6, 7, 2, 0, 0], [5, 6, 7, 8, 9, 10]),         # hypothesis without </s>
        ([5, 5, 5, 5, 2, 0], [5, 5, 5, 5, 5, 5]),          # repeated n-grams: clipped counts
        ([5, 6, 5, 6, 5, 2], [6, 5, 6, 5, 6, 5]),          # repeated bigrams
        ([0, 0, 0, 0, 0, 0], [0, 0, 0, 0, 0, 0]),          # all <pad>: <pad> is an ordinary token
        ([5, 0, 6, 2, 0, 0], [5, 0, 6, 0, 2, 0]),          # <pad> before </s> counts
        ([2, 0, 0, 0, 0, 0], [5, 6, 2, 0, 0, 0]),          # empty reference
        ([5, 6, 2, 0, 0, 0], [2, 0, 0, 0, 0, 0]),          # empty hypothesis: BLEU 0
        ([2, 5, 6, 7, 2, 0], [2, 5, 6, 7, 8, 2]),          # </s> first: only unigrams stop there
        ([5, 2, 6, 7, 8, 2], [5, 2, 6, 7, 9, 2]),          # </s> inside the first window of higher orders
        ([7, 8, 9, 2, 0, 0], [9, 8, 7, 2, 0, 0]),          # unigrams match, no bigram does
        ([2, 2, 2, 2, 2, 2], [5, 6, 2, 0, 0, 0]),          # no reference n-gram: GLEU recall 0/0
        ([5, 6, 7, 2, 0, 0], [2, 2, 2, 2, 2, 2]),          # no hypothesis n-gram: GLEU precision 0/0
    ]
    cases["quirks"] = (np.array([r for r, _ in rows], np.int64).T.copy(),
                       np.array([h for _, h in rows], np.int64).T.copy())
    # T_h != T_r
    cases["unequal"] = (np.array([[5, 6, 7, 8, 9, 2, 0, 0, 0, 0]] * 3, np.int64).T.copy(),
                        np.array([[5, 6, 2], [5, 6, 7], [9, 9, 9]], np.int64).T.copy())
    return cases


def _gleu_rows(gleu, refs, hyps):
    """The reference's sentence_gleu, sentence by sentence where it asserts."""
    try:
        with warnings.catch_warnings():
            warnings.simplefilter("ignore")
            return gleu(refs, hyps), []
    except AssertionError:
        pass
    out, undefined = [], []
    for b in range(refs.shape[1]):
        try:
            with warnings.catch_warnings():
                warnings.simplefilter("ignore")
                out.append(float(gleu(refs[:, b:b + 1], hyps[:, b:b + 1])[0]))
        except AssertionError:
            out.append(0.0)
            undefined.append(b)
    return np.array(out, np.float32), undefined


def main():
    install_stubs()
    shim.install()
    from neuralmonkey.trainers.self_critical_objective import sentence_bleu, sentence_gleu
    from neuralmonkey.evaluators.gleu import GLEUEvaluator

    out = {}
    for tag, (refs, hyps) in _cases().items():
        out[tag + "_refs"], out[tag + "_hyps"] = refs, hyps
        out[tag + "_bleu"] = sentence_bleu(refs, hyps)
        out[tag + "_gleu"], undefined = _gleu_rows(sentence_gleu, refs, hyps)
        out[tag + "_gleu_undefined"] = np.array(undefined, np.int64)

    # GLEUEvaluator over words, as the REINFORCE objective calls it: ([hypothesis], [reference]) per sentence,
    # and one corpus call
    words = ["w{}".format(i) for i in range(6)]
    rng = np.random.RandomState(31)
    hyps = [[words[i] for i in rng.randint(0, 6, size=rng.randint(1, 9))] for _ in range(40)]
    refs = [[words[i] for i in rng.randint(0, 6, size=rng.randint(1, 9))] for _ in range(40)]
    hyps[0], refs[0] = [""], ["w1", "w2"]                 # what an empty sentence becomes after split(" ")
    hyps[1] = ["w1", "w1", "w1", "w1"]
    out["eval_hyps"] = np.array([" ".join(h) for h in hyps])
    out["eval_refs"] = np.array([" ".join(r) for r in refs])
    for n, dedup in ((4, False), (2, False), (4, True)):
        ev = GLEUEvaluator(n=n, deduplicate=dedup)
        key = "eval_n{}_{}".format(n, "dedup" if dedup else "plain")
        out[key + "_sentence"] = np.array([ev([h], [r]) for h, r in zip(hyps, refs)], np.float64)
        out[key + "_corpus"] = np.array(ev(hyps, refs), np.float64)
        out[key + "_name"] = np.array(ev.name)
    path = os.path.join(HERE, "rl_golden.npz")
    np.savez(path, **out)
    print("wrote", path, sorted(out))


if __name__ == "__main__":
    main()
