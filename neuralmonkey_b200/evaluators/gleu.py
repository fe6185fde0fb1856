"""GLEU (reference: neuralmonkey/evaluators/gleu.py): the sentence-level metric of Google's NMT system (Wu et al.,
https://arxiv.org/pdf/1609.08144v2.pdf), the minimum of the recall and the precision of all n-grams up to n.
The n-gram counts are those of `evaluators.bleu`; quirks of the reference kept:

* the "true positives" of a hypothesis add, for every DISTINCT hypothesis n-gram, its reference count - not
  min(hypothesis count, reference count);
* counts are accumulated over the orders 1..n, and the function returns (0, 0) as soon as no hypothesis n-gram has
  been seen after an order;
* no smoothing: a corpus without reference n-grams divides by zero (ZeroDivisionError), as in the reference."""
from typing import List, Tuple

from neuralmonkey_b200.evaluators.bleu import BLEUEvaluator


class GLEUEvaluator:
    def __init__(self, n: int = 4, deduplicate: bool = False, name: str = None) -> None:
        if name is None:
            name = "GLEU-{}".format(n)
            if deduplicate:
                name += "-dedup"
        self.name = name
        self.n = n
        self.deduplicate = deduplicate

    def score_batch(self, hypotheses: List[List[str]], references: List[List[str]]) -> float:
        hypotheses, references = list(hypotheses), list(references)
        if len(hypotheses) != len(references):
            raise ValueError("Hypothesis and reference lists do not have the same length: {} vs {}."
                             .format(len(hypotheses), len(references)))
        if not hypotheses:
            raise ValueError("No hyp/ref pair to evaluate.")
        listed_references = [[s] for s in references]
        if self.deduplicate:
            hypotheses = BLEUEvaluator.deduplicate_sentences(hypotheses)
        return GLEUEvaluator.gleu(hypotheses, listed_references, self.n)

    def __call__(self, decoded: List[List[str]], references: List[List[str]]) -> float:
        return self.score_batch(decoded, references)

    @staticmethod
    def total_precision_recall(hypotheses: List[List[str]], references_list: List[List[List[str]]], ngrams: int,
                               case_sensitive: bool) -> Tuple[float, float]:
        """Modified n-gram precision and recall of a corpus (gleu.py:45-95)."""
        true_positives = generated = target = 0
        for n in range(1, ngrams + 1):
            for hypothesis, references in zip(hypotheses, references_list):
                reference_counts = BLEUEvaluator.merge_max_counters(
                    [BLEUEvaluator.ngram_counts(ref, n, not case_sensitive) for ref in references])
                target += sum(reference_counts.values())
                hypothesis_counts = BLEUEvaluator.ngram_counts(hypothesis, n, not case_sensitive)
                true_positives += sum(reference_counts[gram] for gram in hypothesis_counts)
                generated += sum(hypothesis_counts.values())
            if generated == 0:
                return 0, 0
        return true_positives / generated, true_positives / target

    @staticmethod
    def gleu(hypotheses: List[List[str]], references: List[List[List[str]]], ngrams: int = 4,
             case_sensitive: bool = True) -> float:
        """GLEU of a corpus with one or more references per sentence, without smoothing."""
        prec, recall = GLEUEvaluator.total_precision_recall(hypotheses, references, ngrams, case_sensitive)
        return min(recall, prec)

    @staticmethod
    def compare_scores(score1: float, score2: float) -> int:
        return (score1 > score2) - (score1 < score2)
