"""Generate tests/golden/word2vec_golden.json: the reference's own util/word2vec.py loader (its imports
redirected to this package's vocabulary) run on the reference's tests/data/sample.w2v, which
reference_experiments_late.json bundles.  tests/test_host.py compares this package's loader with it.

    python tests/golden/make_word2vec_golden.py        # needs the reference tree at REF
"""
import json
import os
import sys

REF = "/root/reference"
ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))


def main() -> None:
    sys.path.insert(0, ROOT)
    module = os.path.join(REF, "neuralmonkey", "util", "word2vec.py")
    code = open(module).read().replace("from typeguard import check_argument_types", "") \
        .replace("from neuralmonkey.vocabulary import", "from neuralmonkey_b200.vocabulary import") \
        .replace("check_argument_types()", "").replace("np.float)", "np.float64)")
    ref = {}
    exec(compile(code, module, "exec"), ref)  # pylint: disable=exec-used
    theirs = ref["Word2Vec"](os.path.join(REF, "tests", "data", "sample.w2v"))
    out = {"what": "the reference's util/word2vec.py Word2Vec loader on tests/data/sample.w2v "
                   "(reference_experiments_late.json); written by make_word2vec_golden.py",
           "index_to_word": list(theirs.vocabulary.index_to_word), "embeddings": theirs.embeddings.tolist()}
    with open(os.path.join(os.path.dirname(os.path.abspath(__file__)), "word2vec_golden.json"), "w") as handle:
        json.dump(out, handle)


if __name__ == "__main__":
    main()
