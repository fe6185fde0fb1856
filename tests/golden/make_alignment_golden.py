"""Run the reference's own `WordAlignmentPreprocessor` (neuralmonkey/processors/alignment.py, plain numpy) over the
first lines of tests/data/train.tc.ali and over hand-made lines for the `:` and `/weight` forms, one-based indices,
out-of-range pairs and rows left empty by normalisation; write tests/golden/alignment_golden.json.

    python tests/golden/make_alignment_golden.py        # needs /root/reference
"""
import importlib.util
import json
import os

REFERENCE = "/root/reference"
HERE = os.path.dirname(os.path.abspath(__file__))

HAND_MADE = ["0:0 1:2/0.5 1:1/0.25 3-2/2", "1-1 2-3 3-3 5-5", "0-0 7-1 1-6 20-20", "2-0/0.3 0-0/0.1 1-2", ""]
# (source_len, target_len, normalize, zero_based)
SETTINGS = [(12, 8, True, True), (12, 8, False, True), (4, 3, True, True), (6, 4, True, False),
            (6, 4, False, False), (3, 2, False, True)]


def main() -> None:
    spec = importlib.util.spec_from_file_location(
        "reference_alignment", os.path.join(REFERENCE, "neuralmonkey", "processors", "alignment.py"))
    module = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(module)
    with open(os.path.join(REFERENCE, "tests", "data", "train.tc.ali"), encoding="utf-8") as handle:
        lines = [next(handle).strip() for _ in range(20)]
    cases = []
    for source_len, target_len, normalize, zero_based in SETTINGS:
        pre = module.WordAlignmentPreprocessor(source_len, target_len, normalize=normalize, zero_based=zero_based)
        inputs = (lines if zero_based else []) + HAND_MADE
        for line in inputs:
            cases.append({"line": line, "source_len": source_len, "target_len": target_len,
                          "normalize": normalize, "zero_based": zero_based,
                          "matrix": pre(line.split()).tolist()})
    out = os.path.join(HERE, "alignment_golden.json")
    with open(out, "w", encoding="utf-8") as handle:
        json.dump({"source": "ufal/neuralmonkey @ 8b1465270f6bb28d5417a85cec492f7179036ede", "cases": cases},
                  handle, indent=0)
    print("wrote", out, len(cases), "cases")


if __name__ == "__main__":
    main()
