"""Bundle the INPUTS of the reference's own hot-path experiments - tests/{bahdanau,transformer,beamsearch}.ini
and the toy corpora / vocabularies they name - into tests/golden/reference_experiments.json, so that the
`-m gpu` tests can train them UNCHANGED on a box that has no /root/reference (tests/test_gpu_reference_inis.py
unpacks the bundle into a scratch tree and runs `neuralmonkey-train tests/<name>.ini` from its root).
These are data fixtures (configurations and corpora), the same role tests/golden/*.npz play for tensors.

    python tests/golden/make_reference_bundle.py        # needs /root/reference
"""
import json
import os

REFERENCE = "/root/reference"
FILES = ["tests/bahdanau.ini", "tests/transformer.ini", "tests/beamsearch.ini",
         "tests/data/train.tc.en", "tests/data/train.tc.de", "tests/data/val.tc.en", "tests/data/val.tc.de",
         "tests/data/encoder_vocab.tsv", "tests/data/decoder_vocab.tsv"]


# the INIs that became trainable in the CPU-only part of round 2 (scaled-dot attention objects, edit operations,
# word2vec embeddings): a bundle of their own, so that the first one stays byte for byte what the GPU-verified
# tests read
LATE_FILES = ["tests/factored.ini", "tests/post-edit.ini", "tests/language-model.ini",
              "tests/data/encoder_vocab.tsv", "tests/data/factored_decoder_vocab.tsv",
              "tests/data/factored_surface_vocab.tsv", "tests/data/factored_tag_vocab.tsv",
              "tests/data/multi/train.forms-cs.txt", "tests/data/multi/train.forms-en.txt",
              "tests/data/multi/train.tags-en.txt", "tests/data/multi/val.forms-cs.txt",
              "tests/data/multi/val.forms-en.txt", "tests/data/multi/val.tags-en.txt",
              "tests/data/postedit/dev.mt", "tests/data/postedit/dev.pe", "tests/data/postedit/dev.src",
              "tests/data/postedit/train.mt", "tests/data/postedit/train.pe", "tests/data/postedit/train.src",
              "tests/data/postedit_target_vocab.tsv", "tests/data/sample.w2v", "tests/data/train.tc.en",
              "tests/data/val.tc.en"]


# what the CPU replays of tests_run.sh need beyond the two bundles above (tests/test_reference_tests_run_cpu.py,
# tests/test_reference_inis_cpu.py): small.ini, the run-time dataset INIs, the ten-sentence test corpus and the
# captions / image lists of the flickr30k sample (its .npz feature maps are too large to bundle; the test writes
# seeded stand-ins of the same shape)
RUN_FILES = ["tests/data/flickr30k/train.de", "tests/data/flickr30k/val.de", "tests/data/flickr30k/train_images.npz.txt",
             "tests/data/flickr30k/val_images.npz.txt",
             "tests/small.ini", "tests/test_data.ini", "tests/beamsearch_ensembles.ini",
             "tests/test_data_ensembles_single.ini", "tests/test_data_ensembles_duplicate.ini",
             "tests/test_data_ensembles_all.ini", "tests/data/val10.tc.en", "tests/data/val10.tc.de",
             "tests/data/val10.part1.tc.en", "tests/data/val10.part2.tc.en"]
BUNDLES = ("reference_experiments.json", "reference_experiments_late.json", "reference_experiments_run.json")


def unpack(tree: str) -> None:
    """Every bundle into `tree` (tests/*.ini and tests/data/ as in the reference's tree)."""
    for name in BUNDLES:
        with open(os.path.join(os.path.dirname(os.path.abspath(__file__)), name), encoding="utf-8") as handle:
            bundle = json.load(handle)
        for rel, text in bundle["files"].items():
            path = os.path.join(tree, rel)
            os.makedirs(os.path.dirname(path), exist_ok=True)
            with open(path, "w", encoding="utf-8") as handle:
                handle.write(text)


def write(files, name) -> None:
    bundle = {"source": "ufal/neuralmonkey @ 8b1465270f6bb28d5417a85cec492f7179036ede", "files": {}}
    for rel in files:
        with open(os.path.join(REFERENCE, rel), encoding="utf-8") as handle:
            bundle["files"][rel] = handle.read()
    out = os.path.join(os.path.dirname(os.path.abspath(__file__)), name)
    with open(out, "w", encoding="utf-8") as handle:
        json.dump(bundle, handle, ensure_ascii=False, indent=0)
    print("wrote", out, sum(len(v) for v in bundle["files"].values()), "characters")


def main() -> None:
    write(FILES, "reference_experiments.json")
    write(LATE_FILES, "reference_experiments_late.json")
    write(RUN_FILES, "reference_experiments_run.json")


if __name__ == "__main__":
    main()
