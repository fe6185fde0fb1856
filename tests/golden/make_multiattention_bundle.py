"""Bundle the INPUTS of the reference's multi-source attention experiments - tests/flat-multiattention.ini and
tests/hier-multiattention.ini with the flickr30k sample's captions, image lists and the vocabularies - into
tests/golden/multiattention_experiments.json.  The images themselves are not bundled: the tests write seeded
stand-ins under the listed names (8 x 8 x 2048 `.npz` feature maps for the flat INI, 32 x 32 RGB images for the
hierarchical one).

    python tests/golden/make_multiattention_bundle.py        # needs /root/reference
"""
import json
import os

import numpy as np

REFERENCE = "/root/reference"
NAME = "multiattention_experiments.json"
FILES = ["tests/flat-multiattention.ini", "tests/hier-multiattention.ini",
         "tests/data/flickr30k/train.en", "tests/data/flickr30k/train.de", "tests/data/flickr30k/val.en",
         "tests/data/flickr30k/val.de", "tests/data/flickr30k/train_images.txt", "tests/data/flickr30k/val_images.txt",
         "tests/data/flickr30k/train_images.npz.txt", "tests/data/flickr30k/val_images.npz.txt",
         "tests/data/encoder_vocab.tsv", "tests/data/decoder_vocab.tsv"]


def unpack(tree: str, seed: int = 30) -> None:
    """The bundle into `tree` (as in the reference's tree), plus seeded stand-ins of every listed image."""
    with open(os.path.join(os.path.dirname(os.path.abspath(__file__)), NAME), encoding="utf-8") as handle:
        bundle = json.load(handle)
    for rel, text in bundle["files"].items():
        path = os.path.join(tree, rel)
        os.makedirs(os.path.dirname(path), exist_ok=True)
        with open(path, "w", encoding="utf-8") as handle:
            handle.write(text)
    from PIL import Image
    flickr = os.path.join(tree, "tests", "data", "flickr30k")
    rng = np.random.default_rng(seed)
    for listing in ("train_images.npz.txt", "val_images.npz.txt"):
        for name in open(os.path.join(flickr, listing)).read().split():
            np.savez(os.path.join(flickr, name), rng.standard_normal((8, 8, 2048)).astype(np.float32))
    for listing in ("train_images.txt", "val_images.txt"):
        for name in open(os.path.join(flickr, listing)).read().split():
            Image.fromarray(rng.integers(0, 256, (32, 32, 3), dtype=np.uint8), "RGB").save(os.path.join(flickr, name),
                                                                                           format="PNG")


def main() -> None:
    bundle = {"source": "ufal/neuralmonkey @ 8b1465270f6bb28d5417a85cec492f7179036ede", "files": {}}
    for rel in FILES:
        with open(os.path.join(REFERENCE, rel), encoding="utf-8") as handle:
            bundle["files"][rel] = handle.read()
    out = os.path.join(os.path.dirname(os.path.abspath(__file__)), NAME)
    with open(out, "w", encoding="utf-8") as handle:
        json.dump(bundle, handle, ensure_ascii=False, indent=0)
    print("wrote", out, sum(len(v) for v in bundle["files"].values()), "characters")


if __name__ == "__main__":
    main()
