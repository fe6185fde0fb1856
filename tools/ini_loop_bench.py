"""Throughput of `neuralmonkey-train` ITSELF - the call a user of the reference makes - on the en-de model of
BASELINE.json: text files on disk, an INI, the package's own training loop (dataset iteration, padding, string ->
index, pinned upload, the captured training step).  What bench.py's `e2e` measures starts at id tensors in pinned
host memory; this starts at words.

    python tools/ini_loop_bench.py                       # 30 steps of 256 sentences x 50 tokens, V = 32000
    python tools/ini_loop_bench.py --standins --rnn 16 --vocab 300 --sentences 96 --batch 16    # host logic, CPU

The corpus is synthetic (uniform random words, fixed length, as in bench.py); logging and validation periods are
set beyond the run, so the loop never looks at a loss and never waits for the device (the losses of a step are read
when somebody looks at them).  `NMB200_INI_LOOP_EAGER_LOSS=1` makes the wrapper read every step's loss right away -
the behaviour before that change - for comparison.  Timing: wall clock from the moment the loop enters step
`--skip`+1 (the first steps run eagerly and capture the step's CUDA graph) to the completion of the last step on the
device (one synchronize after the last step was issued).  Prints one JSON line."""
import argparse
import json
import math
import os
import random
import sys
import tempfile
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

INI = """
[main]
name="ini loop bench"
tf_manager=<tf_manager>
output="{out}"
overwrite_output_dir=True
batch_size={batch}
epochs=1
train_dataset=<train_data>
val_dataset=<val_data>
trainer=<trainer>
runners=[<runner>]
postprocess=None
evaluation=[("target_bpe", evaluators.BLEU)]
logging_period=1000000000
validation_period=1000000000
random_seed=2574600

[tf_manager]
class=tf_manager.TensorFlowManager
num_threads=4
num_sessions=1

[train_data]
class=dataset.load
series=["source_bpe", "target_bpe"]
data=["{data}/train.src", "{data}/train.tgt"]

[val_data]
class=dataset.load
series=["source_bpe", "target_bpe"]
data=["{data}/val.src", "{data}/val.tgt"]

[shared_vocabulary]
class=vocabulary.from_wordlist
path="{data}/vocab.txt"
contains_header=False
contains_frequencies=False

; examples/translation.ini:90-125 (the model sections of bench_models.ENDE_INI)
[encoder]
class=encoders.SentenceEncoder
name="sentence_encoder"
rnn_size={rnn}
max_input_len={length}
embedding_size={rnn}
dropout_keep_prob=1.0
data_id="source_bpe"
vocabulary=<shared_vocabulary>

[attention]
class=attention.Attention
name="attention_sentence_encoder"
encoder=<encoder>

[decoder]
class=decoders.Decoder
name="decoder"
encoders=[<encoder>]
rnn_size={rnn}
embedding_size={rnn}
attentions=[<attention>]
dropout_keep_prob=1.0
data_id="target_bpe"
vocabulary=<shared_vocabulary>
max_output_len={length}

[trainer]
class=trainers.cross_entropy_trainer.CrossEntropyTrainer
decoders=[<decoder>]
l2_weight=1.0e-8
clip_norm=1.0
use_cuda_graph={graph}

[runner]
class=runners.runner.GreedyRunner
decoder=<decoder>
output_series="target_bpe"
"""


def write_corpus(data: str, sentences: int, length: int, vocab: int, seed: int = 2574600) -> None:
    os.makedirs(data, exist_ok=True)
    words = ["w{}".format(i) for i in range(vocab - 4)]
    with open(os.path.join(data, "vocab.txt"), "w") as handle:
        handle.write("\n".join(["<pad>", "<s>", "</s>", "<unk>"] + words) + "\n")
    rng = random.Random(seed)
    for name, count in (("train", sentences), ("val", 8)):
        with open(os.path.join(data, name + ".src"), "w") as src, open(os.path.join(data, name + ".tgt"), "w") as tgt:
            for _ in range(count):
                src.write(" ".join(rng.choices(words, k=length)) + "\n")
                tgt.write(" ".join(rng.choices(words, k=length - 1)) + "\n")      # + </s> = length target tokens


def main() -> None:
    ap = argparse.ArgumentParser()
    ap.add_argument("--sentences", type=int, default=256 * 30)
    ap.add_argument("--batch", type=int, default=256)
    ap.add_argument("--length", type=int, default=50)
    ap.add_argument("--vocab", type=int, default=32000)
    ap.add_argument("--rnn", type=int, default=300)
    ap.add_argument("--skip", type=int, default=5, help="steps before the timed ones (eager step, graph capture)")
    ap.add_argument("--standins", action="store_true", help="CPU stand-in operations (host logic check only)")
    args = ap.parse_args()

    import torch
    from neuralmonkey_b200 import runtime
    from neuralmonkey_b200.tf_manager import TensorFlowManager
    on_gpu = not args.standins
    if args.standins:
        from tests import cpu_ops
        from neuralmonkey_b200 import ops
        from neuralmonkey_b200.trainers.generic_trainer import GenericTrainer
        for name in cpu_ops.STAND_INS:
            setattr(ops, name, getattr(cpu_ops, name))
        runtime._device = torch.device("cpu")                       # pylint: disable=protected-access
        GenericTrainer._adam_kernel = cpu_ops.adam_kernel           # pylint: disable=protected-access

    steps_total = math.ceil(args.sentences / args.batch)
    if steps_total <= args.skip + 1:
        raise SystemExit("need more than --skip + 1 steps")
    eager_loss = os.environ.get("NMB200_INI_LOOP_EAGER_LOSS", "0") == "1"
    stamps, done = [], []
    original = TensorFlowManager.execute

    def execute(self, batch, feedables, runners, train=False, compute_losses=True, summaries=True):
        if train:
            stamps.append(time.perf_counter())
        results = original(self, batch, feedables, runners, train=train, compute_losses=compute_losses,
                           summaries=summaries)
        if train:
            if eager_loss:
                for result in results:
                    dict(result.losses)                 # what the loop did before the deferred read
            if len(stamps) == steps_total:
                if on_gpu:
                    torch.cuda.synchronize()
                done.append(time.perf_counter())
        return results

    TensorFlowManager.execute = execute
    with tempfile.TemporaryDirectory() as tmp:
        data, out = os.path.join(tmp, "data"), os.path.join(tmp, "out")
        write_corpus(data, args.sentences, args.length, args.vocab)
        ini = os.path.join(tmp, "experiment.ini")
        with open(ini, "w") as handle:
            handle.write(INI.format(out=out, data=data, batch=args.batch, rnn=args.rnn, length=args.length,
                                    graph="True" if on_gpu else "False"))
        argv, sys.argv = sys.argv, ["neuralmonkey-train", ini]
        stdout = os.dup(1)
        os.dup2(2, 1)                                    # the training log goes to stderr; stdout keeps the JSON line
        try:
            from neuralmonkey_b200.train import main as train_main
            train_main()
        finally:
            sys.stdout.flush()
            os.dup2(stdout, 1)
            sys.argv = argv
    assert len(stamps) == steps_total and done, (len(stamps), steps_total)
    timed_steps = steps_total - args.skip
    full = args.sentences // args.batch
    sentences_timed = args.sentences - args.skip * args.batch if full >= args.skip else 0
    seconds = done[0] - stamps[args.skip]
    host_ms = [(b - a) * 1e3 for a, b in zip(stamps[args.skip:-1], stamps[args.skip + 1:])]
    line = {"what": "neuralmonkey-train on text files: en-de GRU+Bahdanau model, {} sentences x {} target tokens per "
                    "step, V = {}; steady state after {} steps".format(args.batch, args.length, args.vocab, args.skip),
            "metric": "train_target_tokens_per_sec", "unit": "tokens/s",
            "value": sentences_timed * args.length / seconds, "ms_per_step": seconds * 1e3 / timed_steps,
            "steps": timed_steps, "host_ms_between_steps_median": sorted(host_ms)[len(host_ms) // 2] if host_ms else None,
            "loss_read": "every step" if eager_loss else "when looked at (never in this run)",
            "device": "cuda" if on_gpu else "cpu stand-ins (host logic check, not a measurement)"}
    print(json.dumps(line), flush=True)


if __name__ == "__main__":
    main()
