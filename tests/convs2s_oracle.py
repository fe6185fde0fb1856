"""fp64 restatement of the convolutional seq2seq encoder (encoders/facebook_conv.py), pinned to
tests/golden/convs2s_golden.npz (the reference's own SentenceEncoder over the numpy TF stand-in).  Gradients come
from autograd over it.  `conv1d_glu_residual` doubles as the CPU stand-in of `ops.conv1d_glu_residual`; `bpe_model` builds tests/bpe.ini's
model for the one-step tests."""
import os

import numpy as np
import torch

from tests.classifier_oracle import seq_max_pool  # noqa: F401  (the encoder's output: a stand-in below)

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "convs2s_golden.npz")
CASES = ("padded", "t1", "short", "even", "bpe")
# tag: (conv_features, encoder_layers, kernel_width, max_length)
SHAPES = {"padded": (4, 3, 3, 8), "t1": (3, 1, 5, 4), "short": (5, 1, 5, 5), "even": (6, 3, 4, 6), "bpe": (10, 2, 5, 10)}

# the CPU stand-ins of the ops the encoder calls beyond those of tests/cpu_ops.py
STAND_INS = ("conv1d_glu_residual", "seq_max_pool")


def conv1d_same(x, w):
    """tf.nn.conv1d(x, w, 1, 'SAME'): (k-1)//2 zeros before each sequence, the rest after.  x [B,T,C], w [k,C,O]."""
    k, length = w.shape[0], x.shape[1]
    before = (k - 1) // 2
    padded = torch.nn.functional.pad(x, (0, 0, before, k - 1 - before))
    out = 0
    for j in range(k):
        out = out + padded[:, j:j + length] @ w[j]
    return out


def conv1d_glu_residual(x, w, b):
    z = conv1d_same(x, w) + b
    f = x.shape[-1]
    return z[..., :f] * torch.sigmoid(z[..., f:]) + x


def encoder(states, variables, layers, prefix=""):
    """(temporal_states, output) of SentenceEncoder; `variables` maps names below the part's scope."""
    v = {n[len(prefix):]: t for n, t in variables.items() if n.startswith(prefix)}
    ordered = states + v["input_projection/order_embeddings"][:states.shape[1]].unsqueeze(0)
    conv = ordered @ v["order_and_embed/kernel"] + v["order_and_embed/bias"]
    for i in range(layers):
        conv = conv1d_glu_residual(conv, v["encoder_conv_{}/convolution_filters".format(i)],
                                   v["encoder_conv_{}/conv_bias".format(i)])
    out = conv + ordered @ v["input_to_final_state/kernel"] + v["input_to_final_state/bias"]
    return out, out.amax(1)


def golden():
    return np.load(GOLDEN)


def golden_variables(g, tag):
    return {str(n): g[tag + "_var:" + str(n)] for n in g[tag + "_variable_names"]}


def golden_model_outputs(g, tag, device):
    """This package's SentenceEncoder for the golden case `tag`, built on `device` with the golden's variables loaded
    BY NAME (the arena must hold exactly the reference's names and shapes), in inference mode.  Returns
    {output name: tensor}.  The caller has pointed ops / runtime at `device`."""
    from neuralmonkey_b200 import runtime
    from neuralmonkey_b200.encoders.facebook_conv import SentenceEncoder
    from neuralmonkey_b200.model.sequence import EmbeddedSequence
    from neuralmonkey_b200.vocabulary import Vocabulary

    feats, layers, width, max_len = SHAPES[tag]

    def dev(name):
        return torch.from_numpy(np.asarray(g[tag + "_" + name])).to(device=device, dtype=torch.float32)

    class Sequence(EmbeddedSequence):
        """The golden's embedded input, fed as it is (no embedding table of its own)."""
        def declare_variables(self):
            pass

        temporal_states = property(lambda self: dev("states"))
        temporal_mask = property(lambda self: dev("mask"))

    runtime.reset()
    emb = int(g[tag + "_states"].shape[2])
    seq = Sequence(name="seq", vocabulary=Vocabulary(["w"]), data_id="source", embedding_size=emb,
                   max_length=max_len)
    part = SentenceEncoder(name=tag, input_sequence=seq, conv_features=feats, encoder_layers=layers,
                           kernel_width=width)
    part.ensure_declared()
    arena = runtime.arena()
    arena.finalize(runtime.device())
    variables = golden_variables(g, tag)
    assert sorted(arena.order) == sorted(variables), (sorted(arena.order), sorted(variables))
    for name, value in variables.items():
        assert tuple(arena.get(name).shape) == value.shape, name
    arena.load_dict({n: torch.from_numpy(v) for n, v in variables.items()})
    return {"temporal_states": part.temporal_states, "output": part.output, "temporal_mask": part.temporal_mask}


# -- the model of tests/bpe.ini, for one training step ---------------------------------------------------------------
BPE_WORDS = ["w{}".format(i) for i in range(14)]


def bpe_batch(seed=0, sentences=6):
    """A batch of `source_bpe` / `target_bpe` token lists of lengths 1 to 10 (bpe.ini's max_length)."""
    rng = np.random.RandomState(seed)

    class Data:
        series = {"source_bpe": [list(rng.choice(BPE_WORDS, size=rng.randint(1, 11))) for _ in range(sentences)],
                  "target_bpe": [list(rng.choice(BPE_WORDS, size=rng.randint(1, 11))) for _ in range(sentences)]}

        def __len__(self):
            return sentences

        def get_series(self, name):
            return self.series[name]

        def maybe_get_series(self, name):
            return self.series.get(name)
    return Data()


def bpe_model(views=False):
    """bpe.ini's encoder_input, encoder, attention, decoder and trainer (l2_weight 1e-8, clip_norm 1.0, Adadelta).
    With `views` the decoder and the attention read the encoder through the gradient-blocking views, as in the
    second command of the reference's tests_run.sh.  The decoder's dropout is off (keep_prob 1), so that one step
    computes the same thing on any device; the encoder ignores its keep_prob as the reference does.  Returns
    (trainer, [model parts in feeding order]) with the variables declared and the arena finalised."""
    from neuralmonkey_b200 import runtime, tf
    from neuralmonkey_b200.attention import Attention
    from neuralmonkey_b200.decoders import Decoder
    from neuralmonkey_b200.encoders.facebook_conv import SentenceEncoder
    from neuralmonkey_b200.model.gradient_blocking import StatefulView, TemporalStatefulView
    from neuralmonkey_b200.model.sequence import EmbeddedSequence
    from neuralmonkey_b200.trainers import CrossEntropyTrainer
    from neuralmonkey_b200.vocabulary import Vocabulary

    vocab = Vocabulary(BPE_WORDS)
    seq = EmbeddedSequence(name="encoder_input", vocabulary=vocab, data_id="source_bpe", embedding_size=11,
                           max_length=10)
    enc = SentenceEncoder(name="sentence_encoder", input_sequence=seq, conv_features=10, encoder_layers=2,
                          dropout_keep_prob=0.5)
    att = Attention(name="attention_sentence_encoder", encoder=TemporalStatefulView(enc) if views else enc,
                    state_size=8)
    dec = Decoder(name="decoder", encoders=[StatefulView(enc) if views else enc], vocabulary=vocab,
                  data_id="target_bpe", embedding_size=10, attentions=[att], dropout_keep_prob=1.0,
                  max_output_len=10)
    optimizer = tf.AdadeltaOptimizer(learning_rate=1e-4, epsilon=1e-6, rho=0.95, name="adadelta")
    trainer = CrossEntropyTrainer(decoders=[dec], l2_weight=1e-8, clip_norm=1.0, optimizer=optimizer)
    _, parameterizeds = trainer.get_dependencies()
    assert enc in parameterizeds
    for part in parameterizeds:
        part.ensure_declared()
    runtime.arena().finalize(runtime.device())
    return trainer, [seq, enc, att, dec]


def feed_bpe(parts, data):
    for part in parts:
        part.feed_dict(data, train=True)
