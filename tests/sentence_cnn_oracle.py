"""fp64 restatement of the character-level sentence encoder (encoders/sentence_cnn_encoder.py of the reference,
DESIGN.md §7d), with every gradient through torch.autograd, pinned to tests/golden/sentence_cnn_golden.npz (made by
tests/golden/make_sentence_cnn_golden.py from the reference's own class).  `conv1d`, `pool2d` and `highway_gate`
also stand in for the `ops` functions of the same names on the CPU."""
import os
from typing import Dict

import numpy as np
import torch
import torch.nn.functional as F

from oracle import nm_oracle as O
from tests.cnn_oracle import pool2d

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "sentence_cnn_golden.npz")
CASES = ("t12_s5", "t10_s5", "s1", "s_gt_t", "dropout")
OUTPUTS = ("cnn_encoded", "highway_layer", "temporal_states", "output", "temporal_mask")
STAND_INS = ("conv1d", "pool2d", "highway_gate")
SCOPE = "sentence_encoder"


def golden():
    return np.load(GOLDEN)


def config(g, tag):
    """(segment_size, highway_depth, rnn_size, filters, keep_prob, train) of a golden case."""
    s, depth, rnn, keep, train = g[tag + "_config"]
    return int(s), int(depth), int(rnn), [tuple(int(v) for v in f) for f in g[tag + "_filters"]], float(keep), \
        bool(train)


def golden_variables(g, tag) -> Dict[str, np.ndarray]:
    prefix = tag + "_var:"
    return {k[len(prefix):]: g[k] for k in g.files if k.startswith(prefix)}


def feature_dropout_mask(shape, keep_prob):
    """tf_numpy_shim.feature_dropout_mask: every second entry of the last axis dropped, the rest scaled."""
    pattern = torch.from_numpy(np.where(np.arange(int(shape[-1])) % 2 == 0, 1.0 / keep_prob, 0.0))
    return pattern.expand(tuple(int(d) for d in shape)).clone()


def conv1d(x, w, b, padding="same", act=None):
    """tf.nn.conv1d(x, w, 1, 'SAME') + b, then act: x [B,T,Cin], w [k,Cin,Cout]."""
    assert padding == "same"
    k = w.shape[0]
    before = (k - 1) // 2
    xp = F.pad(x.transpose(1, 2), (before, k - 1 - before))
    y = F.conv1d(xp, w.permute(2, 1, 0)).transpose(1, 2)
    if b is not None:
        y = y + b
    return torch.relu(y) if act == "relu" else y


def highway_gate(zh, zt, x):
    t = torch.sigmoid(zt)
    return torch.relu(zh) * t + x * (1.0 - t)


def segment_max(x, s):
    """tf.nn.max_pool over time, ksize = strides = s, SAME."""
    return pool2d(x.unsqueeze(2), s, s, "same", "max").squeeze(2)


def encoder(v: Dict[str, torch.Tensor], states, mask, s, depth, filters, keep=1.0, train=False):
    """The reference's SentenceCNNEncoder over states [B,T,E] / mask [B,T]; v maps local variable names (no part
    scope) to tensors.  Returns {output name: tensor}."""
    x = states * feature_dropout_mask(states.shape, keep).to(states) if train and keep < 1.0 else states
    pooled = [segment_max(conv1d(x, v["conv-maxpool-{}/conv_W".format(w)], v["conv-maxpool-{}/conv_bias".format(w)],
                                 "same", "relu"), s) for w, _ in filters]
    cnn = torch.cat(pooled, 2)
    layer = cnn.reshape(-1, cnn.shape[-1])
    for i in range(depth):
        pre = "highway_layer_{}/".format(i)
        layer = highway_gate(layer @ v[pre + "weight_H"] + v[pre + "bias_H"],
                             layer @ v[pre + "weight_T"] + v[pre + "bias_T"], layer)
    hw = layer.view(cnn.shape)
    lens = torch.ceil(mask.sum(1) / s).to(torch.int64)

    def cell(direction):
        pre = "bidirectional_rnn/{}/OrthoGRUCell/".format(direction)
        return [v[pre + n] for n in ("gates/kernel", "gates/bias", "candidate/kernel", "candidate/bias")]
    out_fw, fin_fw = O.dynamic_gru(hw, lens, *cell("fw"))
    out_bw, fin_bw = O.dynamic_gru(O.reverse_sequence(hw, lens), lens, *cell("bw"))
    out_bw = O.reverse_sequence(out_bw, lens)
    return {"cnn_encoded": cnn, "highway_layer": hw, "temporal_states": torch.cat([out_fw, out_bw], 2),
            "output": torch.cat([fin_fw, fin_bw], 1), "temporal_mask": segment_max(mask.unsqueeze(-1), s).squeeze(-1)}


def probes(g, tag):
    """Fixed weights of the scalar whose gradients the tests compare: sum(temporal_states * p0) + sum(output * p1)."""
    rng = np.random.RandomState(7)
    return (torch.from_numpy(rng.randn(*g[tag + "_temporal_states"].shape)),
            torch.from_numpy(rng.randn(*g[tag + "_output"].shape)))


def oracle_case(g, tag):
    """The restatement at fp64 over the golden's inputs and variables: (outputs, {variable name: gradient},
    gradient of the input states)."""
    s, depth, _rnn, filters, keep, train = config(g, tag)
    v = {n.split("/", 1)[1]: torch.from_numpy(a).double().requires_grad_(True)
         for n, a in golden_variables(g, tag).items()}
    states = torch.from_numpy(g[tag + "_states"]).double().requires_grad_(True)
    mask = torch.from_numpy(g[tag + "_mask"]).double()
    out = encoder(v, states, mask, s, depth, filters, keep, train)
    p0, p1 = probes(g, tag)
    loss = (out["temporal_states"] * p0).sum() + (out["output"] * p1).sum()
    names = sorted(v)
    grads = torch.autograd.grad(loss, [v[n] for n in names] + [states])
    return ({k: t.detach() for k, t in out.items()},
            {SCOPE + "/" + n: gr for n, gr in zip(names, grads[:-1])}, grads[-1])


def model_case(g, tag, device):
    """This package's SentenceCNNEncoder for the golden case `tag` on `device`, the golden's variables loaded BY NAME
    (the arena must hold exactly the reference's names and shapes), with the golden's train mode.  Returns (outputs,
    {variable name: gradient}, gradient of the input states) of the same scalar as `oracle_case`.  The caller has
    pointed ops / runtime at `device` and, for the dropout case, patched in the deterministic mask."""
    from neuralmonkey_b200 import runtime
    from neuralmonkey_b200.encoders import SentenceCNNEncoder
    from neuralmonkey_b200.model.sequence import Sequence

    states = torch.from_numpy(g[tag + "_states"]).to(device).requires_grad_(True)
    mask = torch.from_numpy(g[tag + "_mask"]).to(device)

    class Inputs(Sequence):
        temporal_states = property(lambda self: states)
        temporal_mask = property(lambda self: mask)
        dimension = property(lambda self: int(states.shape[2]))

    s, depth, rnn, filters, keep, train = config(g, tag)
    runtime.reset()
    part = SentenceCNNEncoder(name=SCOPE, input_sequence=Inputs("inputs"), segment_size=s, highway_depth=depth,
                              rnn_size=rnn, filters=filters, dropout_keep_prob=keep)
    part.train_mode = train
    part.ensure_declared()
    arena = runtime.arena()
    arena.finalize(runtime.device())
    variables = golden_variables(g, tag)
    assert sorted(arena.order) == sorted(variables), (sorted(arena.order), sorted(variables))
    for name, value in variables.items():
        assert tuple(arena.get(name).shape) == value.shape, name
    arena.load_dict({n: torch.from_numpy(a) for n, a in variables.items()})
    arena.zero_grad()
    out = {name: getattr(part, name) for name in OUTPUTS}
    p0, p1 = (p.to(device=device, dtype=torch.float32) for p in probes(g, tag))
    loss = (out["temporal_states"] * p0).sum() + (out["output"] * p1).sum()
    loss.backward()
    arena.fold_autograd_grads()
    grads = arena.named_grads()
    return ({k: t.detach().double().cpu() for k, t in out.items()}, grads, states.grad.double().cpu())


# -- a model of tests/small_sent_cnn.ini's shape, for the training-step tests ---------------------------------------------
def build_ini_model(views=False, l2_weight=1.0e-8):
    """tests/small_sent_cnn.ini's encoder, attention, decoder and trainer (dropout off, so two runs match); with
    `views` the attention and the decoder read the encoder through the gradient-blocking views."""
    from neuralmonkey_b200 import runtime, tf
    from neuralmonkey_b200.attention import Attention
    from neuralmonkey_b200.decoders import Decoder
    from neuralmonkey_b200.encoders import SentenceCNNEncoder
    from neuralmonkey_b200.model.gradient_blocking import StatefulView, TemporalStatefulView
    from neuralmonkey_b200.model.sequence import EmbeddedSequence
    from neuralmonkey_b200.trainers import CrossEntropyTrainer
    from neuralmonkey_b200.vocabulary import Vocabulary
    runtime.reset()
    chars = Vocabulary([chr(c) for c in range(97, 123)])
    seq = EmbeddedSequence(name="encoder_input", vocabulary=chars, data_id="source_chars", embedding_size=11,
                           max_length=10)
    enc = SentenceCNNEncoder(name="sentence_encoder", input_sequence=seq, rnn_size=7, highway_depth=3,
                             filters=[(1, 13), (2, 13), (3, 13)], segment_size=5)
    att = Attention(name="attention_sentence_encoder", encoder=TemporalStatefulView(enc) if views else enc)
    dec = Decoder(name="decoder", encoders=[StatefulView(enc) if views else enc], rnn_size=9, embedding_size=9,
                  attentions=[att], data_id="target_chars", max_output_len=10, vocabulary=chars)
    trainer = CrossEntropyTrainer(decoders=[dec], l2_weight=l2_weight, clip_norm=1.0,
                                  optimizer=tf.AdamOptimizer(learning_rate=1e-3))
    for part in trainer.parameterizeds:
        part.ensure_declared()
    runtime.arena().finalize(runtime.device())
    return {"seq": seq, "enc": enc, "att": att, "dec": dec, "trainer": trainer, "arena": runtime.arena()}


def ini_batch(g):
    """Six character sequences of lengths 10, 5, 9, 1, 6, 3 and targets ending in </s>."""
    src = torch.randint(4, 30, (6, 10), generator=g)
    tgt = torch.randint(4, 30, (6, 8), generator=g)
    for b, (ls, lt) in enumerate([(10, 7), (5, 3), (9, 7), (1, 1), (6, 4), (3, 2)]):
        src[b, ls:] = 0
        tgt[b, lt] = 2
        tgt[b, lt + 1:] = 0
    return src, tgt


def feed_ini_model(model, src, tgt, train):
    model["seq"].feed_ids([src], train=train)
    for part in (model["enc"], model["att"]):
        part.reset_batch()
        part.train_mode = train
        part.batch_size = src.shape[0]
    model["dec"].feed_ids(tgt, src.shape[0], train=train)


def ini_step(params, src, tgt, **kwargs):
    """One training step of `build_ini_model(**kwargs)` from `params`: (loss, variables after the step on the CPU)."""
    model = build_ini_model(**kwargs)
    model["arena"].load_dict(params)
    feed_ini_model(model, src, tgt, True)
    loss = float(model["trainer"].train_step()["losses"][0])
    return loss, {n: v.detach().cpu().clone() for n, v in model["arena"].state_dict().items()}
