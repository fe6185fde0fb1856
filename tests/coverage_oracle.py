"""Restatement of the reference's coverage attention (attention/coverage.py over feed_forward.py:125-166) and the CPU
stand-ins of `ops.coverage_fertility` / `ops.coverage_attention`, plus a small decoder over seeded encoder states for
the model-part tests.

The functions work in any dtype: in fp64 they are the yardstick of the kernel tests, in fp32 the stand-ins the host
tests swap in for the ops.  `coverage_attention` steps the way the reference's `attention()` does: each step sums the
weights of the steps before it, and the weights stay differentiable inside the scan."""
import os

import numpy as np
import torch

STAND_INS = ("coverage_attention", "coverage_fertility")
GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "coverage_golden.npz")
CASES = ("fert2_state5", "fert5")


def coverage_fertility(states, fertility_w, max_fertility):
    return 1e-8 + max_fertility * torch.sigmoid((states * fertility_w).sum(-1))


def step(keys, values, mask, fert, y, v, coverage_w, weight_sum):
    """One `attention()` step from the sum of the earlier weights (None before the first step): y [B, A] ->
    (context [B, C], weights [B, Tx], energies [B, Tx])."""
    cov = (torch.zeros_like(fert) if weight_sum is None else weight_sum) / fert
    if mask is not None:
        cov = cov * mask
    e = (v * torch.tanh(keys + y.unsqueeze(1) + coverage_w * cov.unsqueeze(-1))).sum(-1)
    w = torch.softmax(e, dim=-1)
    if mask is not None:
        w = w * mask
        w = w / (w.sum(-1, keepdim=True) + 1e-8)
    return (w.unsqueeze(-1) * values).sum(1), w, e


def coverage_attention(keys, values, mask, fert, qproj, v, coverage_w, cov_in=None):
    total = cov_in
    contexts, weights = [], []
    for q in range(qproj.shape[1]):
        ctx, w, _ = step(keys, values, mask, fert, qproj[:, q], v, coverage_w, total)
        total = w if total is None else total + w
        contexts.append(ctx)
        weights.append(w)
    return torch.stack(contexts, 1), torch.stack(weights, 1).detach(), total


# -- the golden of the reference's own coverage.py (tests/golden/make_coverage_golden.py) ---------------------------
def golden():
    return np.load(GOLDEN)


def golden_variables(g, tag):
    return {str(n): g[tag + "_var:" + str(n)] for n in g[tag + "_variable_names"]}


def restated_golden(g, tag):
    """(fertility [B, Tx], per step: contexts, weights, energies) from the golden's inputs and variables in fp64."""
    var = {n: torch.from_numpy(x).double() for n, x in golden_variables(g, tag).items()}

    def arr(name):
        return torch.from_numpy(np.asarray(g[tag + "_" + name])).double()
    text, mask, queries = arr("text"), arr("mask"), arr("queries")
    keys = text @ var["coverage/attn_key_projection"]
    fert = coverage_fertility(text, var["coverage/fertility_matrix"].reshape(-1), float(g[tag + "_max_fertility"]))
    total, out = None, []
    for q in range(queries.shape[0]):
        y = queries[q] @ var["coverage/Attention/attn_query_projection"] + var["coverage/attn_projection_bias"]
        ctx, w, e = step(keys, text, mask, fert, y, var["coverage/attn_similarity_v"],
                         var["coverage/coverage_matrix"].reshape(-1), total)
        total = w if total is None else total + w
        out.append((ctx, w, e))
    return fert, out


# -- a small decoder ----------------------------------------------------------------------------------------------
WORDS = ["w{}".format(i) for i in range(9)]
LENGTHS = [5, 3, 1]
DIM = 7


def encoder_states(seed=0):
    rng = np.random.RandomState(seed)
    mask = (np.arange(max(LENGTHS))[None, :] < np.array(LENGTHS)[:, None]).astype(np.float32)
    text = (rng.randn(len(LENGTHS), max(LENGTHS), DIM) * mask[..., None]).astype(np.float32)
    return text, mask


def build_model(seed=0, rnn_size=6, embedding_size=6, state_size=None, max_fertility=5, rnn_cell="GRU",
                conditional_gru=False, states=None, dropout_keep_prob=1.0):
    """A decoder with one CoverageAttention over a padded temporal encoder; `states` = (text, mask) overrides the
    seeded encoder states.  Returns (decoder, attention) with the variables declared and the arena finalised on
    runtime.device()."""
    from neuralmonkey_b200 import runtime
    from neuralmonkey_b200.attention import CoverageAttention
    from neuralmonkey_b200.decoders import Decoder
    from neuralmonkey_b200.model.model_part import ModelPart
    from neuralmonkey_b200.model.stateful import TemporalStatefulWithOutput
    from neuralmonkey_b200.vocabulary import Vocabulary

    text, mask = encoder_states(seed) if states is None else states
    dev = runtime.device()

    class Text(ModelPart, TemporalStatefulWithOutput):
        temporal_states = property(lambda self: torch.from_numpy(text).to(dev))
        temporal_mask = property(lambda self: torch.from_numpy(mask).to(dev))
        output = property(lambda self: torch.from_numpy(text.sum(1) / mask.sum(1, keepdims=True)).to(dev))
        dimension = DIM

    runtime.reset()
    enc = Text("text")
    att = CoverageAttention(name="coverage", encoder=enc, state_size=state_size, max_fertility=max_fertility)
    dec = Decoder(encoders=[enc], vocabulary=Vocabulary(WORDS), data_id="target", name="decoder",
                  max_output_len=4, embedding_size=embedding_size, rnn_size=rnn_size, attentions=[att],
                  rnn_cell=rnn_cell, conditional_gru=conditional_gru, dropout_keep_prob=dropout_keep_prob)
    _, parts = dec.get_dependencies()
    for part in parts:
        part.ensure_declared()
    runtime.arena().finalize(runtime.device())
    return dec, att


def target_ids(seed=0):
    from neuralmonkey_b200.vocabulary import Vocabulary, pad_batch
    rng = np.random.RandomState(seed + 1)
    sentences = [list(rng.choice(WORDS, size=n)) for n in (3, 4, 2)]
    return Vocabulary(WORDS).strings_to_indices(pad_batch(sentences, 4, add_start_symbol=False, add_end_symbol=True))


def feed(dec, att, train, ids=None):
    for part in (dec, att):
        part.reset_batch()
        part.train_mode = train
    dec.feed_ids(ids, att.encoder.temporal_states.shape[0], train=train)


def randomize(scale=0.5, seed=3):
    from neuralmonkey_b200 import runtime
    gen = torch.Generator().manual_seed(seed)
    with torch.no_grad():
        for name in runtime.arena().order:
            t = runtime.arena().get(name)
            t.copy_((torch.randn(t.shape, generator=gen) * scale).to(t.device))
