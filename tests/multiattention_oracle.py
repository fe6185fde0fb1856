"""Restatement of the reference's attention combination (attention/combination.py) and the CPU stand-in of
`ops.joint_attention`, plus a small multi-source decoder over seeded encoder states for the model-part tests.

`joint_attention` works in any dtype: in fp64 it is the yardstick of the kernel tests, in fp32 the stand-in the
host tests swap in for the op.  `flat_step` / `hier_step` restate the reference's per-step `attention()` with its
own concatenations and renormalised softmax, from variables fetched by their full names."""
import os

import numpy as np
import torch

STAND_INS = ("joint_attention",)
GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "multiattention_golden.npz")
CASES = ["{}_{}_{}".format(kind, share, sentinel) for kind in ("flat", "hier") for share in ("noshare", "share")
         for sentinel in ("nosentinel", "sentinel")]
STEP = "decoder/attention_decoder"


def joint_attention(keys, values, mask, seg_ends, seg_bias, ckeys, cvalues, cand_bias, qproj, v):
    energies, vals = [], []
    if keys is not None:
        bias = torch.cat([seg_bias[s].expand(e - (seg_ends[s - 1] if s else 0)) for s, e in enumerate(seg_ends)])
        energies.append((v * torch.tanh(keys.unsqueeze(1) + qproj.unsqueeze(2))).sum(-1) + bias)
    if ckeys is not None:
        energies.append((v * torch.tanh(ckeys + qproj.unsqueeze(2))).sum(-1) + cand_bias)
    e = torch.cat(energies, -1)
    w = torch.softmax(e, dim=-1)
    if mask is not None:
        j = ckeys.shape[2] if ckeys is not None else 0
        m = torch.cat([mask, mask.new_ones(mask.shape[0], j)], 1).unsqueeze(1)
        w = w * m
        w = w / (w.sum(-1, keepdim=True) + 1e-8)
    ctx = 0
    tx = keys.shape[1] if keys is not None else 0
    if keys is not None:
        ctx = ctx + torch.einsum("bqt,btc->bqc", w[..., :tx], values)
    if ckeys is not None:
        ctx = ctx + torch.einsum("bqj,bqjc->bqc", w[..., tx:], cvalues)
    return ctx, w


# -- the reference's per-step attention(), restated ------------------------------------------------------------------
def _dense(var, x, scope):
    return x @ var(scope + "/kernel") + var(scope + "/bias")


def _vector_logit(var, step, proj_state, value, scope, share):
    """(context projection [B, A], logit [B]) of `_vector_logit` (combination.py:74-103)."""
    key = _dense(var, value, "{}/{}_logit/vector_projection".format(step, scope))
    logit = (var("attn_v")[0, 0] * torch.tanh(proj_state + key)).sum(-1) + var("{}/{}_logit/vector_bias".format(
        step, scope))
    ctx = key if share else _dense(var, value, "{}/{}_logit/vector_ctx_proj".format(step, scope))
    return ctx, logit


def _sentinel(var, step, query, prev, inp):
    gate = torch.sigmoid(_dense(var, torch.cat([prev, inp], 1), step + "/sentinel/dense"))
    return gate * query


def flat_step(var, step, states, masks, query, prev, inp, share, sentinel):
    """FlatMultiAttention.attention (combination.py:240-321) for one query per row.  `var(name)` returns a
    variable below the attention's scope, or below the decoder's step scope for names starting with `step`."""
    proj_state = _dense(var, query, step + "/dense")
    logits, ctx_projs = [], []
    for i, st in enumerate(states):
        key = st @ var("logits_projections/proj_matrix_{}".format(i)) + var("logits_projections/proj_bias_{}".format(i))
        logits.append((var("attn_v")[0, 0] * torch.tanh(proj_state.unsqueeze(1) + key)).sum(-1)
                      + var("attn_bias_{}".format(i)))
        ctx_projs.append(key if share else st @ var("context_projections/proj_matrix_{}".format(i))
                         + var("context_projections/proj_bias_{}".format(i)))
    masks = list(masks)
    if sentinel:
        value = _sentinel(var, step, query, prev, inp)
        ctx, logit = _vector_logit(var, step, proj_state, value, "sentinel", share)
        logits.append(logit.unsqueeze(1))
        ctx_projs.append(ctx.unsqueeze(1))
        masks.append(torch.ones_like(masks[0][:, :1]))
    soft = torch.softmax(torch.cat(logits, 1), -1) * torch.cat(masks, 1)
    att = soft / (soft.sum(1, keepdim=True) + 1e-8)
    return (att.unsqueeze(2) * torch.cat(ctx_projs, 1)).sum(1), att


def hier_step(var, step, child_names, child_contexts, query, prev, inp, share, sentinel):
    """HierarchicalMultiAttention.attention (combination.py:394-463) given the children's contexts."""
    proj_state = _dense(var, query, step + "/dense")
    ctxs, logits = [], []
    for name, c in zip(child_names, child_contexts):
        ctx, logit = _vector_logit(var, step, proj_state, c, name, share)
        ctxs.append(ctx if share else _dense(var, c, "{}/proj_attn_{}".format(step, name)))
        logits.append(logit)
    if sentinel:
        value = _sentinel(var, step, query, prev, inp)
        ctx, logit = _vector_logit(var, step, proj_state, value, "sentinel", share)
        ctxs.append(ctx if share else _dense(var, value, step + "/proj_sentinel"))
        logits.append(logit)
    att = torch.softmax(torch.stack(logits, 1), -1)
    return (att.unsqueeze(2) * torch.stack(ctxs, 1)).sum(1), att


# -- a small multi-source decoder -------------------------------------------------------------------------------------
WORDS = ["w{}".format(i) for i in range(9)]
LENGTHS = [5, 3, 1]          # the temporal encoder's padded batch
TEMPORAL_DIM, SPATIAL_DIM, GRID = 7, 4, (2, 3)


def encoder_states(seed=0):
    rng = np.random.RandomState(seed)
    mask = (np.arange(max(LENGTHS))[None, :] < np.array(LENGTHS)[:, None]).astype(np.float32)
    text = (rng.randn(len(LENGTHS), max(LENGTHS), TEMPORAL_DIM) * mask[..., None]).astype(np.float32)
    image = rng.randn(len(LENGTHS), GRID[0], GRID[1], SPATIAL_DIM).astype(np.float32)
    return text, mask, image


def build_model(kind, share, sentinel, seed=0, rnn_size=6, embedding_size=6, attention_state_size=8, states=None):
    """A GRU decoder over one temporal and one spatial encoder joined by a `kind` ("flat" / "hier") combination;
    `states` = (text, mask, image) overrides the seeded encoder states.  Returns (decoder, wrapper, children) with
    the variables declared and the arena finalised on runtime.device()."""
    from neuralmonkey_b200 import runtime
    from neuralmonkey_b200.attention import Attention
    from neuralmonkey_b200.attention.combination import FlatMultiAttention, HierarchicalMultiAttention
    from neuralmonkey_b200.decoders import Decoder
    from neuralmonkey_b200.model.model_part import ModelPart
    from neuralmonkey_b200.model.stateful import SpatialStateful, TemporalStatefulWithOutput
    from neuralmonkey_b200.vocabulary import Vocabulary

    text, mask, image = encoder_states(seed) if states is None else states
    dev = runtime.device()

    class Text(ModelPart, TemporalStatefulWithOutput):
        temporal_states = property(lambda self: torch.from_numpy(text).to(dev))
        temporal_mask = property(lambda self: torch.from_numpy(mask).to(dev))
        output = property(lambda self: torch.from_numpy(text.sum(1) / mask.sum(1, keepdims=True)).to(dev))
        dimension = TEMPORAL_DIM

    class Image(ModelPart, SpatialStateful):
        spatial_states = property(lambda self: torch.from_numpy(image).to(dev))
        spatial_mask = None
        dimension = SPATIAL_DIM

    runtime.reset()
    enc_text, enc_image = Text("text"), Image("image")
    children = []
    if kind == "flat":
        wrapper = FlatMultiAttention(name="combination", encoders=[enc_text, enc_image],
                                     attention_state_size=attention_state_size, share_attn_projections=share,
                                     use_sentinels=sentinel)
    else:
        children = [Attention(name="att_text", encoder=enc_text, state_size=5),
                    Attention(name="att_image", encoder=enc_image)]
        wrapper = HierarchicalMultiAttention(name="combination", attentions=children,
                                             attention_state_size=attention_state_size, use_sentinels=sentinel,
                                             share_attn_projections=share)
    dec = Decoder(encoders=[enc_text], vocabulary=Vocabulary(WORDS), data_id="target", name="decoder",
                  max_output_len=4, embedding_size=embedding_size, rnn_size=rnn_size, attentions=[wrapper])
    _, parts = dec.get_dependencies()
    for part in parts:
        part.ensure_declared()
    runtime.arena().finalize(runtime.device())
    return dec, wrapper, children


def target_ids(seed=0):
    from neuralmonkey_b200.vocabulary import Vocabulary, pad_batch
    rng = np.random.RandomState(seed + 1)
    sentences = [list(rng.choice(WORDS, size=n)) for n in (3, 4, 2)]
    return Vocabulary(WORDS).strings_to_indices(pad_batch(sentences, 4, add_start_symbol=False, add_end_symbol=True))


def feed(dec, parts, train, ids=None):
    for part in parts:
        part.reset_batch()
        part.train_mode = train
    dec.feed_ids(ids, len(LENGTHS), train=train)


# -- the golden of the reference's own combination.py (tests/golden/make_multiattention_golden.py) ----------------------
def golden():
    return np.load(GOLDEN)


def golden_variables(g, tag):
    return {str(n): g[tag + "_var:" + str(n)] for n in g[tag + "_variable_names"]}


def case_flags(tag):
    kind, share, sentinel = tag.split("_")
    return kind, share == "share", sentinel == "sentinel"


def restated_golden_step(g, tag, step):
    """flat_step / hier_step over the golden's variables, fetched by their full TF names (fp64)."""
    kind, share, sentinel = case_flags(tag)
    variables = {n: torch.from_numpy(v).double() for n, v in golden_variables(g, tag).items()}

    def var(name):
        return variables[STEP + "/attention_combination" + name[4:] if name.startswith("step/")
                         else "combination/" + name]

    def arr(name):
        return torch.from_numpy(np.asarray(g[tag + "_" + name])).double()
    query, prev, inp = arr("queries")[step], arr("prev")[step], arr("inputs")[step]
    text, mask, image = arr("text"), arr("mask"), arr("image")
    if kind == "flat":
        states = [text, image.reshape(image.shape[0], -1, image.shape[3])]
        masks = [mask, torch.ones(image.shape[0], states[1].shape[1], dtype=torch.float64)]
        return flat_step(var, "step", states, masks, query, prev, inp, share, sentinel)
    child_ctx = []
    for name, states, m in (("att_text", text, mask),
                            ("att_image", image.reshape(image.shape[0], -1, image.shape[3]), None)):
        keys = states @ variables[name + "/attn_key_projection"]
        y = query @ variables[name + "/Attention/attn_query_projection"] + variables[name + "/attn_projection_bias"]
        e = (variables[name + "/attn_similarity_v"] * torch.tanh(keys + y.unsqueeze(1))).sum(-1) \
            + variables[name + "/attn_bias"]
        w = torch.softmax(e, -1)
        if m is not None:
            w = w * m
            w = w / (w.sum(-1, keepdim=True) + 1e-8)
        child_ctx.append((w.unsqueeze(-1) * states).sum(1))
    return hier_step(var, "step", ["att_text", "att_image"], child_ctx, query, prev, inp, share, sentinel)


def golden_model(g, tag):
    """This package's wrapper for the golden case `tag` on runtime.device(), with the golden's variables loaded BY
    NAME: every variable of the wrapper and its children must be one of the reference's, of the same shape.
    Returns (decoder, wrapper, children) fed in inference mode."""
    from neuralmonkey_b200 import runtime
    kind, share, sentinel = case_flags(tag)
    states = tuple(np.asarray(g[tag + "_" + n]) for n in ("text", "mask", "image"))
    dec, wrapper, children = build_model(kind, share, sentinel, states=states)
    arena = runtime.arena()
    variables = golden_variables(g, tag)
    ours = [n for n in arena.order if n.startswith(("combination/", "att_text/", "att_image/",
                                                    STEP + "/attention_combination/"))]
    assert sorted(ours) == sorted(variables), (sorted(ours), sorted(variables))
    for name, value in variables.items():
        if name.startswith("att_"):     # the children are feed-forward Attentions, which keep attn_bias as [1]
            assert arena.get(name).numel() == value.size, name
        else:
            assert tuple(arena.get(name).shape) == value.shape, name
    arena.load_dict({n: torch.from_numpy(v).reshape(arena.get(n).shape) for n, v in variables.items()})
    feed(dec, [wrapper] + children, train=False)
    return dec, wrapper, children
