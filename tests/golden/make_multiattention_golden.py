"""Golden vectors from the reference's own attention combination, `attention/combination.py` (FlatMultiAttention,
HierarchicalMultiAttention over two feed-forward `Attention` children), executed over the numpy TensorFlow
stand-in of tf_numpy_shim.py.

Each case (flat / hier x share_attn_projections x use_sentinels) attends from a temporal encoder (a padded batch,
width 7) and a spatial one (2 x 3 regions, width 4) for three decoder steps, with `attention()` called inside the
decoder's step scope `decoder/attention_decoder` as the reference's decoder calls it (decoders/decoder.py:169,283).
Variables are drawn on demand by the shim and recorded under their full TF names, so what is pinned is the
reference's side: which variables exist and under which scope, their shapes, the logits, the renormalised (flat) or
plain (hierarchical) softmax and the contexts.  The spatial encoder carries an all-ones mask, as a SpatialFiller's.

    python tests/golden/make_multiattention_golden.py   ->  tests/golden/multiattention_golden.npz   (needs /root/reference)
"""
import itertools
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
import tf_numpy_shim as shim  # noqa: E402
from make_convs2s_golden import _install, _part  # noqa: E402

LENGTHS, TEMPORAL_DIM, SPATIAL_DIM, GRID = [5, 3, 1], 7, 4, (2, 3)
RNN, EMB, ATT, STEPS = 6, 6, 8, 3
STEP_SCOPE = "decoder/attention_decoder"
CASES = ["{}_{}_{}".format(kind, "share" if share else "noshare", "sentinel" if sentinel else "nosentinel")
         for kind, share, sentinel in itertools.product(("flat", "hier"), (False, True), (False, True))]


def main():
    tf = _install()
    tf.nn.sigmoid = tf.sigmoid
    from neuralmonkey.attention.combination import FlatMultiAttention, HierarchicalMultiAttention
    from neuralmonkey.attention.feed_forward import Attention
    from neuralmonkey.model.stateful import SpatialStateful, TemporalStateful

    class Text(TemporalStateful):
        def __init__(self, states, mask):
            self._s, self._m = shim.t(states, np.float32), shim.t(mask, np.float32)

        temporal_states = property(lambda self: self._s)
        temporal_mask = property(lambda self: self._m)
        dimension = property(lambda self: TEMPORAL_DIM)

    class Image(SpatialStateful):
        def __init__(self, states):
            self._s = shim.t(states, np.float32)

        spatial_states = property(lambda self: self._s)
        spatial_mask = property(lambda self: shim.t(np.ones(self._s.shape[:3]), np.float32))
        dimension = property(lambda self: SPATIAL_DIM)

    rng = np.random.RandomState(11)
    out = {}
    bsz = len(LENGTHS)
    for tag in CASES:
        kind, share, sentinel = tag.split("_")
        share, sentinel = share == "share", sentinel == "sentinel"
        mask = (np.arange(max(LENGTHS))[None, :] < np.array(LENGTHS)[:, None]).astype(np.float32)
        text = (rng.randn(bsz, max(LENGTHS), TEMPORAL_DIM) * mask[..., None]).astype(np.float32)
        image = rng.randn(bsz, GRID[0], GRID[1], SPATIAL_DIM).astype(np.float32)
        queries = rng.randn(STEPS, bsz, RNN).astype(np.float32)
        prev = rng.randn(STEPS, bsz, RNN).astype(np.float32)
        inputs = rng.randn(STEPS, bsz, EMB).astype(np.float32)
        shim.VARIABLES.clear()
        shim.AUTO[0] = np.random.RandomState(rng.randint(1 << 30))
        enc_text, enc_image = Text(text, mask), Image(image)
        common = dict(attentions_in_time=[], attention_state_size=ATT, _share_projections=share,
                      _use_sentinels=sentinel, att_scope_name="attention_combination", batch_size=bsz,
                      histories={})
        children = []
        if kind == "flat":
            wrapper = _part(FlatMultiAttention, "combination", _encoders=[enc_text, enc_image], **common)
        else:
            children = [_part(Attention, "att_text", encoder=enc_text, dropout_keep_prob=1.0, _state_size=5, batch_size=bsz),
                        _part(Attention, "att_image", encoder=enc_image, dropout_keep_prob=1.0, _state_size=None,
                              batch_size=bsz)]
            wrapper = _part(HierarchicalMultiAttention, "combination", attentions=children, **common)
        state = wrapper.initial_loop_state()
        contexts = []
        for step in range(STEPS):
            with tf.variable_scope(STEP_SCOPE):
                ctx, state = wrapper.attention(shim.t(queries[step], np.float32), shim.t(prev[step], np.float32),
                                               shim.t(inputs[step], np.float32), state)
            contexts.append(np.asarray(ctx, np.float32))
        weights = state.weights if kind == "flat" else state.loop_state.weights
        for name, value in (("text", text), ("mask", mask), ("image", image), ("queries", queries),
                            ("prev", prev), ("inputs", inputs), ("contexts", np.stack(contexts)),
                            ("weights", np.asarray(weights, np.float32))):
            out[tag + "_" + name] = value
        out[tag + "_variable_names"] = np.array(sorted(shim.VARIABLES))
        for name in sorted(shim.VARIABLES):
            out[tag + "_var:" + name] = np.asarray(shim.VARIABLES[name], np.float32)
    np.savez_compressed(os.path.join(HERE, "multiattention_golden.npz"), **out)


if __name__ == "__main__":
    main()
