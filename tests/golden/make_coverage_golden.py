"""Golden vectors from the reference's own coverage attention, `attention/coverage.py` (CoverageAttention), executed
over the numpy TensorFlow stand-in of tf_numpy_shim.py.

Each case attends from a temporal encoder (a padded batch, width 7) for four decoder steps, with `attention()`
called inside the decoder's step scope `decoder/attention_decoder` as the reference's decoder calls it
(decoders/decoder.py:169,283).  Variables are drawn on demand by the shim and recorded under their full TF names,
so what is pinned is the reference's side: which variables exist (no `attn_bias`: `get_energies` never reads it),
their shapes, the fertility, the energies, the renormalised weights and the contexts of every step.  The cases
differ in `max_fertility` and `state_size`.

The reference's `get_energies` asks the loop state's weights for `size()` (coverage.py:52-56), which a TensorFlow
tensor does not have; the weights handed to each step here are a view of the shim's tensor type that has it, the
element count, which is what the expression means.  Nothing in the reference or the shim is changed.

    python tests/golden/make_coverage_golden.py   ->  tests/golden/coverage_golden.npz   (needs /root/reference)
"""
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
import tf_numpy_shim as shim  # noqa: E402
from make_convs2s_golden import _install, _part  # noqa: E402

LENGTHS, DIM, RNN, STEPS = [5, 3, 1], 7, 6, 4
STEP_SCOPE = "decoder/attention_decoder"
CASES = {"fert5": dict(max_fertility=5, state_size=None), "fert2_state5": dict(max_fertility=2, state_size=5)}


class _Sized(shim.T):
    def size(self):     # pylint: disable=invalid-overridden-method
        return int(np.prod(np.ndarray.__getattribute__(self, "shape")))


def main():
    tf = _install()
    tf.greater = lambda a, b: np.asarray(a) > np.asarray(b)
    tf.cond = lambda pred, true_fn, false_fn: true_fn() if bool(pred) else false_fn()
    from neuralmonkey.attention.coverage import CoverageAttention
    from neuralmonkey.model.stateful import TemporalStateful

    class Text(TemporalStateful):
        def __init__(self, states, mask):
            self._s, self._m = shim.t(states, np.float32), shim.t(mask, np.float32)

        temporal_states = property(lambda self: self._s)
        temporal_mask = property(lambda self: self._m)
        dimension = property(lambda self: DIM)

    rng = np.random.RandomState(17)
    out = {}
    bsz = len(LENGTHS)
    for tag, case in sorted(CASES.items()):
        mask = (np.arange(max(LENGTHS))[None, :] < np.array(LENGTHS)[:, None]).astype(np.float32)
        text = (rng.randn(bsz, max(LENGTHS), DIM) * mask[..., None]).astype(np.float32)
        queries = rng.randn(STEPS, bsz, RNN).astype(np.float32)
        shim.VARIABLES.clear()
        shim.AUTO[0] = np.random.RandomState(rng.randint(1 << 30))
        att = _part(CoverageAttention, "coverage", encoder=Text(text, mask), dropout_keep_prob=1.0,
                    _state_size=case["state_size"], max_fertility=case["max_fertility"], batch_size=bsz,
                    histories={})
        energies = []
        get_energies = att.get_energies

        def recording(y, weights_in_time, get_energies=get_energies, energies=energies):
            e = get_energies(y, weights_in_time)
            energies.append(np.asarray(e, np.float32))
            return e
        att.get_energies = recording
        state = att.initial_loop_state()
        contexts = []
        for step in range(STEPS):
            state = state._replace(weights=np.asarray(state.weights).view(_Sized))
            with tf.variable_scope(STEP_SCOPE):
                ctx, state = att.attention(shim.t(queries[step], np.float32), None, None, state)
            contexts.append(np.asarray(ctx, np.float32))
        for name, value in (("text", text), ("mask", mask), ("queries", queries),
                            ("fertility", np.asarray(att.fertility, np.float32)),
                            ("energies", np.stack(energies)), ("contexts", np.stack(contexts)),
                            ("weights", np.asarray(state.weights, np.float32))):
            out[tag + "_" + name] = value
        out[tag + "_max_fertility"] = np.array(case["max_fertility"])
        out[tag + "_variable_names"] = np.array(sorted(shim.VARIABLES))
        for name in sorted(shim.VARIABLES):
            out[tag + "_var:" + name] = np.asarray(shim.VARIABLES[name], np.float32)
    np.savez_compressed(os.path.join(HERE, "coverage_golden.npz"), **out)


if __name__ == "__main__":
    main()
