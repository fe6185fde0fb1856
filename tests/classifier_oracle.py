"""fp64 restatement of the sentence classification / regression maths (encoders/pooling.py, encoders/attentive.py,
encoders/sequence_cnn_encoder.py, decoders/sequence_regressor.py of the reference), differentiated by autograd:
`torch.amax` splits the gradient equally among tied maxima, as TF's reduce_max does.  The same functions, called
with fp32 tensors, are the CPU stand-ins of `ops.seq_max_pool`, `ops.seq_mean_pool`, `ops.attentive_pool`,
`ops.conv1d_max_pool` and `ops.squared_error` (tests/test_host_classifier.py) - TEST INFRASTRUCTURE ONLY."""
import os

import numpy as np
import torch

STAND_INS = ("seq_max_pool", "seq_mean_pool", "attentive_pool", "conv1d_max_pool", "squared_error")


def seq_max_pool(x, mask):
    """reduce_max(x*m + 1e-15*(1-m), axis=1)."""
    if mask is None:
        return x.amax(1)
    if float(mask.sum()) <= 0.5:
        raise ValueError("max pooling over a batch without a single valid position (mask sum <= 0.5)")
    m = mask.to(x.dtype).unsqueeze(-1)
    return (x * m + 1e-15 * (1 - m)).amax(1)


def seq_mean_pool(x, mask):
    m = torch.ones(x.shape[:2], dtype=x.dtype) if mask is None else mask.to(x.dtype)
    return (x * m.unsqueeze(-1)).sum(1) / (m.sum(1, keepdim=True) + 1e-8)


def attentive_pool(energies, mask, states):
    """(weights [B,T,R], weights^T . states [B,R,D])."""
    w = torch.softmax(energies, dim=1)
    if mask is not None:
        w = w * mask.to(w.dtype).unsqueeze(-1)
        w = w / (w.sum(1, keepdim=True) + 1e-8)
    return w, w.transpose(1, 2) @ states


def conv1d_max_pool(x, w, bias):
    """reduce_max(relu(conv1d(x, w, VALID) + bias), axis=1); x [B,T,E], w [width,E,F]."""
    width, e, f = w.shape
    if x.shape[1] < width:
        raise ValueError("the batch is {} positions long, shorter than the filter width {}".format(x.shape[1], width))
    windows = x.unfold(1, width, 1).permute(0, 1, 3, 2)            # [B, L, width, E]
    conv = windows.reshape(x.shape[0], -1, width * e) @ w.reshape(width * e, f) + bias
    return torch.relu(conv).amax(1)


def squared_error(pred, target):
    return ((pred - target.unsqueeze(1)) ** 2).mean()


# -- the golden of tests/golden/make_classifier_golden.py (the reference's own classes over the numpy TF stand-in) --
GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "classifier_golden.npz")
VARIABLE_CASES = ("att_plain", "att_proj", "cnn", "clf_layers", "clf_nolayers", "reg_layers", "reg_nolayers")


def golden():
    return np.load(GOLDEN)


def golden_variables(g, tag):
    return {str(n): g[tag + "_var:" + str(n)] for n in g[tag + "_variable_names"]}


def golden_model_outputs(g, tag, device):
    """This package's model parts for the golden case `tag`, built on `device` with the golden's variables loaded BY
    NAME (the arena must hold exactly the reference's names and shapes), in inference mode.  Returns
    {output name: tensor} under the golden's keys.  The caller has pointed ops / runtime at `device`."""
    from neuralmonkey_b200 import runtime
    from neuralmonkey_b200.decoders.classifier import Classifier
    from neuralmonkey_b200.decoders.sequence_regressor import SequenceRegressor
    from neuralmonkey_b200.encoders.attentive import AttentiveEncoder
    from neuralmonkey_b200.encoders.pooling import SequenceAveragePooling, SequenceMaxPooling
    from neuralmonkey_b200.encoders.sequence_cnn_encoder import SequenceCNNEncoder
    from neuralmonkey_b200.model.stateful import Stateful, TemporalStateful
    from neuralmonkey_b200.vocabulary import Vocabulary

    def dev(name, dtype=torch.float32):
        return torch.from_numpy(np.asarray(g[name])).to(device=device, dtype=dtype)

    class Sequence(TemporalStateful):
        temporal_states = property(lambda self: dev("states"))
        temporal_mask = property(lambda self: dev("mask"))
        dimension = property(lambda self: int(g["states"].shape[2]))

    class Vector(Stateful):
        def __init__(self, key):
            self.key = key

        output = property(lambda self: dev(self.key))
        dimension = property(lambda self: int(g[self.key].shape[1]))

    runtime.reset()
    features = [Vector("features_0"), Vector("features_1")]
    if tag in ("maxpool", "avgpool"):
        cls = SequenceMaxPooling if tag == "maxpool" else SequenceAveragePooling
        return {"output": cls(name=tag, input_sequence=Sequence()).output}
    if tag.startswith("att"):
        proj = tag == "att_proj"
        part = AttentiveEncoder(name=tag, input_sequence=Sequence(), hidden_size=4, num_heads=3,
                                output_size=7 if proj else None, state_proj_size=3 if proj else None)
    elif tag == "cnn":
        # the golden's table has 9 rows: the 4 special symbols (<pad> = 0) and 5 words
        part = SequenceCNNEncoder(name="cnn", vocabulary=Vocabulary(["w{}".format(i) for i in range(5)]),
                                  data_id="source", embedding_size=4, filters=[(2, 3), (3, 2), (6, 2)])
        part._ids = dev("cnn_ids", torch.int64)
    elif tag.startswith("clf"):
        # 5 classes: the 4 special symbols and one label
        part = Classifier(name=tag, encoders=features, vocabulary=Vocabulary(["c0"]), data_id="label",
                          layers=[6, 5] if tag == "clf_layers" else [], dropout_keep_prob=1.0)
        part._labels = dev("labels", torch.int64)
    else:
        part = SequenceRegressor(name=tag, encoders=features, data_id="value",
                                 layers=[6, 5] if tag == "reg_layers" else [], dimension=1 if tag == "reg_layers" else 3)
        part._targets = dev("reg_targets")
    part.ensure_declared()
    arena = runtime.arena()
    arena.finalize(runtime.device())
    variables = golden_variables(g, tag)
    assert sorted(arena.order) == sorted(variables), (sorted(arena.order), sorted(variables))
    for name, value in variables.items():
        assert tuple(arena.get(name).shape) == value.shape, name
    arena.load_dict({n: torch.from_numpy(v) for n, v in variables.items()})
    if tag.startswith("att"):
        return {"weights": part.attention_weights, "temporal_states": part.temporal_states,
                "temporal_mask": part.temporal_mask, "output": part.output}
    if tag == "cnn":
        return {"output": part.output}
    if tag.startswith("clf"):
        return {"logits": part.decoded_logits, "decoded": part.decoded_seq, "logprobs": part.runtime_logprobs,
                "loss": part.cost}
    return {"predictions": part.predictions, "cost": part.cost}


MODEL_CASES = ("maxpool", "avgpool") + VARIABLE_CASES
