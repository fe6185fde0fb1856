"""Shared builders for the parity tests: the same Bahdanau model in the CUDA framework
and in the CPU oracle, fed with the same ids and the same parameters."""
from typing import Dict, Optional

import torch

from oracle import nm_oracle as O


def build_bahdanau(vs=60, vt=70, es=11, he=7, et=9, hd=8, out=9, maxout=True, max_len=10,
                   supress_unk=True, l1=0.0, l2=0.0, clip=None, lr=1e-4, cuda_graph=False, out_act=None):
    """Encoder + attention + decoder + trainer of tests/bahdanau.ini's shape family.  Without maxout, `out_act`
    ("tanh", "relu" or "sigmoid") selects a dense output projection of size `out` with that activation;
    None keeps the decoder's default."""
    from neuralmonkey_b200 import runtime
    from neuralmonkey_b200.attention import Attention
    from neuralmonkey_b200.decoders import Decoder
    from neuralmonkey_b200.decoders.output_projection import maxout_output, nonlinear_output
    from neuralmonkey_b200.encoders import SentenceEncoder
    from neuralmonkey_b200.trainers import CrossEntropyTrainer
    from neuralmonkey_b200 import tf
    from neuralmonkey_b200.vocabulary import Vocabulary

    runtime.reset()
    src_vocab = Vocabulary(["s{}".format(i) for i in range(vs - 4)])
    tgt_vocab = Vocabulary(["t{}".format(i) for i in range(vt - 4)])
    enc = SentenceEncoder(name="sentence_encoder", vocabulary=src_vocab, data_id="source",
                          embedding_size=es, rnn_size=he, max_input_len=max_len)
    att = Attention(name="attention", encoder=enc)
    dec = Decoder(encoders=[enc], vocabulary=tgt_vocab, data_id="target", name="decoder",
                  max_output_len=max_len, rnn_size=hd, embedding_size=et, attentions=[att],
                  output_projection=(maxout_output(out) if maxout else
                                     nonlinear_output(out, out_act) if out_act else None),
                  supress_unk=supress_unk)
    trainer = CrossEntropyTrainer(decoders=[dec], l1_weight=l1, l2_weight=l2, clip_norm=clip,
                                  optimizer=tf.AdamOptimizer(learning_rate=lr), use_cuda_graph=cuda_graph)
    for part in trainer.parameterizeds:
        part.ensure_declared()
    runtime.arena().finalize(runtime.device())
    return {"enc": enc, "att": att, "dec": dec, "trainer": trainer, "arena": runtime.arena()}


def oracle_spec(maxout=True, max_len=10, supress_unk=True):
    return O.RNNDecoderSpec("decoder", "attention", max_len, "maxout" if maxout else "tanh",
                            supress_unk)


def feed(model, src_ids: torch.Tensor, tgt_ids: Optional[torch.Tensor], train: bool):
    """src_ids [B,Tx], tgt_ids [B,Ty] (incl. </s>) int64 CPU tensors."""
    bsz = src_ids.shape[0]
    enc, att, dec = model["enc"], model["att"], model["dec"]
    enc.input_sequence.feed_ids([src_ids], train=train)
    for part in (enc, att):
        part.reset_batch()
        part.train_mode = train
        part.batch_size = bsz
    dec.feed_ids(tgt_ids, bsz, train=train)


def random_batch(bsz, tx, ty, vs, vt, seed=0, ragged=True):
    """Token ids in [4, V); ragged lengths >= 1; targets end with </s> then <pad>."""
    g = torch.Generator().manual_seed(seed)
    src = torch.randint(4, vs, (bsz, tx), generator=g)
    tgt = torch.randint(4, vt, (bsz, ty), generator=g)
    if ragged:
        src_len = torch.randint(1, tx + 1, (bsz,), generator=g)
        tgt_len = torch.randint(1, ty, (bsz,), generator=g)
        src_len[0], tgt_len[0] = tx, ty - 1       # one full-length sentence keeps T fixed
    else:
        src_len = torch.full((bsz,), tx)
        tgt_len = torch.full((bsz,), ty - 1)
    for b in range(bsz):
        src[b, src_len[b]:] = 0
        tgt[b, tgt_len[b]] = 2
        tgt[b, tgt_len[b] + 1:] = 0
    return src, tgt


def oracle_params_for(model, scale=0.3, seed=7, dtype=torch.float32) -> Dict[str, torch.Tensor]:
    """Random O(scale) parameters with the framework's variable names and shapes."""
    arena = model["arena"]
    # sorted: the declaration order follows the iteration order of a set of model parts
    shapes = {n: torch.zeros(arena.variables[n].shape, dtype=dtype) for n in sorted(arena.order)}
    return O.randomize(shapes, scale=scale, seed=seed)


def rel_err(a: torch.Tensor, b: torch.Tensor) -> float:
    a, b = a.double().cpu(), b.double().cpu()
    return float((a - b).norm() / (b.norm() + 1e-30))


def max_abs(a: torch.Tensor, b: torch.Tensor) -> float:
    return float((a.detach().double().cpu() - b.detach().double().cpu()).abs().max())


def training_log_values(log_text: str, name: str):
    """The values of `name` on the lines logged for TRAINING batches: "Epoch e/m  Instances n  ..." lines
    that are not the result line of a validation (the first such line after a "Validation (epoch" header)."""
    values, in_validation = [], False
    for line in log_text.splitlines():
        if "Validation (epoch" in line:
            in_validation = True
        elif "  Instances " in line and "Epoch " in line:
            if in_validation:
                in_validation = False
            elif name + ": " in line:
                values.append(float(line.split(name + ": ")[1].split()[0]))
    return values
