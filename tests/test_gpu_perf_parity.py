"""The BENCHED engine (default `auto` backend: wgmma fp16 / TF32 products, cluster GRU recurrence)
against the fp32 oracle at the PERF dimensions of BASELINE.json - the bar north_star states: train loss within
1e-3.  Parameters are random at a scale that makes every activation matter (the initialisers would leave the
logits at ~0 and the loss at log V whatever the arithmetic does)."""
import pytest
import torch

from oracle import nm_oracle as O
from tests.helpers import build_bahdanau, feed, oracle_params_for

pytestmark = pytest.mark.gpu

ENDE = dict(vs=32000, vt=32000, es=300, he=300, et=300, hd=300, out=300, maxout=False, max_len=50,
            supress_unk=False)


def _ids(bsz, length, vocab, seed, eos):
    g = torch.Generator().manual_seed(seed)
    ids = torch.randint(4, vocab, (bsz, length), generator=g)
    if eos:
        ids[:, -1] = 2
    return ids


@pytest.mark.parametrize("scale", [0.05, 0.1])
def test_ende_train_loss_within_1e3_of_the_oracle(scale):
    model = build_bahdanau(**ENDE, clip=1.0, l2=1e-8)
    params = oracle_params_for(model, scale=scale, seed=11)
    for name in params:
        if name.endswith("gamma"):
            params[name] = 1.0 + params[name]
    model["arena"].load_dict(params)
    src, tgt = _ids(16, 50, 32000, 1, False), _ids(16, 50, 32000, 2, True)
    feed(model, src, tgt, train=True)
    got = float(model["dec"].train_loss)
    spec = O.RNNDecoderSpec("decoder", "attention", 50, "tanh", False)
    with torch.no_grad():
        odec = O.decoder_train(params, spec, O.sentence_encoder(params, "sentence_encoder", src), tgt.t())
    want = float(odec["train_loss"])
    assert abs(got - want) < 1e-3, (got, want)
    # per-token cross-entropies: the fp16/TF32 products stay inside a 1e-2 band
    assert float((model["dec"].train_xents.cpu() - odec["train_xents"]).abs().max()) < 2e-2
    # the optimizer step runs through the CUDA-graph path the bench times and keeps the loss finite
    out = model["trainer"].train_step()
    assert abs(float(out["losses"][0]) - want) < 1e-3


def test_transformer_train_loss_within_1e3_of_the_oracle():
    from tests.test_gpu_transformer import build_transformer, feed_transformer, oracle_encoder
    cfg = dict(vs=32000, vt=32000, dim=512, ff=2048, depth=6, heads=8, max_len=32)
    model = build_transformer(**cfg, tie=True)
    params = oracle_params_for(model, scale=0.03, seed=5)
    for name in params:
        if name.endswith("gamma"):
            params[name] = 1.0 + params[name]
    model["arena"].load_dict(params)
    src, tgt = _ids(4, 32, 32000, 3, False), _ids(4, 32, 32000, 4, True)
    feed_transformer(model, src, tgt, train=True)
    got = float(model["dec"].train_loss)
    spec = O.TransformerDecoderSpec("decoder", 6, 8, 8, 32, True, False)
    with torch.no_grad():
        odec = O.transformer_decoder_train(params, spec, oracle_encoder(params, src, cfg), tgt)
    want = float(odec["loss"])
    assert abs(got - want) < 1e-3, (got, want)
