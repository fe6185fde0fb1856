"""Frozen VGG encoder + Bahdanau captioning decoder (tests/captioning.ini's shape family)."""
import pytest
import torch

from oracle import nm_oracle as O
from tests.helpers import max_abs, oracle_params_for, random_batch

pytestmark = pytest.mark.gpu


def build_captioning(spatial_layer="vgg_16/conv5/conv5_3", vt=50, max_len=8):
    from neuralmonkey_b200 import runtime, tf
    from neuralmonkey_b200.attention import Attention
    from neuralmonkey_b200.decoders import Decoder
    from neuralmonkey_b200.encoders import ImageNet
    from neuralmonkey_b200.trainers import CrossEntropyTrainer
    from neuralmonkey_b200.vocabulary import Vocabulary

    runtime.reset()
    vocab = Vocabulary(["t{}".format(i) for i in range(vt - 4)])
    enc = ImageNet(name="imagenet_vgg", data_id="images", network_type="vgg_16",
                   spatial_layer=spatial_layer)
    att = Attention(name="attention", encoder=enc, state_size=10)
    dec = Decoder(encoders=[enc], vocabulary=vocab, data_id="target", name="decoder",
                  max_output_len=max_len, rnn_size=9, embedding_size=9, attentions=[att])
    trainer = CrossEntropyTrainer(decoders=[dec], l2_weight=1e-8,
                                  optimizer=tf.AdamOptimizer(learning_rate=1e-3))
    for part in trainer.parameterizeds:
        part.ensure_declared()
    runtime.arena().finalize(runtime.device())
    return {"enc": enc, "att": att, "dec": dec, "trainer": trainer, "arena": runtime.arena()}


def _params(model):
    params = oracle_params_for(model, scale=0.3)
    for name in params:  # He-scaled filters keep activations O(1) through 13 layers
        if name.endswith("/weights"):
            fan_in = params[name].shape[0] * params[name].shape[1] * params[name].shape[2]
            params[name] = params[name] / 0.3 * (2.0 / fan_in) ** 0.5
    model["arena"].load_dict(params)
    return params


@pytest.mark.parametrize("layer,size", [("vgg_16/conv1/conv1_2", 8), ("vgg_16/pool2", 12),
                                        ("vgg_16/conv5/conv5_3", 32)])
@pytest.mark.parametrize("backend,rtol", [("simt", 2e-5), ("auto", 5e-3)])
def test_vgg_stack_matches_oracle(layer, size, backend, rtol):
    """simt: implicit-GEMM convolution on the CUDA cores (exact fp32); auto: im2col + wgmma GEMM
    with the bias+ReLU epilogue (TF32 operands)."""
    from neuralmonkey_b200 import ops
    ops.set_gemm_backend(backend)
    try:
        _vgg_check(layer, size, rtol)
    finally:
        ops.set_gemm_backend("auto")


def _vgg_check(layer, size, rtol):
    model = build_captioning(layer)
    params = _params(model)
    images = torch.randn(2, size, size, 3, generator=torch.Generator().manual_seed(1)) * 50.0
    model["enc"].feed_images(images)
    want = O.vgg_features({n: v.double() for n, v in params.items()}, "vgg_16", images.double(), layer)
    got = model["enc"].spatial_states
    assert got.shape == want["spatial_states"].shape
    scale = float(want["spatial_states"].abs().max())
    assert max_abs(got, want["spatial_states"]) < rtol * scale + 1e-6
    assert max_abs(model["enc"].output, want["output"]) < rtol * scale + 1e-6
    assert float(model["enc"].spatial_mask.min()) == 1.0


def test_captioning_train_step_and_frozen_encoder():
    from neuralmonkey_b200 import ops
    try:
        ops.set_gemm_backend("simt")
        model = build_captioning()
        params = _params(model)
        enc, att, dec = model["enc"], model["att"], model["dec"]
        images = torch.randn(3, 32, 32, 3, generator=torch.Generator().manual_seed(2))
        _src, tgt = random_batch(3, 4, 6, 50, 50, seed=3)
        enc.feed_images(images, train=True)
        att.reset_batch()
        att.train_mode, att.batch_size = True, 3
        dec.feed_ids(tgt, 3, train=True)
        oenc = O.vgg_features(params, "vgg_16", images, "vgg_16/conv5/conv5_3")
        spec = O.RNNDecoderSpec("decoder", "attention", 8, "tanh", False)
        odec = O.decoder_train(params, spec, oenc, tgt.t())
        assert abs(float(dec.train_loss) - float(odec["train_loss"])) < 1e-4
        # no VGG variable is trainable: the optimizer never sees them
        arena = model["arena"]
        assert not any(n.startswith("vgg_16") for n in arena.train_names)
        before = arena.state_dict()
        model["trainer"].train_step()
        after = arena.state_dict()
        for name in before:
            if name.startswith("vgg_16"):
                assert torch.equal(before[name], after[name]), name
        assert not torch.equal(before["decoder/state_to_word_W"], after["decoder/state_to_word_W"])
    finally:
        ops.set_gemm_backend("auto")
