"""The ResNet-v2 image encoders on the GPU: nm_conv2d_bn_fwd on both engines against the fp64 restatement of
tests/resnet_oracle.py at every dispatch boundary, its refusals, the encoders at several end points of all three
depths, a captioning model over a frozen resnet_v2_50 (eager and captured steps), and a captioning INI through
bin/neuralmonkey-train."""
import math
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

from tests import resnet_oracle as RO
from tests.helpers import training_log_values

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))

# relative to the output's max-abs: the exact engine only reorders fp32 sums; TF32 operands keep 10 mantissa bits
# (test_gpu_imagenet.py's per-layer tolerance)
TOL = {"simt": 2e-5, "auto": 5e-3}


@pytest.fixture
def engine(request):
    from neuralmonkey_b200 import ops
    ops.set_gemm_backend(request.param)
    yield request.param
    ops.set_gemm_backend("auto")


def _rel(got, want):
    got, want = got.detach().double().cpu(), want.detach().double().cpu()
    return float((got - want).abs().max() / want.abs().max().clamp_min(1e-30))


# (N, H, W, Cin, Cout, k, stride, pads, prologue, output: None | "bias" | "bn", act, residual stride or None)
CASES = [
    (2, 19, 17, 3, 64, 7, 2, (3, 3), False, "bias", None, None),       # the stem: Cin 3 (scalar gather), odd H/W
    (1, 12, 10, 3, 5, 7, 1, (3, 3), False, None, None, None),         # 7x7 SAME at stride 1, Cout 5
    (2, 13, 7, 64, 256, 1, 1, (0, 0), True, "bias", None, None),      # a conv shortcut: prologue + bias
    (1, 15, 15, 64, 64, 1, 2, (0, 0), True, "bn", "relu", None),      # 1x1 / 2, M = 64 (below a tile)
    (1, 8, 16, 64, 64, 1, 1, (0, 0), True, "bn", "relu", None),       # M = 128: one whole tile
    (1, 9, 15, 64, 70, 1, 1, (0, 0), False, "bn", None, None),        # M = 135 across a tile, Cout off the tile
    (3, 10, 12, 64, 64, 3, 1, (1, 1), True, "bn", "relu", None),      # prologue through SAME padding (0 there)
    (2, 15, 15, 128, 128, 3, 2, (1, 1), False, "bn", "relu", None),   # a strided unit's conv2, odd size
    (2, 16, 14, 128, 130, 3, 2, (1, 1), True, "bn", "relu", None),    # even size, Cout across two tiles
    (2, 11, 9, 13, 24, 3, 2, (1, 1), True, "bias", "relu", None),     # Cin 13: the scalar gather with a prologue
    (2, 8, 8, 64, 256, 1, 1, (0, 0), False, "bias", None, 1),         # conv3 + the identity shortcut
    (2, 7, 7, 128, 512, 1, 1, (0, 0), False, "bias", None, 2),        # strided unit: shortcut x[::2, ::2], 13x13
    (2, 4, 4, 128, 512, 1, 1, (0, 0), False, "bias", None, 2),        # the same from an even 8x8 input
    (1, 9, 9, 64, 67, 1, 1, (0, 0), True, "bn", "relu", 1),           # every policy at once, Cout 67
    (2, 7, 5, 13, 9, 3, 2, (1, 1), False, None, "relu", 2),           # residual after a strided 3x3, no bias
]


def _case_tensors(case, seed):
    n, h, w, cin, cout, k, stride, pads, pro, out, act, rs = case
    gen = torch.Generator().manual_seed(seed)
    t = {"x": torch.randn(n, h, w, cin, generator=gen), "w": torch.randn(k, k, cin, cout, generator=gen) / math.sqrt(
        k * k * cin)}
    kw = {"stride": stride, "pads": pads, "act": act}
    if pro:
        kw["in_scale"] = 0.5 + torch.rand(cin, generator=gen)
        kw["in_shift"] = 0.3 * torch.randn(cin, generator=gen)
    if out == "bias":
        kw["bias"] = torch.randn(cout, generator=gen)
    elif out == "bn":
        kw["out_scale"] = 0.5 + torch.rand(cout, generator=gen)
        kw["out_shift"] = 0.3 * torch.randn(cout, generator=gen)
    if rs is not None:
        ho = (h + sum(pads) - k) // stride + 1
        wo = (w + sum(pads) - k) // stride + 1
        # the largest residual whose subsample fits: odd sizes 2*ho - 1 where the case says so (13 for 7)
        hr = ho if rs == 1 else (2 * ho - 1 if h % 2 else 2 * ho)
        wr = wo if rs == 1 else (2 * wo - 1 if w % 2 else 2 * wo)
        kw["res"], kw["res_stride"] = torch.randn(n, hr, wr, cout, generator=gen), rs
    return t["x"], t["w"], kw


def _on_gpu(kw):
    return {k: (v.cuda() if torch.is_tensor(v) else v) for k, v in kw.items()}


@pytest.mark.parametrize("engine", ["simt", "auto"], indirect=True)
@pytest.mark.parametrize("case", CASES)
def test_conv2d_bn_fwd_against_fp64(engine, case):
    from neuralmonkey_b200 import ops
    x, w, kw = _case_tensors(case, sum(case[:7]))
    want = RO.conv2d_bn(x, w, **kw)
    got = ops.conv2d_bn_fwd(x.cuda(), w.cuda(), **_on_gpu(kw))
    assert got.shape == want.shape
    assert _rel(got, want) < TOL[engine]
    again = ops.conv2d_bn_fwd(x.cuda(), w.cuda(), **_on_gpu(kw))
    assert torch.equal(got, again)


def _raw(tensors, **over):
    """nm_conv2d_bn_fwd with a valid 1x1 call's arguments, some replaced."""
    from neuralmonkey_b200 import lib
    x, w, y = tensors
    a = dict(x=lib.ptr(x), w=lib.ptr(w), in_scale=None, in_shift=None, out_scale=None, out_shift=None, bias=None,
             res=None, res_H=0, res_W=0, res_stride=1, y=lib.ptr(y), N=1, H=4, W=4, Cin=8, Cout=8, k=1, stride=1,
             pad_top=0, pad_bottom=0, pad_left=0, pad_right=0, act=0, backend=lib.GEMM_SIMT, stream=lib.stream())
    a.update(over)
    lib.call("nm_conv2d_bn_fwd", *a.values())


def test_conv2d_bn_fwd_refusals_launch_nothing():
    from neuralmonkey_b200 import lib
    x = torch.randn(1, 4, 4, 8, device="cuda")
    w = torch.randn(8, 8, device="cuda")
    v = torch.ones(8, device="cuda")
    res = torch.randn(1, 4, 4, 8, device="cuda")
    y = torch.empty(1, 4, 4, 8, device="cuda")
    _raw((x, w, y))
    _raw((x, w, y), res=lib.ptr(res), res_H=4, res_W=4)
    _raw((x, w, y), res=lib.ptr(res), res_H=3, res_W=4, res_stride=2, H=3, stride=2, k=1)
    torch.cuda.synchronize()
    refusals = [
        (dict(x=None), "null pointer"),
        (dict(y=None), "null pointer"),
        (dict(in_scale=lib.ptr(v)), "in_scale and in_shift"),
        (dict(out_shift=lib.ptr(v)), "out_scale and out_shift"),
        (dict(out_scale=lib.ptr(v), out_shift=lib.ptr(v), bias=lib.ptr(v)), "exclude each other"),
        (dict(act=1), "act must be"),
        (dict(backend=7), "bad backend"),
        (dict(stride=0), "bad sizes"),
        (dict(stride=-2), "bad sizes"),
        (dict(N=0), "bad sizes"),
        (dict(Cout=0), "bad sizes"),
        (dict(k=0), "bad sizes"),
        (dict(pad_top=1), "pads must lie"),
        (dict(k=3, pad_left=3), "pads must lie"),
        (dict(pad_right=-1), "pads must lie"),
        (dict(k=7, H=4, pad_top=1, pad_bottom=1), "window larger"),
        (dict(stride=4096), "out of range"),
        (dict(res=lib.ptr(res), res_H=4, res_W=4, res_stride=3), "res_stride must be 1 or 2"),
        (dict(res=lib.ptr(res), res_H=5, res_W=4), "does not match"),
        (dict(res=lib.ptr(res), res_H=4, res_W=4, res_stride=2), "does not match"),
        (dict(res=lib.ptr(res), res_H=0, res_W=0), "does not match"),
    ]
    for over, message in refusals:
        before = lib.launch_count()
        with pytest.raises(ValueError, match=message):
            _raw((x, w, y), **over)
        assert lib.launch_count() == before, over


def _encoder(net, layer, params):
    from neuralmonkey_b200 import runtime
    from neuralmonkey_b200.encoders import ImageNet
    runtime.reset()
    enc = ImageNet(name="imagenet", data_id="images", network_type=net, spatial_layer=layer)
    enc.ensure_declared()
    arena = runtime.arena()
    arena.finalize(runtime.device())
    arena.load_dict({n: params[n].float() for n in arena.order})
    return enc


def _tf32_tol(net, layer):
    """Each convolution on the path adds an independent TF32 rounding error of up to TOL['auto'] of its output's
    scale; batch norm, ReLU and the identity shortcuts pass it on with gain about 1 (the He-scaled filters and unit
    batch-norm gains here keep every layer's output O(1)), so the errors add like a random walk: sqrt(L) times the
    per-layer tolerance over a path of L convolutions."""
    names = RO.end_point_names(net)
    upto = names[:names.index(layer) + 1]
    convs = 1 + sum(n.endswith(("/conv1", "/conv2", "/conv3")) and "/block" in n for n in upto)
    return TOL["auto"] * math.sqrt(convs)


ENDPOINTS = [
    ("resnet_v2_50", "resnet_v2_50/conv1", 17),
    ("resnet_v2_50", "resnet_v2_50/block1/unit_1/bottleneck_v2/shortcut", 21),
    ("resnet_v2_50", "resnet_v2_50/block1/unit_3/bottleneck_v2/conv2", 21),
    ("resnet_v2_50", "resnet_v2_50/block2/unit_2/bottleneck_v2/conv3", 27),
    ("resnet_v2_50", "resnet_v2_50/block1", 33),
    ("resnet_v2_50", "resnet_v2_50/block2", 35),
    ("resnet_v2_50", "resnet_v2_50/block3", 37),
    ("resnet_v2_50", "resnet_v2_50/block4", 45),
    ("resnet_v2_101", "resnet_v2_101/block3/unit_23/bottleneck_v2/conv2", 33),
    ("resnet_v2_101", "resnet_v2_101/block4", 39),
    ("resnet_v2_152", "resnet_v2_152/block2", 29),
    ("resnet_v2_152", "resnet_v2_152/block4", 41),
]


@pytest.mark.parametrize("engine", ["simt", "auto"], indirect=True)
@pytest.mark.parametrize("net,layer,size", ENDPOINTS)
def test_encoder_end_points_against_the_oracle(engine, net, layer, size):
    params = RO.random_params(net, seed=size)
    enc = _encoder(net, layer, params)
    images = torch.randn(2, size, size, 3, generator=torch.Generator().manual_seed(size)) * 2.0
    enc.feed_images(images)
    want = RO.resnet_v2(params, net, images.double(), layer)[layer]
    got = enc.spatial_states
    assert got.shape == want.shape
    tol = TOL["simt"] if engine == "simt" else _tf32_tol(net, layer)
    err = _rel(got, want)
    print("{} {} {}: rel err {:.3g} (tol {:.3g})".format(engine, net, layer, err, tol))
    assert err < tol
    assert _rel(enc.output, want.mean(dim=(1, 2))) < tol * 2
    assert float(enc.spatial_mask.min()) == 1.0 and enc.spatial_mask.shape == got.shape[:3]


def test_resnet_v2_50_at_229():
    from neuralmonkey_b200 import ops
    net, layer = "resnet_v2_50", "resnet_v2_50/block4"
    params = RO.random_params(net, seed=229)
    images = torch.rand(2, 229, 229, 3, generator=torch.Generator().manual_seed(229)) * 2.0 - 1.0
    want = RO.resnet_v2(params, net, images.double(), layer)[layer]
    assert want.shape == (2, 8, 8, 2048)
    for backend in ("auto", "simt"):
        ops.set_gemm_backend(backend)
        try:
            enc = _encoder(net, layer, params)
            enc.feed_images(images)
            err = _rel(enc.spatial_states, want)
        finally:
            ops.set_gemm_backend("auto")
        tol = TOL["simt"] if backend == "simt" else _tf32_tol(net, layer)
        print("{} 229: rel err {:.3g} (tol {:.3g})".format(backend, err, tol))
        assert err < tol


def _captioning(mode, images, sentences, steps):
    from neuralmonkey_b200 import runtime, tf
    from neuralmonkey_b200.attention import Attention
    from neuralmonkey_b200.dataset import BatchingScheme, Dataset
    from neuralmonkey_b200.decoders.decoder import Decoder
    from neuralmonkey_b200.encoders import ImageNet
    from neuralmonkey_b200.trainers import CrossEntropyTrainer
    from neuralmonkey_b200.vocabulary import Vocabulary
    runtime.reset()
    enc = ImageNet(name="imagenet", data_id="images", network_type="resnet_v2_50",
                   spatial_layer="resnet_v2_50/block4")
    att = Attention(name="attention", encoder=enc, state_size=10)
    dec = Decoder(name="decoder", encoders=[enc], attentions=[att], rnn_size=9, embedding_size=9, data_id="target",
                  max_output_len=6, vocabulary=Vocabulary(["a", "b", "c", "d"]))
    trainer = CrossEntropyTrainer(decoders=[dec], l2_weight=1e-8, optimizer=tf.AdamOptimizer(learning_rate=1e-2),
                                  use_cuda_graph=mode)
    for part in (enc, att, dec):
        part.ensure_declared()
    arena = runtime.arena()
    arena.finalize(runtime.device())
    arena.load_dict({n: v.float() for n, v in RO.random_params("resnet_v2_50", seed=5).items() if n in arena.order})
    before = arena.state_dict()
    losses = []
    for _ in range(steps):
        data = Dataset("toy", {"images": lambda: iter(images), "target": lambda: iter(sentences)},
                       BatchingScheme(batch_size=len(images)))
        for part in (enc, att, dec):
            part.feed_dict(data, train=True)
        losses.append(trainer.train_step()["losses"][0].item())
    if mode:
        assert any(isinstance(v, tuple) for v in trainer._graphs.values()), trainer._graphs
    return losses, before, arena.state_dict()


def test_captioning_with_a_frozen_resnet_eager_and_captured():
    """resnet_v2_50 block4 -> attention decoder, Adam: the decoder learns, no ResNet variable moves, and the
    captured step gives the eager step's losses bit for bit."""
    rng = np.random.RandomState(6)
    images = [rng.uniform(-1, 1, size=(229, 229, 3)).astype(np.float32) for _ in range(3)]
    sentences = [["a", "b", "c"], ["d", "a"], ["b", "b", "d", "c"]]
    results = {}
    try:
        for mode in (False, True):
            results[mode] = _captioning(mode, images, sentences, 8)
    finally:
        from neuralmonkey_b200 import runtime
        runtime.reset()
    losses, before, after = results[False]
    assert all(np.isfinite(losses)) and all(b < a for a, b in zip(losses, losses[1:])), losses
    for name, value in before.items():
        if name.startswith("resnet_v2_50"):
            assert torch.equal(value, after[name]), name
    assert not torch.equal(before["decoder/state_to_word_W"], after["decoder/state_to_word_W"])
    # the captured step: the same losses bit for bit, the same frozen encoder; the attention decoder's captured step
    # moves its variables within the tolerance test_gpu_cnn.py allows it
    assert results[True][0] == losses
    for name, value in after.items():
        if name.startswith("resnet_v2_50"):
            assert torch.equal(results[True][2][name], value), name
        else:
            assert float((results[True][2][name] - value).abs().max()) < 2e-5, name


_INI = """
[main]
name="captioning over a frozen resnet_v2_50"
tf_manager=<tf_manager>
output="{out}"
overwrite_output_dir=True
batch_size=2
epochs=2
train_dataset=<train_data>
val_dataset=<val_data>
trainer=<trainer>
runners=[<runner>]
postprocess=None
evaluation=[("target", evaluators.BLEU)]
logging_period=1
validation_period=2
random_seed=1234

[tf_manager]
class=tf_manager.TensorFlowManager
num_threads=4
num_sessions=1

[image_reader]
class=readers.image_reader.imagenet_reader
prefix="{data}"
target_width=229
target_height=229
zero_one_normalization=True

[train_data]
class=dataset.load
series=["target", "images"]
data=["{data}/train.en", ("{data}/train_images.txt", <image_reader>)]

[val_data]
class=dataset.load
series=["target", "images"]
data=["{data}/val.en", ("{data}/val_images.txt", <image_reader>)]

[imagenet]
class=encoders.imagenet_encoder.ImageNet
name="imagenet_resnet"
data_id="images"
network_type="resnet_v2_50"
spatial_layer="resnet_v2_50/block4"

[attention]
class=attention.Attention
state_size=10
name="attention"
encoder=<imagenet>

[decoder_vocabulary]
class=vocabulary.from_wordlist
path="{data}/vocab.tsv"

[decoder]
class=decoders.decoder.Decoder
name="decoder"
encoders=[<imagenet>]
rnn_size=9
embedding_size=9
attentions=[<attention>]
dropout_keep_prob=0.5
data_id="target"
max_output_len=6
vocabulary=<decoder_vocabulary>

[trainer]
class=trainers.cross_entropy_trainer.CrossEntropyTrainer
decoders=[<decoder>]
l2_weight=1.0e-8

[runner]
class=runners.GreedyRunner
decoder=<decoder>
output_series="target"
"""


def test_captioning_ini_trains_through_neuralmonkey_train(tmp_path):
    from PIL import Image
    data = tmp_path / "data"
    data.mkdir()
    rng = np.random.RandomState(7)
    words = ["a", "dog", "runs", "cat", "sits", "on", "grass"]
    for split, count in (("train", 4), ("val", 2)):
        names = []
        for i in range(count):
            name = "{}_{}.png".format(split, i)
            Image.fromarray(rng.randint(0, 256, size=(240, 250, 3)).astype(np.uint8)).save(str(data / name))
            names.append(name)
        (data / "{}_images.txt".format(split)).write_text("\n".join(names) + "\n")
        (data / "{}.en".format(split)).write_text(
            "\n".join(" ".join(rng.choice(words, size=rng.randint(2, 5))) for _ in range(count)) + "\n")
    (data / "vocab.tsv").write_text("Word\tWord counts\n<pad>\t0\n<s>\t0\n</s>\t0\n<unk>\t0\n" +
                                    "".join("{}\t1\n".format(w) for w in words))
    out = str(tmp_path / "out")
    ini = tmp_path / "resnet.ini"
    ini.write_text(_INI.format(out=out, data=str(data)))
    cmd = [sys.executable, os.path.join(ROOT, "bin", "neuralmonkey-train"), str(ini)]
    env = dict(os.environ, NEURALMONKEY_STRICT="1", PYTHONPATH=ROOT + os.pathsep + os.environ.get("PYTHONPATH", ""))
    res = subprocess.run(cmd, capture_output=True, text=True, timeout=900, cwd=str(tmp_path), env=env)
    assert res.returncode == 0, res.stdout[-3000:] + res.stderr[-3000:]
    log_text = open(os.path.join(out, "experiment.log")).read()
    assert "Training finished" in log_text and "Validation (epoch" in log_text
    losses = training_log_values(log_text, "target/train_xent")
    assert losses and all(np.isfinite(losses)), losses
