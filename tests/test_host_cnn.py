"""The CNN encoder's host side on the CPU: layer-spec validation and shapes, the model part over the fp64 stand-ins
of tests/cnn_oracle.py (variable names, masks, the temporal view, moving statistics), `image_reader` on the
reference's scene-text images, the Adadelta update, and the reference's tests/str.ini through `neuralmonkey-train`
(inputs from tests/golden/reference_experiments_str.json).  The kernels themselves are tested in
tests/test_gpu_cnn.py."""
import os
import sys

import numpy as np
import pytest
import torch

from tests import cnn_oracle as CO
from tests import cpu_ops
from tests.golden.make_str_bundle import unpack

pytestmark = [pytest.mark.filterwarnings("ignore:Converting a tensor with requires_grad")]

STR_SPECS = [("C", 3, 1, "valid", 4), ("M", 2, 2, "same"), ("R", 3, 12), ("A", 2, 1, "same")]


def _adadelta_stand_in(trainer, grad_scale, denominator, lr_t, lr_t_dev):
    """GenericTrainer._adam_kernel over the arena on the CPU, for either optimizer."""
    from neuralmonkey_b200 import runtime, tf
    opt = trainer.optimizer
    if not isinstance(opt, tf.AdadeltaOptimizer):
        return cpu_ops.adam_kernel(trainer, grad_scale, denominator, lr_t, lr_t_dev)
    from oracle import nm_oracle as O
    arena = runtime.arena()
    scale = float(grad_scale) / (float(denominator) if denominator is not None else 1.0)
    trainer._l1l2_buf = torch.zeros(2)
    accum, accum_update = arena.optimizer_slot(opt)
    with torch.no_grad():
        for name in trainer.var_list:
            var = arena.get(name)
            grad = arena.grad(name) * scale
            if O.is_regularizable(name):
                grad = grad + 2.0 * trainer.l2_weight * var
            info = arena.variables[name]
            sl = slice(info.offset, info.offset + var.numel())
            p, g = {0: var.clone()}, {0: grad}
            a, u = {0: accum[sl].view(var.shape).clone()}, {0: accum_update[sl].view(var.shape).clone()}
            CO.adadelta_step(p, g, a, u, float(lr_t), opt.rho, opt.epsilon, trainer.clip_norm)
            var.copy_(p[0])
            accum[sl].copy_(a[0].reshape(-1))
            accum_update[sl].copy_(u[0].reshape(-1))


@pytest.fixture
def cpu_model(monkeypatch):
    from neuralmonkey_b200 import ops, runtime
    from neuralmonkey_b200.trainers.generic_trainer import GenericTrainer
    for op in cpu_ops.STAND_INS:
        monkeypatch.setattr(ops, op, getattr(cpu_ops, op))
    for op in ("conv2d", "batch_norm", "pool2d"):
        monkeypatch.setattr(ops, op, getattr(CO, op))
    monkeypatch.setattr(runtime, "_device", torch.device("cpu"))
    monkeypatch.setattr(GenericTrainer, "_adam_kernel", _adadelta_stand_in)
    yield
    runtime.reset()


def _cnn(specs=STR_SPECS, hw=(32, 256), pixel=1, bn=True, fc=None):
    from neuralmonkey_b200.encoders.cnn_encoder import CNNEncoder
    return CNNEncoder(name="cnn", data_id="images", convolutions=specs, image_height=hw[0], image_width=hw[1],
                      pixel_dim=pixel, batch_normalize=bn, fully_connected=fc)


@pytest.mark.parametrize("specs,bn,message", [
    ([("C", 3, 1, "valid")], True, "needs to have 5 members"),
    ([("C", 3, 1, "full", 4)], True, "Padding must be 'same' or 'valid'"),
    ([("C", 3.0, 1, "same", 4)], True, "needs to have 5 members"),
    ([("C", 3, 2, "same", 4)], True, "Layer 1"),             # stride only reaches the mask: refused
    ([("C", 0, 1, "same", 4)], True, "must be positive"),
    ([("M", 2, 2)], True, "max-pooling layer"),
    ([("A", 2, 2, "full")], True, "Padding must be"),
    ([("M", 64, 1, "valid")], True, "smaller than the window"),
    ([("R", 3)], True, "residual block"),
    ([("R", 3, 8)], False, "requires batch normalization"),
    ([("X", 3, 1, "same", 4)], True, "Unknown type"),
    ([("C", 3, 1, "same", 4), ("C", 5, 3, "valid", 4)], True, "Layer 2"),
])
def test_every_spec_error_raises(specs, bn, message):
    with pytest.raises(ValueError, match=message):
        _cnn(specs, bn=bn)


def test_str_shapes_and_variable_names(cpu_model):
    from neuralmonkey_b200 import runtime
    from neuralmonkey_b200.encoders.cnn_encoder import CNNTemporalView
    cnn = _cnn()
    view = CNNTemporalView(name="cnn_in_time", cnn=cnn)
    assert [s for s, _ in cnn.shapes] == [(30, 254, 4), (15, 127, 4), (15, 127, 12), (14, 126, 12)]
    assert view.dimension == 14 * 12
    cnn.ensure_declared()
    arena = runtime.arena()
    arena.finalize(runtime.device())
    names = set(arena.order)
    block = "cnn/convolutions/layer_2_resnet_block/"
    for want in ["cnn/convolutions/layer_0_convolution/conv2d/kernel", "cnn/convolutions/layer_0_convolution/conv2d/bias",
                 "cnn/convolutions/layer_0_convolution/batch_normalization/gamma",
                 block + "project_input/conv2d/kernel", block + "project_input/batch_normalization/moving_variance",
                 block + "conv_a/batch_normalization/beta", block + "conv_a/conv2d/kernel",
                 block + "conv_b/conv2d/bias", block + "conv_b/batch_normalization/moving_mean"]:
        assert want in names, want
    assert arena.get("cnn/convolutions/layer_0_convolution/conv2d/kernel").shape == (3, 3, 1, 4)
    assert arena.get(block + "conv_a/conv2d/kernel").shape == (3, 3, 4, 12)
    moving = {n for n in names if "moving_" in n}
    assert moving and not moving & set(arena.train_names)      # saved, never trained, no L2


@pytest.mark.parametrize("case", ["str", "residual_same_channels_fc", "plain"])
def test_encoder_over_the_stand_ins_against_the_oracle(cpu_model, case):
    from neuralmonkey_b200 import runtime
    from neuralmonkey_b200.encoders.cnn_encoder import CNNTemporalView
    cfg = {"str": (STR_SPECS, (32, 40), 1, True, None),
           "residual_same_channels_fc": ([("C", 2, 1, "same", 6), ("R", 3, 6), ("M", 2, 2, "valid")], (12, 14), 3,
                                         True, [10, 5]),
           "plain": ([("C", 5, 1, "same", 8), ("A", 3, 2, "valid"), ("C", 2, 1, "valid", 5)], (15, 18), 2, False,
                     None)}[case]
    specs, hw, pixel, bn, fc = cfg
    cnn = _cnn(specs, hw, pixel, bn, fc)
    cnn.dropout_keep_prob = 1.0
    view = CNNTemporalView(name="view", cnn=cnn)
    cnn.ensure_declared()
    arena = runtime.arena()
    arena.finalize(runtime.device())
    rng = np.random.RandomState(0)
    images = rng.randint(0, 256, size=(3, hw[0], hw[1], pixel)).astype(np.float32)
    images[:, :, -12:] = 0
    before = {n: arena.get(n).detach().clone() for n in arena.order}
    cnn.feed_images(torch.from_numpy(images / np.float32(255.0)), train=True)
    p = {n: v.double().clone() for n, v in before.items()}
    want = CO.cnn_encoder(p, "cnn", specs, torch.from_numpy(images).double() / 255.0, bn, True, fc)
    assert torch.allclose(view.temporal_states.double(), want["temporal_states"], atol=1e-5)
    assert torch.equal(view.temporal_mask.double(), want["temporal_mask"])
    assert torch.allclose(cnn.output.double(), want["output"], atol=1e-5)
    assert cnn.spatial_mask.shape[:3] == cnn.spatial_states.shape[:3]
    # the column mask: the blank right margin of every image is masked out at the end of the sequence
    assert float(view.temporal_mask[:, -1].sum()) == 0.0 and float(view.temporal_mask[:, 0].sum()) == 3.0
    for n in arena.order:
        if "moving_" in n:
            assert torch.allclose(arena.get(n).double(), p[n], atol=1e-6), n


def test_image_reader_on_the_str_images(tmp_path):
    from PIL import Image
    from neuralmonkey_b200.readers.image_reader import image_reader
    unpack(str(tmp_path))
    prefix = str(tmp_path / "tests" / "data" / "str")
    reader = image_reader(pad_w=256, pad_h=32, channels=1, prefix=prefix, rescale_w=True, rescale_h=True, mode="F")
    images = list(reader([os.path.join(prefix, "val_files.txt")]))
    assert len(images) == 10
    names = open(os.path.join(prefix, "val_files.txt")).read().split()
    for name, img in zip(names, images):
        assert img.shape == (32, 256, 1) and img.dtype == np.float64
        src = Image.open(os.path.join(prefix, name)).convert("F")
        want = np.array(src if src.size == (256, 32) else src.resize((256, 32), Image.BILINEAR))
        assert np.array_equal(img[:, :, 0], want)
    # keep_aspect_ratio: the image fits inside 32 x 256 and the rest is zero padding
    reader = image_reader(pad_w=256, pad_h=32, channels=1, prefix=prefix, rescale_w=True, rescale_h=True,
                          keep_aspect_ratio=True, mode="L")
    img = next(iter(reader([os.path.join(prefix, "val_files.txt")])))
    src = Image.open(os.path.join(prefix, names[0]))
    ratio = min(32 / src.size[1], 256 / src.size[0])
    w, h = int(src.size[0] * ratio), int(src.size[1] * ratio)
    assert not img[h:].any() and not img[:, w:].any()
    # crop without rescaling: centred, the odd pixel dropped on the right / bottom
    reader = image_reader(pad_w=20, pad_h=10, channels=3, prefix=prefix)
    img = next(iter(reader([os.path.join(prefix, "val_files.txt")])))
    full = np.array(src.convert("RGB"))
    dy, dx = (full.shape[0] - 10) // 2, (full.shape[1] - 20) // 2
    assert np.array_equal(img, full[dy:dy + 10, dx:dx + 20].astype(np.float64))


@pytest.mark.parametrize("kwargs,message", [
    (dict(keep_aspect_ratio=True), "keep the aspect ratio while not rescaling"),
    (dict(rescale_w=True), "aspect ratio must be kept"),
])
def test_image_reader_validation(kwargs, message):
    from neuralmonkey_b200.readers.image_reader import image_reader
    with pytest.raises(ValueError, match=message):
        image_reader(pad_w=8, pad_h=8, **kwargs)


def test_image_reader_refuses_wrong_channel_count(tmp_path):
    from neuralmonkey_b200.readers.image_reader import image_reader
    unpack(str(tmp_path))
    prefix = str(tmp_path / "tests" / "data" / "str")
    reader = image_reader(pad_w=256, pad_h=32, channels=1, prefix=prefix, mode="RGB")
    with pytest.raises(ValueError, match="pre-declared number of channels 1, but 3"):
        next(iter(reader([os.path.join(prefix, "val_files.txt")])))


def test_adadelta_optimizer_is_exposed():
    from neuralmonkey_b200 import tf
    opt = tf.train.AdadeltaOptimizer(learning_rate=1e-4, epsilon=1e-6, rho=0.95)
    assert (opt.learning_rate, opt.rho, opt.epsilon) == (1e-4, 0.95, 1e-6)


def test_batch_norm_refuses_data_parallel_training(cpu_model, monkeypatch):
    from neuralmonkey_b200 import distributed
    cnn = _cnn(hw=(32, 40))
    monkeypatch.setattr(distributed, "world_size", lambda: 2)
    with pytest.raises(RuntimeError, match="one rank"):
        cnn.feed_images(torch.zeros(2, 32, 40, 1), train=True)
    cnn.feed_images(torch.zeros(2, 32, 40, 1), train=False)     # inference is per sentence: allowed


def test_reference_str_ini_trains_over_the_stand_ins(cpu_model, monkeypatch, tmp_path):
    from neuralmonkey_b200 import runtime
    monkeypatch.setenv("NEURALMONKEY_STRICT", "1")
    unpack(str(tmp_path / "tree"))
    monkeypatch.chdir(tmp_path / "tree")
    out = str(tmp_path / "str")
    monkeypatch.setattr(sys, "argv", ["neuralmonkey-train", "tests/str.ini", "-s", 'main.output="{}"'.format(out)])
    try:
        from neuralmonkey_b200.train import main
        main()
    finally:
        runtime.reset()
    log_text = open(os.path.join(out, "experiment.log")).read()
    assert "Training finished" in log_text and "Validation (epoch" in log_text


# -- against the reference's own code (tests/golden/make_cnn_golden.py -> cnn_golden.npz) ----------------------------
GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "cnn_golden.npz")
GOLDEN_CASES = {
    "str": (STR_SPECS, (32, 64, 1), True, None),
    "residual": ([("C", 2, 1, "same", 6), ("R", 3, 6), ("R", 5, 9), ("M", 2, 2, "valid")], (12, 14, 3), True, [10, 5]),
    "plain": ([("C", 5, 1, "same", 8), ("A", 3, 2, "valid"), ("C", 2, 1, "valid", 5), ("M", 3, 1, "same")],
              (15, 18, 2), False, None),
}
OUTPUTS = ("spatial_states", "spatial_mask", "output", "temporal_states", "temporal_mask")


def golden_case(tag):
    """(variables {name: fp32 array}, images [B,H,W,C] 0..255, {mode: {output: array}}, moving statistics after the
    training pass) of one case of the golden file."""
    g = np.load(GOLDEN)
    names = [str(n) for n in g[tag + "_variable_names"]]
    variables = {n: g[tag + "_var:" + n] for n in names}
    outputs = {mode: {o: g["{}_{}_{}".format(tag, mode, o)] for o in OUTPUTS} for mode in ("train", "eval")}
    moving = {k.split(":", 1)[1]: g[k] for k in g.files if k.startswith(tag + "_moving_after:")}
    return variables, g[tag + "_images"], outputs, moving


@pytest.mark.parametrize("tag", sorted(GOLDEN_CASES))
def test_oracle_against_the_reference_code(tag):
    """The fp64 restatement of tests/cnn_oracle.py against the reference's CNNEncoder / CNNTemporalView."""
    specs, _hw, bn, fc = GOLDEN_CASES[tag]
    variables, images, outputs, moving = golden_case(tag)
    for mode in ("train", "eval"):
        p = {n: torch.from_numpy(v).double() for n, v in variables.items()}
        got = CO.cnn_encoder(p, "cnn", specs, torch.from_numpy(images) / 255.0, bn, mode == "train", fc)
        for name in OUTPUTS:
            want = torch.from_numpy(outputs[mode][name])
            assert got[name].shape == want.shape, name
            # (the stand-in's dense layers run in fp32)
            assert torch.allclose(got[name], want, rtol=1e-6, atol=1e-6), (mode, name)
        if mode == "train":
            for name, want in moving.items():
                assert torch.allclose(p[name], torch.from_numpy(want), rtol=1e-6, atol=1e-7), name


@pytest.mark.parametrize("tag", sorted(GOLDEN_CASES))
def test_model_part_against_the_reference_code(cpu_model, tag):
    """The model part over the fp64 stand-ins, with the golden's variables loaded BY NAME: the same variable names
    and shapes as the reference's graph, the same outputs in training and inference, the same moving statistics."""
    from neuralmonkey_b200 import runtime
    from neuralmonkey_b200.encoders.cnn_encoder import CNNTemporalView
    specs, (h, w, c), bn, fc = GOLDEN_CASES[tag]
    variables, images, outputs, moving = golden_case(tag)
    for mode in ("train", "eval"):
        runtime.reset()
        cnn = _cnn(specs, (h, w), c, bn, fc)
        cnn.dropout_keep_prob = 1.0
        view = CNNTemporalView(name="cnn_in_time", cnn=cnn)
        cnn.ensure_declared()
        arena = runtime.arena()
        arena.finalize(runtime.device())
        assert sorted(arena.order) == sorted(variables)
        assert all(tuple(arena.get(n).shape) == v.shape for n, v in variables.items())
        arena.load_dict({n: torch.from_numpy(v) for n, v in variables.items()})
        cnn.feed_images(torch.from_numpy((images / 255.0).astype(np.float32)), train=mode == "train")
        got = {"spatial_states": cnn.spatial_states, "spatial_mask": cnn.spatial_mask, "output": cnn.output,
               "temporal_states": view.temporal_states, "temporal_mask": view.temporal_mask}
        for name in OUTPUTS:
            want = torch.from_numpy(outputs[mode][name])
            assert torch.allclose(got[name].double(), want, rtol=1e-5, atol=1e-5), (mode, name)
        for name, want in moving.items():
            expected = torch.from_numpy(want) if mode == "train" else torch.from_numpy(variables[name]).double()
            assert torch.allclose(arena.get(name).double(), expected, rtol=1e-6, atol=1e-6), (mode, name)
    runtime.reset()


def test_adadelta_against_the_restated_tf_update():
    g = np.load(GOLDEN)
    p = {0: torch.from_numpy(g["adadelta_var0"])}
    acc, upd = {0: torch.zeros_like(p[0])}, {0: torch.zeros_like(p[0])}
    for step, grad in enumerate(g["adadelta_grads"]):
        CO.adadelta_step(p, {0: torch.from_numpy(grad)}, acc, upd, float(g["adadelta_lr"]), float(g["adadelta_rho"]),
                         float(g["adadelta_eps"]))
        assert torch.allclose(p[0], torch.from_numpy(g["adadelta_trajectory"][step]), rtol=1e-12, atol=1e-12)


def test_image_reader_against_the_reference_reader(tmp_path):
    from neuralmonkey_b200.readers.image_reader import image_reader
    unpack(str(tmp_path))
    g = np.load(GOLDEN)
    prefix = str(tmp_path / "tests" / "data" / "str")
    list_file = str(tmp_path / "files.txt")
    with open(list_file, "w") as handle:
        handle.write("\n".join(str(n) for n in g["reader_files"]) + "\n")
    readers = {"rescale": dict(pad_w=256, pad_h=32, channels=1, rescale_w=True, rescale_h=True, mode="F"),
               "aspect": dict(pad_w=256, pad_h=32, channels=1, rescale_w=True, rescale_h=True,
                              keep_aspect_ratio=True, mode="L"),
               "crop": dict(pad_w=20, pad_h=10, channels=3)}
    for tag, kwargs in readers.items():
        got = np.stack(list(image_reader(prefix=prefix, **kwargs)([list_file])))
        assert got.dtype == np.float64
        assert np.array_equal(got.astype(np.float32), g["reader_" + tag]), tag
