"""Golden vectors from the reference's own `encoders/cnn_encoder.py` (`CNNEncoder`, `CNNTemporalView`) and
`readers/image_reader.py` (`image_reader`), executed over the numpy TensorFlow stand-in of tf_numpy_shim.py.

The TF 1.x layers the encoder calls are restated here in numpy fp64 (TensorFlow is not available):
  tf.layers.conv2d               stride 1; `same` pads k-1, (k-1)//2 before and the rest after; kernel + bias
  tf.layers.batch_normalization  momentum 0.99, epsilon 1e-3, gamma and beta; training: the batch mean and the biased
                                 batch variance, moving_variance moved toward the Bessel-corrected one (the fused 4-D
                                 kernel); inference: the moving statistics
  tf.layers.max_pooling2d        `valid` / `same` (padding ignored by the max)
  tf.layers.average_pooling2d    `valid` / `same` (divides by the pixels inside the image)
Layer variables are named as tf.layers names them: `<scope>/conv2d/kernel`, `<scope>/batch_normalization/gamma`, ...
(the first layer of a kind in a variable scope has the bare name, later ones `_1`, `_2`, ...).  What this pins is
the reference's side: layer order, the residual block, the masks, the temporal view, the fully connected head, the
variable names.  Adadelta over three steps is TF's ApplyAdadelta update restated.

    python tests/golden/make_cnn_golden.py   ->  tests/golden/cnn_golden.npz      (needs /root/reference)
"""
import collections
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
REFERENCE = "/root/reference"
sys.path.insert(0, HERE)
import tf_numpy_shim as shim  # noqa: E402
from make_host_golden import install_stubs  # noqa: E402

# (tag, convolutions, (height, width, channels), batch_normalize, fully_connected)
CASES = [
    ("str", [("C", 3, 1, "valid", 4), ("M", 2, 2, "same"), ("R", 3, 12), ("A", 2, 1, "same")], (32, 64, 1), True,
     None),
    ("residual", [("C", 2, 1, "same", 6), ("R", 3, 6), ("R", 5, 9), ("M", 2, 2, "valid")], (12, 14, 3), True,
     [10, 5]),
    ("plain", [("C", 5, 1, "same", 8), ("A", 3, 2, "valid"), ("C", 2, 1, "valid", 5), ("M", 3, 1, "same")],
     (15, 18, 2), False, None),
]
BATCH = 3
MOVING_AFTER = {}
_LAYER_COUNT = collections.Counter()


def _layer_name(base):
    scope = shim._full_name("")
    key = (scope, base)
    n = _LAYER_COUNT[key]
    _LAYER_COUNT[key] += 1
    return base if n == 0 else "{}_{}".format(base, n)


def _var(name, shape, kind="normal"):
    full = shim._full_name(name)
    if full not in shim.VARIABLES:
        rng = shim.AUTO[0]
        value = rng.randn(*shape) * 0.3
        if kind == "positive":
            value = np.abs(value) + 0.5
        elif kind == "ones":
            value = value + 1.0
        shim.VARIABLES[full] = np.asarray(value, np.float32)
    return np.asarray(shim.VARIABLES[full], np.float64)


def _same_pads(size, k, stride):
    out = -(-size // stride)
    total = max((out - 1) * stride + k - size, 0)
    return total // 2, total - total // 2


def _conv2d(inputs, filters, kernel_size, strides=1, padding="valid", activation=None, **kwargs):
    assert strides in (1, (1, 1))
    x = np.asarray(inputs, np.float64)
    k = int(kernel_size)
    name = _layer_name("conv2d")
    with shim._scope_cm(name):
        w = _var("kernel", (k, k, x.shape[3], filters))
        b = _var("bias", (filters,))
    if padding == "same":
        pt, pb = _same_pads(x.shape[1], k, 1)
        pl, pr = _same_pads(x.shape[2], k, 1)
        x = np.pad(x, ((0, 0), (pt, pb), (pl, pr), (0, 0)))
    ho, wo = x.shape[1] - k + 1, x.shape[2] - k + 1
    out = np.zeros((x.shape[0], ho, wo, filters))
    for ky in range(k):
        for kx in range(k):
            out += x[:, ky:ky + ho, kx:kx + wo, :] @ w[ky, kx]
    out = shim.t(out + b, np.float64)
    return activation(out) if activation is not None else out


def _batch_normalization(inputs, training=False, **kwargs):
    x = np.asarray(inputs, np.float64)
    c = x.shape[-1]
    name = _layer_name("batch_normalization")
    with shim._scope_cm(name):
        gamma, beta = _var("gamma", (c,), "ones"), _var("beta", (c,))
        mean_name, var_name = shim._full_name("moving_mean"), shim._full_name("moving_variance")
        moving_mean, moving_var = _var("moving_mean", (c,)), _var("moving_variance", (c,), "positive")
    if training:
        mean = x.mean(axis=(0, 1, 2))
        var = ((x - mean) ** 2).mean(axis=(0, 1, 2))
        p = x.size // c
        MOVING_AFTER[mean_name] = 0.99 * moving_mean + 0.01 * mean
        MOVING_AFTER[var_name] = 0.99 * moving_var + 0.01 * var * p / (p - 1)
    else:
        mean, var = moving_mean, moving_var
    return shim.t(gamma * (x - mean) / np.sqrt(var + 1e-3) + beta, np.float64)


def _pool(x, k, stride, padding, is_max):
    x = np.asarray(x, np.float64)
    n, h, w, c = x.shape
    if padding == "same":
        (pt, pb), (pl, pr) = _same_pads(h, k, stride), _same_pads(w, k, stride)
        ho, wo = -(-h // stride), -(-w // stride)
    else:
        pt = pb = pl = pr = 0
        ho, wo = (h - k) // stride + 1, (w - k) // stride + 1
    out = np.zeros((n, ho, wo, c))
    for i in range(ho):
        for j in range(wo):
            y0, x0 = i * stride - pt, j * stride - pl
            win = x[:, max(y0, 0):min(y0 + k, h), max(x0, 0):min(x0 + k, w), :]
            out[:, i, j, :] = win.max(axis=(1, 2)) if is_max else win.mean(axis=(1, 2))
    return shim.t(out, np.float64)


def _adadelta(rng):
    """Three steps of tf.train.AdadeltaOptimizer (ApplyAdadelta) at str.ini's rho / epsilon, a larger lr."""
    lr, rho, eps = 0.5, 0.95, 1e-6
    var = var0 = rng.randn(3, 5)
    accum, accum_update = np.zeros_like(var), np.zeros_like(var)
    grads, trajectory = rng.randn(3, 3, 5), []
    for g in grads:
        accum = rho * accum + (1 - rho) * g * g
        update = np.sqrt(accum_update + eps) / np.sqrt(accum + eps) * g
        accum_update = rho * accum_update + (1 - rho) * update * update
        var = var - lr * update
        trajectory.append(var)
    return {"adadelta_var0": var0, "adadelta_grads": grads, "adadelta_trajectory": np.stack(trajectory), "adadelta_lr": lr,
            "adadelta_rho": rho, "adadelta_eps": eps}


def main():
    install_stubs()
    tf = shim.install()
    tf.layers.conv2d = _conv2d
    tf.layers.batch_normalization = _batch_normalization
    tf.layers.max_pooling2d = lambda x, pool_size, strides, padding="valid", **k: _pool(x, pool_size, strides,
                                                                                         padding, True)
    tf.layers.average_pooling2d = lambda x, pool_size, strides, padding="valid", **k: _pool(x, pool_size, strides,
                                                                                             padding, False)
    tf.sign = lambda x: shim.t(np.sign(np.asarray(x)))
    tf.greater = lambda a, b: shim.t(np.greater(np.asarray(a), b))
    tf.to_float = lambda x: shim.t(np.asarray(x, np.float64))
    sys.path.insert(0, REFERENCE)
    from neuralmonkey.encoders.cnn_encoder import CNNEncoder, CNNTemporalView
    from neuralmonkey.readers.image_reader import image_reader

    rng = np.random.RandomState(31)
    out = {}
    for tag, convolutions, (h, w, c), bn, fc in CASES:
        images = rng.randint(0, 256, size=(BATCH, h, w, c)).astype(np.float64)
        images[:, :, -(w // 4):] = 0                  # a blank right margin: masked columns
        images[1, :, -(w // 2):] = 0
        out[tag + "_images"] = images
        shim.VARIABLES.clear()
        shim.AUTO[0] = np.random.RandomState(rng.randint(1 << 30))
        for mode in ("train", "eval"):
            MOVING_AFTER.clear()
            _LAYER_COUNT.clear()
            cnn = object.__new__(CNNEncoder)
            cnn.__dict__.update(dict(
                _variable_scope=shim.VarScope("cnn"), _reuse=None, _name="cnn", data_id="images",
                dropout_keep_prob=1.0, image_height=h, image_width=w, pixel_dim=c, convolutions=convolutions,
                fully_connected=fc, batch_normalize=bn, train_mode=mode == "train",
                _dataset={"images": shim.t(images / 255.0, np.float64)}))
            view = object.__new__(CNNTemporalView)
            view.__dict__.update(dict(_variable_scope=shim.VarScope("cnn_in_time"), _reuse=None,
                                      _name="cnn_in_time", _cnn=cnn))
            key = "{}_{}_".format(tag, mode)
            out[key + "spatial_states"] = np.asarray(cnn.spatial_states, np.float64)
            out[key + "spatial_mask"] = np.asarray(cnn.spatial_mask, np.float64)
            out[key + "output"] = np.asarray(cnn.output, np.float64)
            out[key + "temporal_states"] = np.asarray(view.temporal_states, np.float64)
            out[key + "temporal_mask"] = np.asarray(view.temporal_mask, np.float64)
            if mode == "train":
                out[tag + "_variable_names"] = np.array(sorted(shim.VARIABLES))
                for name in sorted(shim.VARIABLES):
                    out[tag + "_var:" + name] = np.asarray(shim.VARIABLES[name])
                for name in sorted(MOVING_AFTER):
                    out[tag + "_moving_after:" + name] = MOVING_AFTER[name]
    out.update(_adadelta(rng))

    prefix = os.path.join(REFERENCE, "tests/data/str")
    list_file = os.path.join(HERE, "_str_golden_files.txt")
    names = open(os.path.join(prefix, "val_files.txt")).read().split()[:4]
    with open(list_file, "w") as handle:
        handle.write("\n".join(names) + "\n")
    readers = {"rescale": dict(pad_w=256, pad_h=32, channels=1, rescale_w=True, rescale_h=True, mode="F"),
               "aspect": dict(pad_w=256, pad_h=32, channels=1, rescale_w=True, rescale_h=True,
                              keep_aspect_ratio=True, mode="L"),
               "crop": dict(pad_w=20, pad_h=10, channels=3)}
    try:
        for tag, kwargs in readers.items():
            images = list(image_reader(prefix=prefix, **kwargs)([list_file]))
            out["reader_" + tag] = np.stack(images).astype(np.float32)
    finally:
        os.remove(list_file)
    out["reader_files"] = np.array(names)
    np.savez_compressed(os.path.join(HERE, "cnn_golden.npz"), **out)
    print("wrote", os.path.join(HERE, "cnn_golden.npz"), len(out), "arrays")


if __name__ == "__main__":
    main()
