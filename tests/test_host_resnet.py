"""The ResNet-v2 image encoders' host side on the CPU: the fp64 oracle of tests/resnet_oracle.py against hand-computed
values, end points, shapes and variables of all three depths, constructor errors, and the model part over a CPU
stand-in of ops.conv2d_bn_fwd against the oracle.  The kernels are tested in tests/test_gpu_resnet.py."""
import pytest
import torch

from tests import resnet_oracle as RO

NETS = ["resnet_v2_50", "resnet_v2_101", "resnet_v2_152"]


def test_oracle_conv2d_same_stride_2_by_hand():
    """5x5 input, 3x3 window of ones, stride 2: pads 1 before and 1 after, windows at rows/cols -1, 1, 3."""
    x = torch.arange(25, dtype=torch.float64).view(1, 1, 5, 5)
    w = torch.ones(3, 3, 1, 1, dtype=torch.float64)
    got = RO.conv2d_same(x, w, 2)[0, 0]

    def window(r, c):
        return sum(5 * i + j for i in range(r - 1, r + 2) for j in range(c - 1, c + 2) if 0 <= i < 5 and 0 <= j < 5)
    want = torch.tensor([[window(r, c) for c in (0, 2, 4)] for r in (0, 2, 4)], dtype=torch.float64)
    assert torch.equal(got, want)
    assert float(got[0, 0]) == 0 + 1 + 5 + 6
    # a 4x4 input at stride 2 has the same pads (1, 1), unlike TF's SAME (0 before, 1 after)
    x4 = torch.arange(16, dtype=torch.float64).view(1, 1, 4, 4)
    assert float(RO.conv2d_same(x4, w, 2)[0, 0, 0, 0]) == 0 + 1 + 4 + 5


def test_oracle_same_max_pool_odd_size_by_hand():
    """5x5, 3x3/2 SAME: 3x3 output, pad total (3-1)*2+3-5 = 2 -> 1 before, 1 after; -inf never wins."""
    x = -torch.arange(25, dtype=torch.float64).view(1, 1, 5, 5) - 1.0
    got = RO.max_pool_same(x, 3, 2)[0, 0]
    want = torch.tensor([[-1, -2, -4], [-6, -7, -9], [-16, -17, -19]], dtype=torch.float64)
    assert torch.equal(got, want)
    # 6x6: pad total (3-1)*2+3-6 = 1 -> 0 before, 1 after
    y = torch.arange(36, dtype=torch.float64).view(1, 1, 6, 6)
    assert torch.equal(RO.max_pool_same(y, 3, 2)[0, 0], torch.tensor([[14, 16, 17], [26, 28, 29], [32, 34, 35]],
                                                                      dtype=torch.float64))


def _count(net):
    """slim's end points: conv1, 3 convs + the unit per unit, a conv shortcut where the depth changes (the first
    unit of each block), one per block."""
    units = RO.units(net)
    return 1 + sum(4 + (din != depth) for _s, din, depth, _b, _st, _l in units) + len(RO.BLOCKS[net])


@pytest.mark.parametrize("net", NETS)
def test_end_points_and_count(net):
    from neuralmonkey_b200.encoders.imagenet_encoder import resnet_layers
    names = [l[0] for l in resnet_layers(net)]
    assert names == RO.end_point_names(net)
    assert len(names) == _count(net) == len(set(names))
    assert names[:7] == [net + "/conv1"] + [net + "/block1/unit_1/bottleneck_v2/" + c
                                            for c in ("shortcut", "conv1", "conv2", "conv3")] + [
        net + "/block1/unit_1/bottleneck_v2", net + "/block1/unit_2/bottleneck_v2/conv1"]
    assert names[-2:] == [net + "/block4/unit_3/bottleneck_v2", net + "/block4"]
    assert sum(n.endswith("/shortcut") for n in names) == 4


@pytest.mark.parametrize("net", NETS)
@pytest.mark.parametrize("size,sides", [(229, (115, 58, 29, 15, 8, 8)), (224, (112, 56, 28, 14, 7, 7))])
def test_shape_table(net, size, sides):
    """The end-point shapes, on the meta device (no arithmetic)."""
    p = {n: torch.empty(s, device="meta", dtype=torch.float64) for n, s in RO.variable_shapes(net).items()}
    images = torch.empty(1, size, size, 3, device="meta", dtype=torch.float64)
    points = RO.resnet_v2(p, net, images)
    assert list(points) == RO.end_point_names(net)
    assert points[net + "/conv1"].shape == (1, sides[0], sides[0], 64)
    assert RO.max_pool_same(torch.empty(1, 64, sides[0], sides[0], device="meta"), 3, 2).shape[2] == sides[1]
    for b, (side, depth) in enumerate(zip(sides[2:], (256, 512, 1024, 2048)), 1):
        assert points["{}/block{}".format(net, b)].shape == (1, side, side, depth)
    from neuralmonkey_b200.encoders.imagenet_encoder import resnet_layers
    for name, channels, _vars in resnet_layers(net):
        assert points[name].shape[3] == channels, name


@pytest.mark.parametrize("net", NETS)
def test_variables(net):
    from neuralmonkey_b200.encoders.imagenet_encoder import resnet_layers
    declared = {}
    for _name, _channels, variables in resnet_layers(net):
        for var, shape in variables:
            assert var not in declared, var
            declared[var] = tuple(shape)
    assert declared == RO.variable_shapes(net)
    shortcuts = sorted(v for v in declared if v.endswith("/shortcut/weights"))
    assert shortcuts == ["{}/block{}/unit_1/bottleneck_v2/shortcut/weights".format(net, b) for b in range(1, 5)]
    assert declared[net + "/block1/unit_1/bottleneck_v2/shortcut/weights"] == (1, 1, 64, 256)
    assert declared[net + "/block2/unit_1/bottleneck_v2/preact/gamma"] == (256,)
    assert declared[net + "/block4/unit_3/bottleneck_v2/conv2/weights"] == (3, 3, 512, 512)
    assert not any(v.endswith("conv2/biases") or v.endswith("conv1/biases") and "/block" in v for v in declared)


@pytest.fixture
def cpu_resnet(monkeypatch):
    from neuralmonkey_b200 import ops, runtime
    from tests import cnn_oracle as CO
    monkeypatch.setattr(ops, "conv2d_bn_fwd", conv2d_bn_fwd_stand_in)
    monkeypatch.setattr(ops, "pool2d", CO.pool2d)
    monkeypatch.setattr(runtime, "_device", torch.device("cpu"))
    runtime.reset()
    yield
    runtime.reset()


def conv2d_bn_fwd_stand_in(x, w, **kwargs):
    """ops.conv2d_bn_fwd on the CPU: the oracle's fp64 restatement of the op, rounded to fp32."""
    return RO.conv2d_bn(x, w, **kwargs).float()


def _encoder(net, layer):
    from neuralmonkey_b200 import runtime
    from neuralmonkey_b200.encoders import ImageNet
    enc = ImageNet(name="imagenet", data_id="images", network_type=net, spatial_layer=layer)
    enc.ensure_declared()
    runtime.arena().finalize(runtime.device())
    return enc


@pytest.mark.parametrize("net,layer,size", [
    ("resnet_v2_50", "resnet_v2_50/conv1", 9),
    ("resnet_v2_50", "resnet_v2_50/block1/unit_1/bottleneck_v2/shortcut", 13),
    ("resnet_v2_50", "resnet_v2_50/block1/unit_3/bottleneck_v2/conv2", 13),
    ("resnet_v2_50", "resnet_v2_50/block2/unit_1/bottleneck_v2/conv3", 21),
    ("resnet_v2_50", "resnet_v2_50/block2", 21),
    ("resnet_v2_101", "resnet_v2_101/block3", 19),
    ("resnet_v2_152", "resnet_v2_152/block4", 23),
])
def test_model_part_over_the_stand_in_against_the_oracle(cpu_resnet, net, layer, size):
    from neuralmonkey_b200 import runtime
    enc = _encoder(net, layer)
    arena = runtime.arena()
    params = RO.random_params(net, seed=3)
    declared = set(arena.order)
    assert declared <= set(params)
    # only the variables up to the end point, none of them trainable
    assert not declared & set(arena.train_names)
    names = RO.end_point_names(net)
    needed = RO.resnet_v2({n: torch.empty(s, device="meta") for n, s in RO.variable_shapes(net).items()}, net,
                          torch.empty(1, size, size, 3, device="meta"), layer)
    assert list(needed) == names[:names.index(layer) + 1]
    arena.load_dict({n: params[n].float() for n in declared})
    images = torch.randn(2, size, size, 3, generator=torch.Generator().manual_seed(size), dtype=torch.float64)
    enc.feed_images(images.float())
    want = RO.resnet_v2({n: params[n].float().double() for n in declared}, net, images.float().double(), layer)[layer]
    got = enc.spatial_states
    assert got.shape == want.shape
    scale = float(want.abs().max())
    assert float((got.double() - want).abs().max()) < 1e-5 * scale
    assert torch.allclose(enc.output.double(), want.mean(dim=(1, 2)), atol=1e-5 * scale)
    assert enc.spatial_mask.shape == got.shape[:3] and float(enc.spatial_mask.min()) == 1.0
    assert enc.dimension == got.shape[3]
    assert (enc.height, enc.width) == (229, 229)


@pytest.mark.parametrize("kwargs,error,message", [
    ({"network_type": "resnet_v2_18"}, ValueError, "not among the supported"),
    ({"network_type": "alexnet_v2"}, NotImplementedError, "resnet_v2_50"),
    ({"network_type": "resnet_v2_50", "spatial_layer": "resnet_v2_50/pool1"}, ValueError,
     "does not contain endpoint 'resnet_v2_50/pool1'"),
    ({"network_type": "resnet_v2_50", "spatial_layer": "resnet_v2_50/block2/unit_1/bottleneck_v2/preact"},
     ValueError, "does not contain endpoint"),
    ({"network_type": "resnet_v2_50", "spatial_layer": "resnet_v2_50/block2/unit_2/bottleneck_v2/shortcut"},
     ValueError, "does not contain endpoint"),
    ({"network_type": "resnet_v2_50", "spatial_layer": "resnet_v2_50/postnorm"}, ValueError,
     "does not contain endpoint"),
    ({"network_type": "resnet_v2_101", "spatial_layer": "resnet_v2_50/block4"}, ValueError,
     "does not contain endpoint"),
    ({"network_type": "resnet_v2_50", "spatial_layer": "resnet_v2_50/block4", "encoded_layer": "resnet_v2_50/logits"},
     NotImplementedError, "encoded_layer"),
])
def test_constructor_errors(kwargs, error, message):
    from neuralmonkey_b200.encoders import ImageNet
    with pytest.raises(error, match=message):
        ImageNet(name="imagenet", data_id="images", **kwargs)

