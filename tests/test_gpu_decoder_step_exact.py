"""The fused attention-decoder step (csrc/decoder_step.cu) exactly at every branch of its launch plan: each named case
of tests/decoder_step_plan.py, searched at this device's SM count, against an fp64 restatement of the step computed on
the device.  Also every output written and nothing past `rows`, misaligned bases, masks down to a fully masked
encoder row, saturated attention energies, every parent index, optional outputs, repeat calls, the refusals (raised
before any launch) and the decoding engine stepping instead of the kernel where the kernel refuses the shape."""
import pytest
import torch

from tests import decoder_step_plan as P
from tests.helpers import build_bahdanau, feed, max_abs, oracle_params_for, random_batch
from tests.test_gpu_decode import _run_step, _step_inputs, _step_reference

pytestmark = pytest.mark.gpu

TOL = 3e-5
SPARE = 8          # rows past `rows` in every output buffer: must stay NaN
WEIGHT_BASES = ("wg", "wc", "wq", "wo", "keys", "values")


def _sms() -> int:
    return torch.cuda.get_device_properties(0).multi_processor_count


def _dims(d: P.Dims, masked=True):
    return (d.rows, d.group, d.E, d.H, d.A, d.C, d.Tx, d.O, d.maxout, masked)


def _supported(d: P.Dims, aligned=True) -> bool:
    from neuralmonkey_b200 import lib
    return bool(lib.load().nm_attn_decoder_step_supported(d.rows, d.group, d.E, d.H, d.A, d.C, d.Tx, d.O,
                                                          int(d.maxout), int(aligned)))


def _inputs(dims):
    """_step_inputs on the device, every product's weights scaled to a fan-in of at most 256: the 3e-5 tolerance
    then holds for fp32 sums over thousands of terms as it does at the en-de sizes."""
    p, symbols, h_prev, parent = _step_inputs(dims, "cuda")
    rows, group, E, H, A, C, Tx, O = dims[:8]
    for k, fan_in in (("wg", E + H), ("wc", E + H), ("wq", H), ("v", A), ("wo", H + E + C)):
        p[k] *= min(1.0, (256.0 / fan_in) ** 0.5)
    return p, symbols, h_prev, parent


def _misaligned(t: torch.Tensor) -> torch.Tensor:
    """A copy of `t` whose base is one float past a 16-byte boundary."""
    buf = torch.empty(t.numel() + 4, device=t.device)
    view = buf[1:1 + t.numel()].view(t.shape)
    view.copy_(t)
    return view


def _use_cluster(monkeypatch, cl):
    monkeypatch.setenv("NMB200_DECSTEP_CLUSTER", str(cl) if cl else "")


def _check(dims, p, symbols, h_prev, parent, act="tanh"):
    """Launch with NaN-filled outputs; every element of the first `rows` rows matches fp64, none past them is
    written, and the embedded input is the table row bit for bit."""
    rows = dims[0]
    want = dict(zip(("h", "ctx", "w", "out"), _step_reference(p, symbols, h_prev, parent, dims[1], act)))
    got = _run_step(dims, p, symbols, h_prev, parent, act, spare=SPARE)
    for name, ref in want.items():
        assert not torch.isnan(got[name][:rows]).any(), name
        assert max_abs(got[name][:rows], ref) < TOL, (name, max_abs(got[name][:rows], ref))
    assert torch.equal(got["x"][:rows], p["table"][symbols])
    for name, buf in got.items():
        assert torch.isnan(buf[rows:]).all(), "{} written past rows".format(name)
    return got


# ---- every branch of the plan ----------------------------------------------------------------------------------

@pytest.mark.parametrize("case", [c for c in P.CASES if c.near is None], ids=lambda c: c.name)
def test_case_against_fp64(monkeypatch, case):
    d = P.find_shape(case, _sms())
    _use_cluster(monkeypatch, case.cl)
    assert _supported(d, case.aligned)
    p, symbols, h_prev, parent = _inputs(_dims(d))
    if not case.aligned:
        for k in WEIGHT_BASES:
            p[k] = _misaligned(p[k])
    _check(_dims(d), p, symbols, h_prev, parent)


def test_restatement_matches_the_library(monkeypatch):
    """nm_attn_decoder_step_supported agrees with the restated plan over a grid of shapes and cluster sizes."""
    sms = _sms()
    for cl in (None, 1, 2, 4, 8):
        _use_cluster(monkeypatch, cl)
        for rows in (1, 21, 8 * sms + 5):
            for E, H, A, C, O in ((32, 32, 64, 48, 32), (33, 32, 64, 512, 32), (33, 32, 64, 513, 32),
                                  (32, 32, 64, 2048, 32), (32, 32, 64, 2052, 32), (300, 300, 600, 600, 300),
                                  (32, 900, 2048, 2048, 1024), (32, 904, 2048, 2048, 1024)):
                for Tx in (1, 50, 1000, 3000, 6440, 20000):
                    for maxout in (False, True):
                        for aligned in (False, True):
                            d = P.Dims(rows, 1, E, H, A, C, Tx, O, maxout)
                            want = P.plan(d, sms, aligned, cl).refusal is None
                            assert _supported(d, aligned) == want, (d, aligned, cl)
    for case in P.CASES:
        _use_cluster(monkeypatch, case.cl)
        d = P.find_shape(case, sms)
        assert _supported(d, case.aligned) == (case.near is None), case.name


# ---- refusals ------------------------------------------------------------------------------------------------

@pytest.mark.parametrize("case", [c for c in P.CASES if c.near is not None], ids=lambda c: c.name)
def test_refusal_before_launch_and_the_shape_next_to_it(monkeypatch, case):
    from neuralmonkey_b200 import lib
    d = P.find_shape(case, _sms())
    _use_cluster(monkeypatch, case.cl)
    assert not _supported(d) and _supported(case.near(d))
    dims = _dims(d)
    p, symbols, h_prev, parent = _inputs(dims)
    res = {name: torch.full((d.rows, w), float("nan"), device="cuda")
           for name, w in (("h", d.H), ("out", d.O), ("x", d.E), ("ctx", d.C), ("w", d.Tx))}
    torch.cuda.synchronize()
    before = lib.launch_count()
    with pytest.raises(ValueError):
        _run_step(dims, p, symbols, h_prev, parent, res=res)
    assert lib.launch_count() == before
    assert all(torch.isnan(t).all() for t in res.values())
    near = _dims(case.near(d))
    _check(near, *_inputs(near))


# ---- bases, masks, saturation, parents, outputs ------------------------------------------------------------------

VEC = P.Dims(21, 1, 32, 32, 64, 48, 13, 32, False)
SCALAR = P.Dims(21, 1, 33, 32, 64, 48, 13, 32, False)


@pytest.mark.parametrize("base", WEIGHT_BASES)
def test_one_misaligned_base_takes_the_scalar_variant(monkeypatch, base):
    """One base off by a float: the scalar variant runs (bit for bit the result with all six misaligned) and
    matches fp64."""
    _use_cluster(monkeypatch, None)
    dims = _dims(VEC)
    p, symbols, h_prev, parent = _inputs(dims)
    everything = dict(p, **{k: _misaligned(p[k]) for k in WEIGHT_BASES})
    ref = _run_step(dims, everything, symbols, h_prev, parent)
    one = dict(p, **{base: _misaligned(p[base])})
    got = _check(dims, one, symbols, h_prev, parent)
    for name in ref:
        assert torch.equal(got[name][:VEC.rows], ref[name]), name


@pytest.mark.parametrize("shape", [VEC, SCALAR], ids=["vector", "scalar"])
@pytest.mark.parametrize("kind", ["none", "partial", "one_valid_key", "fully_masked_row"])
def test_masks(monkeypatch, shape, kind):
    _use_cluster(monkeypatch, None)
    d = shape._replace(rows=24, group=3)
    dims = _dims(d)
    p, symbols, h_prev, parent = _inputs(dims)
    nb, tx = d.rows // d.group, d.Tx
    if kind == "none":
        p["mask"] = None
    else:
        lens = torch.tensor([tx, 5, 1, tx - 1, 3, 7, 2, 9][:nb], device="cuda")
        if kind == "one_valid_key":
            lens[:] = 1
        p["mask"] = (torch.arange(tx, device="cuda")[None, :] < lens[:, None]).float()
        if kind == "one_valid_key":      # the valid key last in one row
            p["mask"][1] = 0.0
            p["mask"][1, tx - 1] = 1.0
        if kind == "fully_masked_row":
            p["mask"][2] = 0.0
    got = _check(dims, p, symbols, h_prev, parent)
    if kind == "fully_masked_row":   # softmax * 0 / (0 + 1e-8)
        rows = slice(2 * d.group, 3 * d.group)
        assert torch.equal(got["w"][rows], torch.zeros_like(got["w"][rows]))
        assert torch.equal(got["ctx"][rows], torch.zeros_like(got["ctx"][rows]))


@pytest.mark.parametrize("shape", [VEC, SCALAR], ids=["vector", "scalar"])
def test_saturated_energies(monkeypatch, shape):
    """|keys + query| beyond 44 (where exp(2x) of the fast tanh overflows) in single encoder rows: finite, and as
    fp64."""
    _use_cluster(monkeypatch, None)
    dims = _dims(shape)
    p, symbols, h_prev, parent = _inputs(dims)
    p["keys"][3] *= 150.0
    p["keys"][7, :, : shape.A // 2] = 60.0
    p["keys"][7, :, shape.A // 2:] = -60.0
    got = _check(dims, p, symbols, h_prev, parent)
    for name in ("h", "ctx", "w", "out"):
        assert torch.isfinite(got[name][:shape.rows]).all(), name


@pytest.mark.parametrize("shape", [VEC, SCALAR], ids=["vector", "scalar"])
@pytest.mark.parametrize("group", [1, 3, 8, 16])
def test_every_parent_index(monkeypatch, shape, group):
    _use_cluster(monkeypatch, None)
    d = shape._replace(rows=3 * group, group=group)
    dims = _dims(d)
    p, symbols, h_prev, _ = _inputs(dims)
    r = torch.arange(d.rows, device="cuda")
    for shift in range(group):       # every hypothesis of every sentence continues every parent once
        parent = ((r + shift) % group).int()
        _check(dims, p, symbols, h_prev, parent)


@pytest.mark.parametrize("shape", [VEC, SCALAR], ids=["vector", "scalar"])
@pytest.mark.parametrize("missing", ["x", "ctx", "w"])
def test_optional_output_null(monkeypatch, shape, missing):
    """One optional output NULL at a time: the others bit for bit the full launch's."""
    _use_cluster(monkeypatch, None)
    dims = _dims(shape)
    p, symbols, h_prev, parent = _inputs(dims)
    full = _run_step(dims, p, symbols, h_prev, parent)
    got = _run_step(dims, p, symbols, h_prev, parent, outputs=tuple(n for n in ("x", "ctx", "w") if n != missing))
    assert set(got) == set(full) - {missing}
    for name in got:
        assert torch.equal(got[name], full[name]), name


@pytest.mark.parametrize("name", ["ende_beam_cl1", "scalar_odd_C", "tcv_1"])
def test_repeat_calls_are_bit_identical(monkeypatch, name):
    case = next(c for c in P.CASES if c.name == name)
    d = P.find_shape(case, _sms())
    _use_cluster(monkeypatch, case.cl)
    dims = _dims(d)
    args = _inputs(dims)
    first = _run_step(dims, *args)
    for _ in range(2):
        again = _run_step(dims, *args)
        for k in first:
            assert torch.equal(again[k], first[k]), k


# ---- the decoding engine where the kernel refuses the shape --------------------------------------------------------

# C = 2 x 301 = 602: scalar variant (C % 4 != 0), wider than its 512-column context
WIDE = dict(vs=60, vt=70, es=11, he=301, et=9, hd=8, out=9, maxout=True, max_len=10, supress_unk=True)
NARROW = dict(WIDE, he=7)


def _model(cfg, bsz, seed):
    from neuralmonkey_b200 import ops
    ops.set_gemm_backend("simt")
    model = build_bahdanau(**cfg)
    model["arena"].load_dict(oracle_params_for(model))
    src, tgt = random_batch(bsz, 8, 7, cfg["vs"], cfg["vt"], seed=seed)
    return model, src, tgt


@pytest.mark.parametrize("cfg,fused", [(WIDE, False), (NARROW, True)], ids=["refused", "supported"])
def test_engine_greedy_steps_where_the_kernel_refuses(cfg, fused):
    from neuralmonkey_b200 import ops
    try:
        model, src, tgt = _model(cfg, 5, seed=3)
        dec = model["dec"]
        dec.use_fused_decoding = False
        feed(model, src, tgt, train=False)
        base = {k: getattr(dec, k).clone() for k in ("runtime_symbols", "runtime_mask", "runtime_loss")}
        dec.use_fused_decoding = True
        feed(model, src, tgt, train=False)
        assert torch.equal(dec.runtime_symbols, base["runtime_symbols"])
        assert torch.equal(dec.runtime_mask, base["runtime_mask"])
        assert abs(float(dec.runtime_loss) - float(base["runtime_loss"])) < 1e-4
        engine = dec.decode_engine
        assert engine is not None and engine.fits(5, 1) == fused
        assert bool(engine.bufs) == fused        # the engine allocated (and ran) only for the supported shape
    finally:
        ops.set_gemm_backend("auto")


@pytest.mark.parametrize("cfg,fused", [(WIDE, False), (NARROW, True)], ids=["refused", "supported"])
def test_engine_beam_steps_where_the_kernel_refuses(cfg, fused):
    from neuralmonkey_b200 import lib, ops
    from neuralmonkey_b200.decoders import BeamSearchDecoder
    try:
        model, src, _ = _model(cfg, 3, seed=4)
        bs = BeamSearchDecoder(name="bs", parent_decoder=model["dec"], beam_size=4, max_steps=7,
                               length_normalization=0.6)
        bs.use_fused_step = False
        feed(model, src, None, train=False)
        bs.reset_batch()
        base = bs.outputs
        bs.use_fused_step = True
        feed(model, src, None, train=False)
        bs.reset_batch()
        before = lib.launch_count()
        got = bs.outputs
        engine = model["dec"].decode_engine
        assert lib.launch_count() > before and engine.fits(12, 4) == fused
        assert bool(engine.bufs) == fused        # the engine allocated (and ran) only for the supported shape
        a, b = got.last_search_step_output, base.last_search_step_output
        assert torch.equal(a.token_ids, b.token_ids)
        assert max_abs(a.scores, b.scores) < 1e-5
        assert torch.equal(got.last_search_state.lengths, base.last_search_state.lengths)
    finally:
        ops.set_gemm_backend("auto")
