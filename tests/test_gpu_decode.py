"""The fused attention-decoder step (csrc/decoder_step.cu) and the decoding engine built on it
(decoders/rnn_decode.py): the kernel against an fp64 restatement of Decoder.next_state
(decoders/decoder.py:279-358 + attention/feed_forward.py:125-166 + output_projection.py:115-160 of the
reference) for every cluster size, and whole greedy / beam decodes against the step-by-step path and
the oracle - bit-exact on the integer side."""
import pytest
import torch

from oracle import nm_oracle as O
from tests.helpers import (build_bahdanau, feed, max_abs, oracle_params_for, oracle_spec, random_batch)

pytestmark = pytest.mark.gpu

TOY = dict(vs=60, vt=70, es=11, he=7, et=9, hd=8, out=9, maxout=True, max_len=10, supress_unk=True)
MID = dict(vs=120, vt=200, es=32, he=16, et=32, hd=32, out=32, maxout=False, max_len=12,
           supress_unk=False)


ACT_FN = {"none": lambda z: z, "tanh": torch.tanh, "relu": torch.relu, "sigmoid": torch.sigmoid}


def _step_reference(p, symbols, h_prev, parent, group, act="tanh", chunk=64):
    """fp64 restatement of one step for rows [rows]; p: dict of fp32 tensors, on the CPU or the device (computed
    there, the attention `chunk` rows at a time).  `act` is the activation of a dense output projection (ignored
    with maxout)."""
    d = {k: (v.double() if torch.is_tensor(v) and v.dtype == torch.float32 else v) for k, v in p.items()}
    rows, dev = symbols.shape[0], d["keys"].device
    x = d["table"][symbols]
    src = torch.arange(rows, device=dev)
    if parent is not None:
        src = (src // group) * group + parent.long()
    h = h_prev.double()[src]
    gates = torch.sigmoid(torch.cat([x, h], 1) @ d["wg"] + d["bg"])
    hd = h.shape[1]
    r, u = gates[:, :hd], gates[:, hd:]
    c = torch.tanh(torch.cat([x, r * h], 1) @ d["wc"] + d["bc"])
    hn = u * h + (1 - u) * c
    q = hn @ d["wq"] + d["bq"]
    ws, ctxs = [], []
    for s in range(0, rows, chunk):
        enc = torch.arange(s, min(rows, s + chunk), device=dev) // group
        e = (torch.tanh(d["keys"][enc] + q[s:s + chunk, None, :]) * d["v"]).sum(-1) + d["ab"]
        w = torch.softmax(e, -1)
        if d["mask"] is not None:
            w = w * d["mask"][enc]
            w = w / (w.sum(-1, keepdim=True) + 1e-8)
        ws.append(w)
        ctxs.append(torch.bmm(w[:, None, :], d["values"][enc])[:, 0])
    w, ctx = torch.cat(ws), torch.cat(ctxs)
    z = torch.cat([hn, x, ctx], 1) @ d["wo"] + d["bo"]
    if p["maxout"]:
        o = z.shape[1] // 2
        out = torch.maximum(z[:, :o], z[:, o:])
    else:
        out = ACT_FN[act](z)
    return hn, ctx, w, out


def _step_inputs(dims, device="cpu"):
    """Random parameters, symbols, previous states and parents of one step (fp32 tensors on `device`)."""
    rows, group, e, h, a, c, tx, o, maxout, masked = dims[:10]
    g = torch.Generator(device).manual_seed(rows * 7 + tx)
    vocab, nb = 50, rows // group

    def rnd(*shape, scale=0.3):
        return torch.randn(*shape, generator=g, device=device) * scale

    p = dict(table=rnd(vocab, e), wg=rnd(e + h, 2 * h), bg=rnd(2 * h) + 1.0, wc=rnd(e + h, h), bc=rnd(h),
             wq=rnd(h, a), bq=rnd(a), v=rnd(a), ab=rnd(1), keys=rnd(nb, tx, a, scale=0.7),
             values=rnd(nb, tx, c, scale=0.7), wo=rnd(h + e + c, (2 if maxout else 1) * o), bo=rnd((2 if maxout else 1) * o),
             maxout=maxout, mask=None)
    if masked:
        lens = torch.randint(1, tx + 1, (nb,), generator=g, device=device)
        lens[0] = tx
        p["mask"] = (torch.arange(tx, device=device)[None, :] < lens[:, None]).float()
    symbols = torch.randint(0, vocab, (rows,), generator=g, device=device)
    h_prev = rnd(rows, h, scale=0.5)
    parent = torch.randint(0, group, (rows,), generator=g, device=device).int() if group > 1 else None
    return p, symbols, h_prev, parent


def _run_step(dims, p, symbols, h_prev, parent, act="tanh", x_in=None, outputs=("x", "ctx", "w"), spare=0,
              res=None):
    """One nm_attn_decoder_step_fwd launch; symbols go through the table unless x_in [rows, E] is given.  The
    optional outputs not named in `outputs` are passed as NULL.  Returns {name: CUDA tensor} of NaN-filled outputs
    with `spare` rows past `rows` (or writes into `res`)."""
    from neuralmonkey_b200 import lib
    rows, group, e, h, a, c, tx, o, maxout, masked = dims[:10]
    dv = {k: (v.cuda() if torch.is_tensor(v) else v) for k, v in p.items()}
    if res is None:
        res = {name: torch.full((rows + spare, width), float("nan"), device="cuda")
               for name, width in (("h", h), ("out", o), ("x", e), ("ctx", c), ("w", tx))
               if name in ("h", "out") + tuple(outputs)}
    # held in variables until the launch has run: the kernel only gets their raw pointers
    sym_d, hp_d = symbols.cuda(), h_prev.cuda()
    x_d = x_in.cuda() if x_in is not None else None
    par_d = parent.cuda() if parent is not None else None
    lib.call("nm_attn_decoder_step_fwd", lib.ptr(sym_d), lib.ptr(dv["table"]), lib.ptr(x_d), lib.ptr(hp_d),
             lib.ptr(par_d),
             lib.ptr(dv["wg"]), lib.ptr(dv["bg"]), lib.ptr(dv["wc"]), lib.ptr(dv["bc"]), lib.ptr(dv["wq"]),
             lib.ptr(dv["bq"]), lib.ptr(dv["v"]), lib.ptr(dv["ab"]), lib.ptr(dv["keys"]), lib.ptr(dv["values"]),
             lib.ptr(dv["mask"]), lib.ptr(dv["wo"]), lib.ptr(dv["bo"]), lib.ptr(res.get("x")), lib.ptr(res["h"]),
             lib.ptr(res.get("ctx")), lib.ptr(res.get("w")), lib.ptr(res["out"]), rows, group, e, h, a, c, tx, o,
             lib.NM_ACT[act], int(maxout), lib.stream())
    torch.cuda.synchronize()
    return res


@pytest.mark.parametrize("cluster", ["", "1", "2", "4", "8"])
@pytest.mark.parametrize("dims", [
    # rows, group, E, H, A, C, Tx, O, maxout, masked, act of a dense output
    (5, 1, 9, 8, 14, 14, 7, 9, True, True, "tanh"),            # tests/bahdanau.ini dims: scalar variant
    (21, 1, 32, 32, 64, 48, 13, 32, False, True, "tanh"),      # 16-byte rows: TMA-staged tiles, ragged last cluster
    (24, 3, 32, 40, 64, 64, 50, 32, True, False, "tanh"),      # beam rows sharing an encoder row, no mask
    (64, 8, 300, 300, 600, 600, 50, 300, False, True, "tanh"),  # en-de dims, beam 8
    # every other activation of a dense output projection
    (21, 1, 32, 32, 64, 48, 13, 32, False, True, "none"),
    (21, 1, 32, 32, 64, 48, 13, 32, False, True, "relu"),
    (21, 1, 32, 32, 64, 48, 13, 32, False, True, "sigmoid"),
    (64, 8, 300, 300, 600, 600, 50, 300, False, True, "none"),
    (64, 8, 300, 300, 600, 600, 50, 300, False, True, "relu"),
    (64, 8, 300, 300, 600, 600, 50, 300, False, True, "sigmoid"),
    # scalar variant with beam rows and a parent gather, both output kinds
    (12, 3, 9, 8, 14, 14, 7, 9, True, True, "tanh"),
    (12, 3, 9, 8, 14, 14, 7, 9, False, False, "relu"),
])
def test_step_kernel_against_fp64(monkeypatch, dims, cluster):
    act = dims[10]
    monkeypatch.setenv("NMB200_DECSTEP_CLUSTER", cluster)
    p, symbols, h_prev, parent = _step_inputs(dims)
    want = _step_reference(p, symbols, h_prev, parent, dims[1], act)
    got = _run_step(dims, p, symbols, h_prev, parent, act)
    assert torch.equal(got["x"].cpu(), p["table"][symbols])
    tol = 3e-5
    assert max_abs(got["h"], want[0]) < tol
    assert max_abs(got["w"], want[2]) < tol
    assert max_abs(got["ctx"], want[1]) < tol
    assert max_abs(got["out"], want[3]) < tol


STEP_DIMS = [(21, 1, 32, 32, 64, 48, 13, 32, False, True),    # vector variant
             (12, 3, 9, 8, 14, 14, 7, 9, True, True)]         # scalar variant, parent gather


@pytest.mark.parametrize("dims", STEP_DIMS)
def test_step_kernel_x_in_equals_the_table_path(dims):
    """Already-embedded inputs (x_in) give bit for bit the step fed through the table; `symbols` is then
    ignored, so other (valid) ids may be passed beside it."""
    p, symbols, h_prev, parent = _step_inputs(dims)
    base = _run_step(dims, p, symbols, h_prev, parent)
    x_in = p["table"][symbols]
    got = _run_step(dims, p, (symbols + 1) % p["table"].shape[0], h_prev, parent, x_in=x_in)
    for name in base:
        assert torch.equal(got[name], base[name]), name
    assert torch.equal(got["x"].cpu(), x_in)


@pytest.mark.parametrize("dims", STEP_DIMS)
def test_step_kernel_without_optional_outputs(dims):
    """x_out, ctx_out and weights_out NULL (as the decoding engine calls it): h_out and out unchanged."""
    p, symbols, h_prev, parent = _step_inputs(dims)
    base = _run_step(dims, p, symbols, h_prev, parent)
    got = _run_step(dims, p, symbols, h_prev, parent, outputs=())
    assert set(got) == {"h", "out"}
    assert torch.equal(got["h"], base["h"]) and torch.equal(got["out"], base["out"])


def test_step_kernel_rejects_null_pointers():
    from neuralmonkey_b200 import lib
    with pytest.raises(ValueError):
        lib.call("nm_attn_decoder_step_fwd", None, None, None, None, None, None, None, None, None, None, None,
                 None, None, None, None, None, None, None, None, None, None, None, None, 4, 1, 8, 8, 8, 8, 8, 8, 1,
                 0, lib.stream())


def _setup(cfg, backend, bsz, tx, ty, seed):
    from neuralmonkey_b200 import ops
    ops.set_gemm_backend(backend)
    model = build_bahdanau(**cfg)
    params = oracle_params_for(model)
    model["arena"].load_dict(params)
    src, tgt = random_batch(bsz, tx, ty, cfg["vs"], cfg["vt"], seed=seed)
    return model, params, src, tgt


@pytest.mark.parametrize("cfg,backend", [(TOY, "simt"), (MID, "simt"), (MID, "auto"),
                                         (dict(MID, out_act="relu"), "simt")])
def test_fused_greedy_equals_the_stepwise_loop(cfg, backend):
    """Same symbols, masks, argmax and (to rounding) states / losses as the host loop over next_state; three
    decodes so that the CUDA-graph replay (from the second time a shape shows up) is compared too."""
    from neuralmonkey_b200 import lib, ops
    try:
        model, params, src, tgt = _setup(cfg, backend, 9, 8, 7, seed=5)
        dec = model["dec"]
        assert dec.decode_engine is not None
        dec.use_fused_decoding = False
        feed(model, src, tgt, train=False)
        base = {k: getattr(dec, k).clone() for k in
                ("runtime_symbols", "runtime_mask", "runtime_output_states", "runtime_logits", "runtime_xents",
                 "runtime_loss", "runtime_argmax", "decoded")}
        dec.use_fused_decoding = True
        for rep in range(3):
            feed(model, src, tgt, train=False)
            _ = model["att"].hidden_features, model["att"].attention_states, dec.initial_state   # encoder side
            before = lib.launch_count()
            sym = dec.runtime_symbols
            launched = lib.launch_count() - before
            steps = sym.shape[0]
            if backend == "simt":
                assert torch.equal(sym, base["runtime_symbols"]), rep
                assert torch.equal(dec.runtime_mask, base["runtime_mask"])
                assert torch.equal(dec.runtime_argmax, base["runtime_argmax"])
                assert max_abs(dec.runtime_output_states, base["runtime_output_states"]) < 2e-5
            else:
                # the step-by-step path runs its projections in TF32 and its recurrence on the tensor cores,
                # the fused step is exact fp32: same decode up to near-ties
                n = min(steps, base["runtime_symbols"].shape[0])
                assert float((sym[:n] == base["runtime_symbols"][:n]).float().mean()) > 0.9
                assert max_abs(dec.runtime_output_states[:1], base["runtime_output_states"][:1]) < 2e-2
                continue
            assert max_abs(dec.runtime_xents, base["runtime_xents"]) < (1e-4 if backend == "simt" else 2e-2)
            assert abs(float(dec.runtime_loss) - float(base["runtime_loss"])) < (1e-4 if backend == "simt" else 2e-2)
            keep = torch.ones(cfg["vt"], dtype=torch.bool)
            keep[3] = not cfg["supress_unk"]
            assert max_abs(dec.runtime_logits[..., keep.cuda()], base["runtime_logits"][..., keep.cuda()]) < (
                2e-5 if backend == "simt" else 2e-2)
            assert torch.equal(dec.decoded, base["decoded"]) or backend != "simt"
            if rep == 0:    # eager issue: three launches of libnmb200 per step (graph replays are not counted)
                chunk = dec.decode_engine.CHUNK
                issued = min(-(-steps // chunk) * chunk, cfg["max_len"])    # whole chunks of steps are issued
                assert launched == 3 * issued, (launched, steps)
    finally:
        ops.set_gemm_backend("auto")


def test_fused_greedy_against_the_oracle_bit_exact_symbols():
    from neuralmonkey_b200 import ops
    try:
        model, params, src, tgt = _setup(TOY, "simt", 7, 9, 8, seed=11)
        feed(model, src, tgt, train=False)
        dec = model["dec"]
        og = O.decoder_greedy(params, oracle_spec(), O.sentence_encoder(params, "sentence_encoder", src), tgt.t())
        assert torch.equal(dec.runtime_symbols.cpu(), og["output_symbols"])
        assert torch.equal(dec.runtime_mask.cpu(), og["runtime_mask"])
        assert abs(float(dec.runtime_loss) - float(og["runtime_loss"])) < 1e-4
        w = model["att"].histories["decoder_run"]          # [time, batch, Tx] attention weights of the run
        assert w.shape[0] == og["output_symbols"].shape[0] and w.shape[1] == src.shape[0]
        assert max_abs(w.sum(-1)[dec.runtime_mask], torch.ones_like(w.sum(-1)[dec.runtime_mask])) < 1e-4
    finally:
        ops.set_gemm_backend("auto")


@pytest.mark.parametrize("cfg,backend,bsz,beam,alpha", [(TOY, "simt", 1, 3, 0.6), (TOY, "simt", 4, 4, 1.0),
                                                        (MID, "simt", 5, 8, 0.0), (MID, "auto", 3, 5, 0.6),
                                                        (MID, "simt", 3, 16, 0.6)])
def test_fused_beam_search_equals_the_stepwise_loop(cfg, backend, bsz, beam, alpha):
    from neuralmonkey_b200 import ops
    from neuralmonkey_b200.decoders import BeamSearchDecoder
    try:
        model, params, src, tgt = _setup(cfg, backend, bsz, 8, 7, seed=21 + bsz)
        bs = BeamSearchDecoder(name="bs", parent_decoder=model["dec"], beam_size=beam, max_steps=9,
                               length_normalization=alpha)
        bs.use_fused_step = False
        feed(model, src, None, train=False)
        bs.reset_batch()
        base = bs.outputs
        bs.use_fused_step = True
        for rep in range(3):
            feed(model, src, None, train=False)
            bs.reset_batch()
            got = bs.outputs
            a, b = got.last_search_step_output, base.last_search_step_output
            if backend == "simt":
                assert torch.equal(a.token_ids, b.token_ids), rep
                assert torch.equal(got.last_search_state.lengths, base.last_search_state.lengths)
                assert torch.equal(got.last_search_state.finished, base.last_search_state.finished)
                assert max_abs(a.scores, b.scores) < 1e-5
                assert max_abs(got.last_search_state.logprob_sum, base.last_search_state.logprob_sum) < 1e-4
            else:
                # after a near-tie the two paths may pick other words and stop at other steps; the layout
                # [steps + 1, batch, beam] with at most max_steps = 9 search steps, and the id range, still hold
                assert a.token_ids.shape[1:] == b.token_ids.shape[1:] == (bsz, beam)
                assert 1 <= a.token_ids.shape[0] <= 10 and 1 <= b.token_ids.shape[0] <= 10
                assert 0 <= int(a.token_ids.min()) and int(a.token_ids.max()) < cfg["vt"]
                assert max_abs(a.scores[:, 0], b.scores[:, 0]) < 5e-2
    finally:
        ops.set_gemm_backend("auto")
