"""Differentiable host-side wrappers over the libnmb200 C ABI.

torch.autograd only *sequences* the calls: every forward and every backward is a
libnmb200 kernel launched on the current CUDA stream through ctypes.  Parameters
may carry an ``nm_grad`` attribute (a view into the flat gradient arena of
``neuralmonkey_b200.params.ParameterArena``); the backward passes then accumulate
weight gradients straight into that arena (GEMM epilogue ``beta = 1``) and return
``None`` to autograd, so no torch kernels run on the weight-gradient path.
"""
from typing import Optional, Sequence, Tuple

import ctypes

import torch

from neuralmonkey_b200 import lib
from neuralmonkey_b200.lib import call, ptr

_GEMM_BACKEND = lib.GEMM_AUTO


def set_gemm_backend(name: str) -> None:
    """'auto' (wgmma tensor cores when TMA-addressable), 'simt' (exact fp32) or 'tc'."""
    global _GEMM_BACKEND
    _GEMM_BACKEND = {"auto": lib.GEMM_AUTO, "simt": lib.GEMM_SIMT, "tc": lib.GEMM_TC}[name]


def gemm_backend() -> int:
    return _GEMM_BACKEND


def _f32(t: torch.Tensor) -> torch.Tensor:
    if t.dtype != torch.float32:
        raise TypeError("expected float32, got {}".format(t.dtype))
    return t


def _rows(t: torch.Tensor) -> Tuple[torch.Tensor, int]:
    """2-D view with unit inner stride; returns (tensor, leading dimension)."""
    if t.dim() != 2:
        raise ValueError("expected a 2-D tensor")
    if t.stride(1) != 1 and t.size(1) != 1:
        t = t.contiguous()
    ld = t.stride(0) if t.size(0) > 1 else max(t.size(1), t.stride(0))
    if ld < t.size(1):
        t = t.contiguous()
        ld = t.size(1)
    return t, ld


def kmajor_tf32(t: torch.Tensor) -> torch.Tensor:
    """t^T rounded to TF32 (cvt.rna): a [cols, rows] view of a fresh buffer whose row pitch is a multiple of 4 floats
    (nm_transpose_tf32).  The K-major form of a GEMM operand whose reduction dimension is strided."""
    t, ld = _rows(_f32(t))
    rows, cols = t.shape
    ld_t = (rows + 3) // 4 * 4
    buf = torch.empty(cols, ld_t, device=t.device, dtype=torch.float32)
    call("nm_transpose_tf32", ptr(t), ld, ptr(buf), ld_t, rows, cols, lib.stream())
    return buf[:, :rows]


def _on_tensor_cores(trans_a: bool, trans_b: bool, m: int, n: int, k: int, a: torch.Tensor, lda: int,
                     b: torch.Tensor, ldb: int, backend: int) -> bool:
    """nm_gemm's own choice of engine: wgmma unless the backend is the exact one or the operands are not
    TMA-addressable (row pitches multiples of 4 floats, 16-byte aligned bases)."""
    return (backend != lib.GEMM_SIMT and m > 0 and n > 0 and k > 0
            and lib.load().nm_gemm_uses_tc(int(trans_a), int(trans_b), m, n, k, lda, ldb, n) == 1
            and a.data_ptr() % 16 == 0 and b.data_ptr() % 16 == 0)


def _tn_on_tensor_cores(x: torch.Tensor, dy: torch.Tensor) -> bool:
    """Whether the weight-gradient product x^T . dy (both stored [K, *]) runs on the tensor cores."""
    x, ldx = _rows(x)
    dy, ldy = _rows(dy)
    return _on_tensor_cores(True, False, x.size(1), dy.size(1), x.size(0), x, ldx, dy, ldy, _GEMM_BACKEND)


def gemm(a: torch.Tensor, b: torch.Tensor, out: torch.Tensor, trans_a: bool = False,
         trans_b: bool = False, bias: Optional[torch.Tensor] = None, act: Optional[str] = None,
         beta: float = 0.0, backend: Optional[int] = None) -> torch.Tensor:
    """out = act(op(a) @ op(b) + bias) + beta*out, all through nm_gemm (no torch math).

    On the tensor-core path an operand stored MN-major (a with trans_a, b without trans_b) is handed over as its
    K-major TF32 copy (kmajor_tf32), which the kernel loads by TMA: wgmma reads TF32 operands K-major only, and the
    kernel's own way of reading MN-major ones - its producer threads transposing every tile - is several times
    slower.  The copy carries the operand bits those threads would make, so the result is the same.  The exact
    engine always reads the operands as given."""
    a, lda = _rows(_f32(a))
    b, ldb = _rows(_f32(b))
    if out.dim() != 2 or (out.stride(1) != 1 and out.size(1) != 1):
        raise ValueError("gemm output must be a 2-D tensor with unit inner stride")
    ldc = out.stride(0) if out.size(0) > 1 else max(out.size(1), out.stride(0))
    m, k = (a.size(1), a.size(0)) if trans_a else (a.size(0), a.size(1))
    kb, n = (b.size(1), b.size(0)) if trans_b else (b.size(0), b.size(1))
    if k != kb or out.size(0) != m or out.size(1) != n:
        raise ValueError("gemm shape mismatch: op(a) [{},{}] op(b) [{},{}] out {}".format(
            m, k, kb, n, tuple(out.shape)))
    backend = _GEMM_BACKEND if backend is None else backend
    if (trans_a or not trans_b) and _on_tensor_cores(trans_a, trans_b, m, n, k, a, lda, b, ldb, backend):
        if trans_a:
            a, lda = _rows(kmajor_tf32(a))
            trans_a = False
        if not trans_b:
            b, ldb = _rows(kmajor_tf32(b))
            trans_b = True
    call("nm_gemm", int(trans_a), int(trans_b), m, n, k, ptr(a), lda, ptr(b), ldb, ptr(out), ldc,
         ptr(bias), lib.NM_ACT[act], float(beta), backend, lib.stream())
    return out


def _sink(t: torch.Tensor) -> Optional[torch.Tensor]:
    return getattr(t, "nm_grad", None)


# -- weight gradients off the critical path ----------------------------------------------------------------
# The backward pass is a chain: every layer's input gradient feeds the next (older) layer, while its WEIGHT
# gradient feeds nothing until the optimizer runs.  A trainer may therefore open a window
# (`weight_grad_stream(True)` ... `join_weight_grads()`) in which the weight / bias gradient products of the dense
# layers and of the vocabulary projection are issued on a second stream: they fill the SMs the chain leaves idle
# (launch latencies, short grids, the 120-CTA recurrences) instead of lengthening it.  Both streams only ever ADD
# into disjoint parts of the flat gradient buffer: a variable's contributions all travel on the same stream.
# Inside a CUDA-graph capture the fork and the join become graph edges.  Off unless a trainer opens the window.
_wg = {"stream": None, "keep": [], "open": False}


def weight_grad_stream(enable: bool) -> None:
    if enable and lib.profiling():
        enable = False      # (the per-call profiler times calls one by one: no overlap while it runs)
    if enable and _wg["stream"] is None:
        _wg["stream"] = torch.cuda.Stream()
    _wg["open"] = bool(enable)


def join_weight_grads() -> None:
    """The current stream waits for every weight gradient issued so far (and their operands may be freed)."""
    if _wg["keep"]:
        torch.cuda.current_stream().wait_stream(_wg["stream"])
        del _wg["keep"][:]


def _off_the_chain(fn, *operands) -> None:
    """Run `fn` (kernels that only add into the gradient buffer) on the weight-gradient stream when a trainer
    has opened the window, else right here.  `operands` are kept alive until the join."""
    if not _wg["open"]:
        fn()
        return
    side = _wg["stream"]
    side.wait_stream(torch.cuda.current_stream())      # the operands were produced on the chain's stream
    with torch.cuda.stream(side):
        fn()
    _wg["keep"].append(operands)


def _gru_weight_grads(x2, directions, e, h):
    """Weight / bias gradients of the directions of a GRU layer over one input x2 [B*T, E].  A direction is
    (hprev [B*T, H], rh [B*T, H], dxproj [B*T, 3H], wg, wc, sinks); rows [:E] of its kernels come from x2, rows
    [E:] from the recurrent operand, against dzg = dxproj[:, :2H] and dzc = dxproj[:, 2H:].  With every variable
    in the gradient buffer all launches leave the backward chain (`_off_the_chain`) and a None 4-tuple per
    direction is returned; otherwise (dWg, dbg, dWc, dbc) per direction with None for buffered ones.

    On the tensor cores the products take K-major TF32 copies (see `gemm`), each made once: x2 for all the
    directions, dxproj per direction (dzg^T and dzc^T are row ranges of its copy), hprev and rh."""
    def products(outs):
        x2t = None
        for (hp2, rh2, dxp, _wg, _wc, _sinks), (dwg, dwc, beta_g, beta_c) in zip(directions, outs):
            dzg, dzc = dxp[:, :2 * h], dxp[:, 2 * h:]
            if all(_tn_on_tensor_cores(x, dz) for x, dz in ((x2, dzg), (hp2, dzg), (x2, dzc), (rh2, dzc))):
                if x2t is None:
                    x2t = kmajor_tf32(x2)
                dxpt = kmajor_tf32(dxp)
                x, hp, rh, dg, dc = x2t, kmajor_tf32(hp2), kmajor_tf32(rh2), dxpt[:2 * h], dxpt[2 * h:]
                trans = (False, True)       # x^T . dz = (x^T) . (dz^T)^T
            else:
                x, hp, rh, dg, dc = x2, hp2, rh2, dzg, dzc
                trans = (True, False)
            gemm(x, dg, dwg[:e], *trans, beta=beta_g)
            gemm(hp, dg, dwg[e:], *trans, beta=beta_g)
            gemm(x, dc, dwc[:e], *trans, beta=beta_c)
            gemm(rh, dc, dwc[e:], *trans, beta=beta_c)

    if all(s is not None for d in directions for s in d[5]):
        def into_the_buffer():
            products([(sg, sc, 1.0, 1.0) for sg, _, sc, _ in (d[5] for d in directions)])
            for d in directions:
                _bias_grad(d[2][:, :2 * h], d[5][1])
                _bias_grad(d[2][:, 2 * h:], d[5][3])
        _off_the_chain(into_the_buffer, x2, *(t for d in directions for t in d[:3]))
        return [(None, None, None, None)] * len(directions)
    outs, grads = [], []
    for hp2, rh2, dxp, wg, wc, (sg, sbg, sc, sbc) in directions:
        dwg = sg if sg is not None else torch.empty_like(wg)
        dwc = sc if sc is not None else torch.empty_like(wc)
        outs.append((dwg, dwc, 1.0 if sg is not None else 0.0, 1.0 if sc is not None else 0.0))
        grads.append((None if sg is not None else dwg, _bias_grad(dxp[:, :2 * h], sbg),
                      None if sc is not None else dwc, _bias_grad(dxp[:, 2 * h:], sbc)))
    products(outs)
    return grads


def _weight_grad(a: torch.Tensor, b: torch.Tensor, trans_a: bool, trans_b: bool,
                 sink: Optional[torch.Tensor], shape) -> Optional[torch.Tensor]:
    """op(a) @ op(b) accumulated into `sink` (returns None) or returned as a new tensor."""
    if sink is not None:
        gemm(a, b, sink, trans_a, trans_b, beta=1.0)
        return None
    out = torch.empty(shape, device=a.device, dtype=torch.float32)
    return gemm(a, b, out, trans_a, trans_b)


def _bias_grad(dy: torch.Tensor, sink: Optional[torch.Tensor]) -> Optional[torch.Tensor]:
    dy2, ld = _rows(dy)
    if sink is not None:
        call("nm_colsum", ptr(dy2), dy2.size(0), dy2.size(1), ld, ptr(sink), 1, lib.stream())
        return None
    out = torch.empty(dy2.size(1), device=dy.device, dtype=torch.float32)
    call("nm_colsum", ptr(dy2), dy2.size(0), dy2.size(1), ld, ptr(out), 0, lib.stream())
    return out


# ---------------------------------------------------------------------------
# K1 embedding
# ---------------------------------------------------------------------------
class _Embed(torch.autograd.Function):
    @staticmethod
    def forward(ctx, ids, table, mask):
        ids = ids.contiguous()
        n = ids.numel()
        v, e = table.shape
        out = torch.empty(tuple(ids.shape) + (e,), device=table.device, dtype=torch.float32)
        mask_c = mask.contiguous() if mask is not None else None
        call("nm_embed_fwd", ptr(ids), ptr(table), ptr(mask_c), ptr(out), n, e, v, lib.stream())
        ctx.save_for_backward(ids, mask_c)
        ctx.shape = (v, e)
        ctx.sink = _sink(table)
        return out

    @staticmethod
    def backward(ctx, dout):
        ids, mask = ctx.saved_tensors
        v, e = ctx.shape
        dout = dout.contiguous()
        if ctx.sink is not None:
            dtable, ret = ctx.sink, None
        else:
            dtable = torch.zeros(v, e, device=dout.device, dtype=torch.float32)
            ret = dtable
        call("nm_embed_bwd", ptr(ids), ptr(dout), ptr(mask), ptr(dtable), ids.numel(), e, v,
             lib.stream())
        return None, ret, None


def embed(ids: torch.Tensor, table: torch.Tensor, mask: Optional[torch.Tensor] = None) -> torch.Tensor:
    """table[ids] * mask[..., None]  (model/sequence.py:181-191; autoregressive.py:269-272)."""
    return _Embed.apply(ids, table, mask)


# ---------------------------------------------------------------------------
# dense projection
# ---------------------------------------------------------------------------
class _Linear(torch.autograd.Function):
    @staticmethod
    def forward(ctx, x, w, b, act):
        shape = x.shape
        x2 = x.reshape(-1, shape[-1])
        y = torch.empty(x2.size(0), w.size(1), device=x.device, dtype=torch.float32)
        gemm(x2, w, y, bias=b, act=act)
        ctx.save_for_backward(x2, w, y if act is not None else None)
        ctx.act = act
        ctx.has_bias = b is not None
        ctx.sinks = (_sink(w), _sink(b) if b is not None else None)
        ctx.in_shape = shape
        return y.view(tuple(shape[:-1]) + (w.size(1),))

    @staticmethod
    def backward(ctx, dy):
        x2, w, y = ctx.saved_tensors
        dy2 = dy.reshape(-1, dy.shape[-1])
        dy2, _ = _rows(dy2)
        if ctx.act is not None:
            dpre = torch.empty_like(y)
            dyc = dy2.contiguous()
            call("nm_act_bwd", ptr(y), ptr(dyc), ptr(dpre), y.numel(), lib.NM_ACT[ctx.act],
                 lib.stream())
        else:
            dpre = dy2
        dx = dw = db = None
        if ctx.needs_input_grad[0]:
            dx = torch.empty(x2.shape, device=dy.device, dtype=torch.float32)
            gemm(dpre, w, dx, trans_b=True)
            dx = dx.view(ctx.in_shape)
        w_sink, b_sink = ctx.sinks
        want_w, want_b = ctx.needs_input_grad[1], ctx.has_bias and ctx.needs_input_grad[2]
        if (want_w and w_sink is not None) and (not want_b or b_sink is not None):
            # both accumulate into the gradient buffer: nothing to return.  gemm makes the K-major copies of x2 and
            # dpre here, so that they too run on the weight-gradient stream
            def into_the_buffer():
                _weight_grad(x2, dpre, True, False, w_sink, w.shape)
                if want_b:
                    _bias_grad(dpre, b_sink)
            _off_the_chain(into_the_buffer, x2, dpre)
            return dx, None, None, None
        if want_w:
            dw = _weight_grad(x2, dpre, True, False, w_sink, w.shape)
        if want_b:
            db = _bias_grad(dpre, b_sink)
        return dx, dw, db, None


def linear(x: torch.Tensor, w: torch.Tensor, b: Optional[torch.Tensor] = None,
           act: Optional[str] = None) -> torch.Tensor:
    """act(x @ w + b) over the last dim; w is [in, out] (tf.layers.dense layout)."""
    return _Linear.apply(x, w, b, act)


class _Dropout(torch.autograd.Function):
    """y = dropout(x) (+ residual), masks drawn inside the kernel (K15, csrc/dropout.cu); the backward pass
    re-draws the mask of the same (site, step) instead of reading one."""

    @staticmethod
    def forward(ctx, x, residual, keep_prob, site):
        from neuralmonkey_b200 import runtime
        xc = _f32(x).contiguous()
        rc = None if residual is None else _f32(residual).expand_as(x).contiguous()
        y = torch.empty_like(xc)
        state = runtime.dropout_state()
        call("nm_dropout_apply", ptr(xc), ptr(rc), ptr(y), xc.numel(), float(keep_prob), ptr(state), int(site),
             lib.stream())
        ctx.keep_prob, ctx.site, ctx.state = float(keep_prob), int(site), state
        ctx.has_residual = residual is not None
        return y

    @staticmethod
    def backward(ctx, dy):
        dyc = dy.contiguous()
        dx = torch.empty_like(dyc)
        call("nm_dropout_apply", ptr(dyc), None, ptr(dx), dyc.numel(), ctx.keep_prob, ptr(ctx.state), ctx.site,
             lib.stream())
        return dx, (dy if ctx.has_residual else None), None, None


def dropout(x: torch.Tensor, keep_prob: float, residual: Optional[torch.Tensor] = None) -> torch.Tensor:
    """x with each element kept with probability keep_prob and scaled by 1/keep_prob, plus `residual`."""
    from neuralmonkey_b200 import runtime
    return _Dropout.apply(x, residual, keep_prob, runtime.next_dropout_site())


def dropout_mask(shape, keep_prob: float, device=None) -> torch.Tensor:
    """A mask tensor (entries 0 or 1/keep_prob) for the kernels that take one as an operand."""
    from neuralmonkey_b200 import runtime
    mask = torch.empty(tuple(int(d) for d in shape), device=runtime.device(), dtype=torch.float32)
    call("nm_dropout_mask", ptr(mask), mask.numel(), float(keep_prob), ptr(runtime.dropout_state()),
         runtime.next_dropout_site(), lib.stream())
    return mask


class _Maxout(torch.autograd.Function):
    @staticmethod
    def forward(ctx, z):
        z2 = z.reshape(-1, z.shape[-1]).contiguous()
        m, two_o = z2.shape
        o = two_o // 2
        y = torch.empty(m, o, device=z.device, dtype=torch.float32)
        which = torch.empty(m, o, device=z.device, dtype=torch.uint8)
        call("nm_maxout_fwd", ptr(z2), ptr(y), ptr(which), m, o, lib.stream())
        ctx.save_for_backward(which)
        ctx.in_shape = z.shape
        return y.view(tuple(z.shape[:-1]) + (o,))

    @staticmethod
    def backward(ctx, dy):
        (which,) = ctx.saved_tensors
        m, o = which.shape
        dy2 = dy.reshape(m, o).contiguous()
        dz = torch.empty(m, 2 * o, device=dy.device, dtype=torch.float32)
        call("nm_maxout_bwd", ptr(dy2), ptr(which), ptr(dz), m, o, lib.stream())
        return dz.view(ctx.in_shape)


def maxout(z: torch.Tensor) -> torch.Tensor:
    """y[..., j] = max(z[..., j], z[..., O + j])  (nn/projection.py:7-35 as executed)."""
    return _Maxout.apply(z)


# ---------------------------------------------------------------------------
# gate arithmetic of the step-wise cell variants (N4): one launch per step and direction
# ---------------------------------------------------------------------------
class _NematusGate(torch.autograd.Function):
    @staticmethod
    def forward(ctx, sg, gi, sc, ci, state):
        sg, gi, sc, ci, state = (t.contiguous() for t in (sg, gi, sc, ci, state))
        bsz, h = state.shape
        out = torch.empty_like(state)
        saved = torch.empty(bsz, 3 * h, device=state.device, dtype=torch.float32)
        call("nm_nematus_gate_fwd", ptr(sg), ptr(gi), ptr(sc), ptr(ci), ptr(state), ptr(out), ptr(saved), bsz, h,
             lib.stream())
        ctx.save_for_backward(saved, sc, state)
        return out

    @staticmethod
    def backward(ctx, dout):
        saved, sc, state = ctx.saved_tensors
        bsz, h = state.shape
        dout = dout.contiguous()
        dgates = torch.empty(bsz, 2 * h, device=state.device, dtype=torch.float32)
        dcpre, dsc, dstate = torch.empty_like(state), torch.empty_like(state), torch.empty_like(state)
        call("nm_nematus_gate_bwd", ptr(dout), ptr(saved), ptr(sc), ptr(state), ptr(dgates), ptr(dcpre), ptr(dsc),
             ptr(dstate), bsz, h, lib.stream())
        return dgates, dgates, dsc, dcpre, dstate


def nematus_gru_gate(state_gates: torch.Tensor, input_gates: torch.Tensor, state_cand: torch.Tensor,
                     input_cand: torch.Tensor, state: torch.Tensor) -> torch.Tensor:
    """NematusGRUCell after its projections (nn/ortho_gru_cell.py:86-105): [r,u] = sigmoid(state_gates +
    input_gates); cand = tanh(state_cand * r + input_cand); u * state + (1 - u) * cand."""
    return _NematusGate.apply(state_gates, input_gates, state_cand, input_cand, state)


class _LSTMGate(torch.autograd.Function):
    @staticmethod
    def forward(ctx, z, c):
        z, c = z.contiguous(), c.contiguous()
        bsz, h = c.shape
        new_c, new_h = torch.empty_like(c), torch.empty_like(c)
        saved = torch.empty(bsz, 5 * h, device=c.device, dtype=torch.float32)
        call("nm_lstm_gate_fwd", ptr(z), ptr(c), ptr(new_c), ptr(new_h), ptr(saved), bsz, h, lib.stream())
        ctx.save_for_backward(saved, c)
        return new_c, new_h

    @staticmethod
    def backward(ctx, dnew_c, dnew_h):
        saved, c = ctx.saved_tensors
        bsz, h = c.shape
        dz = torch.empty(bsz, 4 * h, device=c.device, dtype=torch.float32)
        dc = torch.empty_like(c)
        call("nm_lstm_gate_bwd", ptr(dnew_c.contiguous() if dnew_c is not None else None),
             ptr(dnew_h.contiguous() if dnew_h is not None else None), ptr(saved), ptr(c), ptr(dz), ptr(dc), bsz, h,
             lib.stream())
        return dz, dc


def lstm_gate(z: torch.Tensor, c: torch.Tensor):
    """tf LSTMCell defaults after the [x, h] projection: z = (i, j, f, o); returns (c', h') with
    c' = sigmoid(f + 1) * c + sigmoid(i) * tanh(j), h' = sigmoid(o) * tanh(c')."""
    return _LSTMGate.apply(z, c)


# ---------------------------------------------------------------------------
# K7 layer norm
# ---------------------------------------------------------------------------
class _LayerNorm(torch.autograd.Function):
    @staticmethod
    def forward(ctx, x, gamma, beta, eps):
        x2 = x.reshape(-1, x.shape[-1]).contiguous()
        m, d = x2.shape
        y = torch.empty_like(x2)
        mean = torch.empty(m, device=x.device, dtype=torch.float32)
        rstd = torch.empty(m, device=x.device, dtype=torch.float32)
        call("nm_layernorm_fwd", ptr(x2), ptr(gamma), ptr(beta), ptr(y), ptr(mean), ptr(rstd), m, d,
             float(eps), lib.stream())
        ctx.save_for_backward(x2, gamma, mean, rstd)
        ctx.sinks = (_sink(gamma), _sink(beta))
        ctx.in_shape = x.shape
        return y.view(x.shape)

    @staticmethod
    def backward(ctx, dy):
        x2, gamma, mean, rstd = ctx.saved_tensors
        m, d = x2.shape
        dy2 = dy.reshape(m, d).contiguous()
        dx = torch.empty_like(x2)
        sg, sb = ctx.sinks
        if sg is not None and sb is not None:
            # the input gradient continues the chain; the parameter gradients only add into the gradient buffer
            call("nm_layernorm_bwd", ptr(x2), ptr(gamma), ptr(mean), ptr(rstd), ptr(dy2), ptr(dx), None, None, m, d,
                 lib.stream())
            _off_the_chain(lambda: call("nm_layernorm_bwd", ptr(x2), ptr(gamma), ptr(mean), ptr(rstd), ptr(dy2), None,
                                        ptr(sg), ptr(sb), m, d, lib.stream()), x2, dy2, mean, rstd)
            return dx.view(ctx.in_shape), None, None, None
        dg = sg if sg is not None else torch.zeros(d, device=dy.device, dtype=torch.float32)
        db = sb if sb is not None else torch.zeros(d, device=dy.device, dtype=torch.float32)
        call("nm_layernorm_bwd", ptr(x2), ptr(gamma), ptr(mean), ptr(rstd), ptr(dy2), ptr(dx), ptr(dg),
             ptr(db), m, d, lib.stream())
        return (dx.view(ctx.in_shape), None if sg is not None else dg,
                None if sb is not None else db, None)


def layer_norm(x: torch.Tensor, gamma: torch.Tensor, beta: torch.Tensor,
               eps: float = 1e-6) -> torch.Tensor:
    """tf_utils.layer_norm (tf_utils.py:189-219)."""
    return _LayerNorm.apply(x, gamma, beta, eps)


# ---------------------------------------------------------------------------
# K2 GRU layer (input projection hoisted onto the tensor cores + recurrent kernels)
# ---------------------------------------------------------------------------
class _GRULayer(torch.autograd.Function):
    @staticmethod
    def forward(ctx, x, wg, bg, wc, bc, h0, lengths, reverse, drop_mask, sm_budget):
        # x [B,T,E]; wg [E+H,2H], bg [2H]; wc [E+H,H], bc [H]   (TF GRUCell kernels)
        bsz, t, e = x.shape
        h = wc.size(1)
        x2 = x.reshape(bsz * t, e)
        xproj = torch.empty(bsz * t, 3 * h, device=x.device, dtype=torch.float32)
        gemm(x2, wg[:e], xproj[:, :2 * h], bias=bg)
        gemm(x2, wc[:e], xproj[:, 2 * h:], bias=bc)
        states = torch.empty(bsz, t, h, device=x.device, dtype=torch.float32)
        raw = torch.empty_like(states) if drop_mask is not None else None
        final = torch.empty(bsz, h, device=x.device, dtype=torch.float32)
        gates = torch.empty(bsz, t, 3 * h, device=x.device, dtype=torch.float32)
        hprev = torch.empty(bsz, t, h, device=x.device, dtype=torch.float32)
        rh = torch.empty(bsz, t, h, device=x.device, dtype=torch.float32)
        h0c = h0.contiguous() if h0 is not None else None
        dm = drop_mask.contiguous() if drop_mask is not None else None
        call("nm_gru_seq_fwd", ptr(xproj), ptr(wg[e:]), ptr(wc[e:]), ptr(h0c), ptr(lengths), ptr(dm),
             int(reverse), ptr(states), ptr(raw), ptr(final), ptr(gates), ptr(hprev), ptr(rh), bsz, t,
             h, int(sm_budget), lib.stream())
        ctx.save_for_backward(x2, wg, wc, lengths, gates, hprev, rh, dm)
        ctx.dims = (bsz, t, e, h)
        ctx.reverse = reverse
        ctx.sm_budget = sm_budget
        ctx.has_h0 = h0 is not None
        ctx.sinks = (_sink(wg), _sink(bg), _sink(wc), _sink(bc))
        return states, final, (raw if raw is not None else states)

    @staticmethod
    def backward(ctx, dstates, dfinal, draw):
        x2, wg, wc, lengths, gates, hprev, rh, dm = ctx.saved_tensors
        bsz, t, e, h = ctx.dims
        dev = x2.device
        dstates = dstates.contiguous() if dstates is not None else None
        dfinal = dfinal.contiguous() if dfinal is not None else None
        if draw is not None:
            if dm is None:  # raw aliases states: autograd delivers the two gradients separately
                dstates = draw.contiguous() if dstates is None else dstates + draw
                draw = None
            else:
                draw = draw.contiguous()
        dxproj = torch.empty(bsz * t, 3 * h, device=dev, dtype=torch.float32)
        dh0 = torch.empty(bsz, h, device=dev, dtype=torch.float32) if ctx.has_h0 else None
        work = torch.empty(2 * bsz * h, device=dev, dtype=torch.float32)
        call("nm_gru_seq_bwd", ptr(wg[e:]), ptr(wc[e:]), ptr(lengths), ptr(dm), int(ctx.reverse),
             ptr(gates), ptr(hprev), ptr(dstates), ptr(draw), ptr(dfinal), ptr(dxproj), ptr(dh0),
             ptr(work), bsz, t, h, int(ctx.sm_budget), lib.stream())
        dzg, dzc = dxproj[:, :2 * h], dxproj[:, 2 * h:]
        [(dwg, dbg, dwc, dbc)] = _gru_weight_grads(
            x2, [(hprev.view(bsz * t, h), rh.view(bsz * t, h), dxproj, wg, wc, ctx.sinks)], e, h)
        dx = None
        if ctx.needs_input_grad[0]:
            dx = torch.empty(bsz * t, e, device=dev, dtype=torch.float32)
            gemm(dzg, wg[:e], dx, trans_b=True)
            gemm(dzc, wc[:e], dx, trans_b=True, beta=1.0)
            dx = dx.view(bsz, t, e)
        return (dx, dwg, dbg, dwc, dbc, dh0, None, None, None, None)


def gru_layer(x: torch.Tensor, gates_kernel: torch.Tensor, gates_bias: torch.Tensor,
              cand_kernel: torch.Tensor, cand_bias: torch.Tensor,
              h0: Optional[torch.Tensor] = None, lengths: Optional[torch.Tensor] = None,
              reverse: bool = False,
              drop_mask: Optional[torch.Tensor] = None, sm_budget: int = 0):
    """dynamic_rnn over a TF-1.12 GRUCell (encoders/recurrent.py:71-110).

    Returns (outputs [B,T,H], final state [B,H], raw outputs [B,T,H] = outputs before
    `drop_mask`); with `lengths` (int32) the outputs past
    each length are zero and the state is carried, with `reverse` the sequence is walked
    backwards inside its length (tf.reverse_sequence semantics)."""
    return _GRULayer.apply(x, gates_kernel, gates_bias, cand_kernel, cand_bias, h0, lengths, reverse,
                           drop_mask, sm_budget)


class _BiGRULayer(torch.autograd.Function):
    """Forward and backward direction of a bidirectional GRU layer over the same input.  Their recurrences
    go through one entry point each way (nm_gru_seq_fwd_pair / nm_gru_seq_bwd_pair), which runs the two
    directions one after the other, each on the whole GPU."""

    @staticmethod
    def forward(ctx, x, lengths, wg_f, bg_f, wc_f, bc_f, wg_b, bg_b, wc_b, bc_b):
        bsz, t, e = x.shape
        h = wc_f.size(1)
        x2 = x.reshape(bsz * t, e)
        dev = x.device
        saved = []
        outs = []
        bufs = []
        for wg, bg, wc, bc in ((wg_f, bg_f, wc_f, bc_f), (wg_b, bg_b, wc_b, bc_b)):
            xproj = torch.empty(bsz * t, 3 * h, device=dev, dtype=torch.float32)
            gemm(x2, wg[:e], xproj[:, :2 * h], bias=bg)
            gemm(x2, wc[:e], xproj[:, 2 * h:], bias=bc)
            states = torch.empty(bsz, t, h, device=dev, dtype=torch.float32)
            final = torch.empty(bsz, h, device=dev, dtype=torch.float32)
            gates = torch.empty(bsz, t, 3 * h, device=dev, dtype=torch.float32)
            hprev = torch.empty(bsz, t, h, device=dev, dtype=torch.float32)
            rh = torch.empty(bsz, t, h, device=dev, dtype=torch.float32)
            bufs.append((xproj, states, final, gates, hprev, rh))
        (xp_f, st_f, fi_f, ga_f, hp_f, rh_f), (xp_b, st_b, fi_b, ga_b, hp_b, rh_b) = bufs
        call("nm_gru_seq_fwd_pair",
             ptr(xp_f), ptr(wg_f[e:]), ptr(wc_f[e:]), 0, ptr(st_f), ptr(fi_f), ptr(ga_f), ptr(hp_f), ptr(rh_f),
             ptr(xp_b), ptr(wg_b[e:]), ptr(wc_b[e:]), 1, ptr(st_b), ptr(fi_b), ptr(ga_b), ptr(hp_b), ptr(rh_b),
             ptr(lengths), bsz, t, h, lib.stream())
        ctx.save_for_backward(x2, lengths, wg_f, wc_f, wg_b, wc_b, ga_f, hp_f, rh_f, ga_b, hp_b, rh_b)
        ctx.dims = (bsz, t, e, h)
        ctx.sinks = tuple(_sink(w) for w in (wg_f, bg_f, wc_f, bc_f, wg_b, bg_b, wc_b, bc_b))
        return st_f, fi_f, st_b, fi_b

    @staticmethod
    def backward(ctx, dst_f, dfi_f, dst_b, dfi_b):
        x2, lengths, wg_f, wc_f, wg_b, wc_b, ga_f, hp_f, rh_f, ga_b, hp_b, rh_b = ctx.saved_tensors
        bsz, t, e, h = ctx.dims
        dev = x2.device

        def c(g):
            return g.contiguous() if g is not None else None

        dst_f, dfi_f, dst_b, dfi_b = c(dst_f), c(dfi_f), c(dst_b), c(dfi_b)
        dxp_f = torch.empty(bsz * t, 3 * h, device=dev, dtype=torch.float32)
        dxp_b = torch.empty(bsz * t, 3 * h, device=dev, dtype=torch.float32)
        work = torch.empty(2 * bsz * h, device=dev, dtype=torch.float32)
        call("nm_gru_seq_bwd_pair",
             ptr(wg_f[e:]), ptr(wc_f[e:]), 0, ptr(ga_f), ptr(hp_f), ptr(dst_f), ptr(dfi_f), ptr(dxp_f),
             ptr(wg_b[e:]), ptr(wc_b[e:]), 1, ptr(ga_b), ptr(hp_b), ptr(dst_b), ptr(dfi_b), ptr(dxp_b),
             ptr(lengths), ptr(work), bsz, t, h, lib.stream())
        dx = torch.empty(bsz * t, e, device=dev, dtype=torch.float32) if ctx.needs_input_grad[0] else None
        directions = ((wg_f, wc_f, hp_f, rh_f, dxp_f, ctx.sinks[:4]), (wg_b, wc_b, hp_b, rh_b, dxp_b, ctx.sinks[4:]))
        if dx is not None:          # the chain first: the input gradient is what the older layers wait for
            for i, (wg, wc, _hp, _rh, dxp, _sinks) in enumerate(directions):
                gemm(dxp[:, :2 * h], wg[:e], dx, trans_b=True, beta=0.0 if i == 0 else 1.0)
                gemm(dxp[:, 2 * h:], wc[:e], dx, trans_b=True, beta=1.0)
        grads = _gru_weight_grads(x2, [(hp.view(bsz * t, h), rh.view(bsz * t, h), dxp, wg, wc, sinks)
                                       for wg, wc, hp, rh, dxp, sinks in directions], e, h)
        return (dx.view(bsz, t, e) if dx is not None else None, None) + tuple(g for d in grads for g in d)


def gru_bilayer(x: torch.Tensor, lengths: torch.Tensor, cell_fw, cell_bw):
    """tf.nn.bidirectional_dynamic_rnn over two TF-1.12 GRUCells (encoders/recurrent.py:82-95).  cell_* =
    (gates kernel, gates bias, candidate kernel, candidate bias).  Returns (outputs fw [B,T,H], final fw [B,H],
    outputs bw, final bw); the backward direction walks each sentence from its last token
    (tf.reverse_sequence semantics), outputs at their original time index."""
    return _BiGRULayer.apply(x, lengths, *cell_fw, *cell_bw)


# ---------------------------------------------------------------------------
# K4 Bahdanau attention
# ---------------------------------------------------------------------------
class _Bahdanau(torch.autograd.Function):
    @staticmethod
    def forward(ctx, keys, values, mask, qproj, v, bias):
        bsz, tx, a = keys.shape
        c = values.size(2)
        nq = qproj.size(1)
        keys, values, qproj = keys.contiguous(), values.contiguous(), qproj.contiguous()
        mask_c = mask.contiguous() if mask is not None else None
        dev = keys.device
        energies = torch.empty(bsz, nq, tx, device=dev, dtype=torch.float32)
        weights = torch.empty(bsz, nq, tx, device=dev, dtype=torch.float32)
        ctxv = torch.empty(bsz, nq, c, device=dev, dtype=torch.float32)
        call("nm_bahdanau_fwd", ptr(keys), ptr(values), ptr(mask_c), ptr(qproj), ptr(v), ptr(bias),
             ptr(energies), ptr(weights), ptr(ctxv), bsz, tx, nq, a, c, lib.stream())
        ctx.save_for_backward(keys, values, mask_c, qproj, v, energies, weights)
        ctx.sinks = (_sink(v), _sink(bias))
        ctx.mark_non_differentiable(weights)
        ctx.set_materialize_grads(False)
        return ctxv, weights, energies

    @staticmethod
    def backward(ctx, dctx, _dweights, denergies):
        keys, values, mask, qproj, v, energies, weights = ctx.saved_tensors
        bsz, tx, a = keys.shape
        c = values.size(2)
        nq = qproj.size(1)
        dev = keys.device
        dctx = dctx.contiguous() if dctx is not None else torch.zeros(bsz, nq, c, device=dev, dtype=torch.float32)
        denergies = denergies.contiguous() if denergies is not None else None
        dkeys = torch.empty_like(keys)
        dvalues = torch.empty_like(values)
        dq = torch.empty_like(qproj)
        sv, sb = ctx.sinks
        dv = sv if sv is not None else torch.zeros(a, device=dev, dtype=torch.float32)
        db = sb if sb is not None else torch.zeros(1, device=dev, dtype=torch.float32)
        work = torch.empty(bsz * nq * tx, device=dev, dtype=torch.float32)
        call("nm_bahdanau_bwd", ptr(keys), ptr(values), ptr(mask), ptr(qproj), ptr(v), ptr(energies),
             ptr(weights), ptr(dctx), ptr(denergies), ptr(dkeys), ptr(dvalues), ptr(dq), ptr(dv), ptr(db), ptr(work),
             bsz, tx, nq, a, c, lib.stream())
        return (dkeys, dvalues, None, dq, None if sv is not None else dv,
                None if sb is not None else db)


def bahdanau_attention(keys: torch.Tensor, values: torch.Tensor, mask: Optional[torch.Tensor],
                       qproj: torch.Tensor, v: torch.Tensor,
                       bias: torch.Tensor) -> Tuple[torch.Tensor, torch.Tensor]:
    """Attention.attention (attention/feed_forward.py:125-166) for all query steps at once.

    keys [B,Tx,A], values [B,Tx,C], mask [B,Tx] or None, qproj [B,NQ,A], v [A], bias [1].
    Returns (contexts [B,NQ,C], weights [B,NQ,Tx])."""
    ctxv, weights, _energies = _Bahdanau.apply(keys, values, mask, qproj, v, bias)
    return ctxv, weights


def bahdanau_attention_energies(keys: torch.Tensor, values: torch.Tensor, mask: Optional[torch.Tensor],
                                qproj: torch.Tensor, v: torch.Tensor,
                                bias: torch.Tensor) -> Tuple[torch.Tensor, torch.Tensor, torch.Tensor]:
    """`bahdanau_attention` that also returns the pre-softmax energies e [B,NQ,Tx] of the same evaluation, as a
    differentiable output: a loss on them (`alignment_xent`) reaches keys, qproj, v and bias through the same
    nm_bahdanau_bwd call as the gradient of the contexts.  Returns (contexts, weights, energies)."""
    return _Bahdanau.apply(keys, values, mask, qproj, v, bias)


# ---------------------------------------------------------------------------
# K21 supervised attention (decoders.word_alignment_decoder)
# ---------------------------------------------------------------------------
class _AlignmentXent(torch.autograd.Function):
    @staticmethod
    def forward(ctx, energies, target, pad):
        bsz, nq, tx = energies.shape
        energies, target, pad = energies.contiguous(), target.contiguous(), pad.contiguous()
        dev = energies.device
        loss = torch.empty((), device=dev, dtype=torch.float32)
        work = torch.empty(bsz * nq, device=dev, dtype=torch.float32)
        call("nm_alignment_xent_fwd", ptr(energies), ptr(target), ptr(pad), ptr(loss), ptr(work), bsz, nq, tx,
             lib.stream())
        ctx.save_for_backward(energies, target, pad)
        return loss

    @staticmethod
    def backward(ctx, dloss):
        energies, target, pad = ctx.saved_tensors
        bsz, nq, tx = energies.shape
        de = torch.empty_like(energies)
        call("nm_alignment_xent_bwd", ptr(energies), ptr(target), ptr(pad), ptr(dloss.contiguous()),
             ptr(de), bsz, nq, tx, lib.stream())
        return de, None, None


def alignment_xent(energies: torch.Tensor, target: torch.Tensor, pad: torch.Tensor) -> torch.Tensor:
    """The training loss of WordAlignmentDecoder (decoders/word_alignment_decoder.py:100-108): a scalar

        sum_{b,q} pad[b,q] * sum_t target[b,q,t] * (logsumexp_t energies[b,q,t] - energies[b,q,t]),

    softmax cross-entropy over all Tx positions.  energies, target [B,NQ,Tx], pad [B,NQ]; differentiable in the
    energies only.  The sum is taken in a fixed order: repeat calls give the same bits."""
    for t in (energies, target, pad):
        _f32(t)
    if target.shape != energies.shape or pad.shape != energies.shape[:2]:
        raise ValueError("alignment_xent: energies {}, target {}, pad {}".format(
            tuple(energies.shape), tuple(target.shape), tuple(pad.shape)))
    return _AlignmentXent.apply(energies, target, pad)


# ---------------------------------------------------------------------------
# Coverage attention (attention.coverage)
# ---------------------------------------------------------------------------
class _CoverageFertility(torch.autograd.Function):
    @staticmethod
    def forward(ctx, states, fertility_w, max_fertility):
        bsz, tx, c = states.shape
        states = states.contiguous()
        fert = torch.empty(bsz, tx, device=states.device, dtype=torch.float32)
        call("nm_coverage_fertility_fwd", ptr(states), ptr(fertility_w), float(max_fertility), ptr(fert),
             bsz, tx, c, lib.stream())
        ctx.save_for_backward(states, fertility_w)
        ctx.max_fertility = max_fertility
        ctx.sink = _sink(fertility_w)
        return fert

    @staticmethod
    def backward(ctx, dfert):
        states, fertility_w = ctx.saved_tensors
        bsz, tx, c = states.shape
        dev = states.device
        dfert = dfert.contiguous()
        dstates = torch.empty_like(states)
        dfw = ctx.sink if ctx.sink is not None else torch.zeros(c, device=dev, dtype=torch.float32)
        work = torch.empty(bsz * c, device=dev, dtype=torch.float32)
        call("nm_coverage_fertility_bwd", ptr(states), ptr(fertility_w), ctx.max_fertility,
             ptr(dfert), ptr(dstates), ptr(dfw), ptr(work), bsz, tx, c, lib.stream())
        return dstates, None if ctx.sink is not None else dfw, None


def coverage_fertility(states: torch.Tensor, fertility_w: torch.Tensor, max_fertility: float) -> torch.Tensor:
    """CoverageAttention.fertility (attention/coverage.py:47-50): 1e-8 + max_fertility * sigmoid(states .
    fertility_w) in fp32 dot products.  states [B,Tx,C], fertility_w [C] -> fert [B,Tx]."""
    return _CoverageFertility.apply(states, fertility_w, float(max_fertility))


class _CoverageAttention(torch.autograd.Function):
    @staticmethod
    def forward(ctx, keys, values, mask, fert, qproj, v, coverage_w, cov_in):
        bsz, tx, a = keys.shape
        c = values.size(2)
        nq = qproj.size(1)
        keys, values, fert, qproj = keys.contiguous(), values.contiguous(), fert.contiguous(), qproj.contiguous()
        mask_c = mask.contiguous() if mask is not None else None
        cov_in_c = cov_in.contiguous() if cov_in is not None else None
        dev = keys.device
        energies = torch.empty(bsz, nq, tx, device=dev, dtype=torch.float32)
        weights = torch.empty(bsz, nq, tx, device=dev, dtype=torch.float32)
        coverage = torch.empty(bsz, nq, tx, device=dev, dtype=torch.float32)
        ctxv = torch.empty(bsz, nq, c, device=dev, dtype=torch.float32)
        cov_out = torch.empty(bsz, tx, device=dev, dtype=torch.float32)
        call("nm_coverage_attention_fwd", ptr(keys), ptr(values), ptr(mask_c), ptr(fert), ptr(qproj), ptr(v),
             ptr(coverage_w), ptr(cov_in_c), ptr(energies), ptr(weights), ptr(coverage), ptr(ctxv), ptr(cov_out),
             bsz, tx, nq, a, c, lib.stream())
        ctx.save_for_backward(keys, values, mask_c, fert, qproj, v, coverage_w, energies, weights, coverage)
        ctx.sinks = (_sink(v), _sink(coverage_w))
        ctx.has_cov_in = cov_in is not None
        ctx.mark_non_differentiable(weights)
        return ctxv, weights, cov_out

    @staticmethod
    def backward(ctx, dctx, _dweights, dcov_out):
        keys, values, mask, fert, qproj, v, coverage_w, energies, weights, coverage = ctx.saved_tensors
        bsz, tx, a = keys.shape
        c = values.size(2)
        nq = qproj.size(1)
        dev = keys.device
        dctx = dctx.contiguous()
        dcov_out = dcov_out.contiguous() if dcov_out is not None else None
        dkeys = torch.empty_like(keys)
        dvalues = torch.empty_like(values)
        dq = torch.empty_like(qproj)
        dfert = torch.empty_like(fert)
        dcov_in = torch.empty(bsz, tx, device=dev, dtype=torch.float32) if ctx.has_cov_in else None
        sv, sc = ctx.sinks
        dv = sv if sv is not None else torch.zeros(a, device=dev, dtype=torch.float32)
        dcw = sc if sc is not None else torch.zeros(a, device=dev, dtype=torch.float32)
        work = torch.empty(2 * bsz * a, device=dev, dtype=torch.float32)
        call("nm_coverage_attention_bwd", ptr(keys), ptr(values), ptr(mask), ptr(fert), ptr(qproj), ptr(v),
             ptr(coverage_w), ptr(energies), ptr(weights), ptr(coverage), ptr(dctx), ptr(dcov_out), ptr(dkeys),
             ptr(dvalues), ptr(dq), ptr(dfert), ptr(dcov_in), ptr(dv), ptr(dcw), ptr(work), bsz, tx, nq, a, c,
             lib.stream())
        return (dkeys, dvalues, None, dfert, dq, None if sv is not None else dv, None if sc is not None else dcw,
                dcov_in)


def coverage_attention(keys: torch.Tensor, values: torch.Tensor, mask: Optional[torch.Tensor], fert: torch.Tensor,
                       qproj: torch.Tensor, v: torch.Tensor, coverage_w: torch.Tensor,
                       cov_in: Optional[torch.Tensor] = None) -> Tuple[torch.Tensor, torch.Tensor, torch.Tensor]:
    """CoverageAttention.attention (attention/coverage.py:52-61 in feed_forward.py:125-166) for NQ consecutive
    decoder steps, as one scan.

    keys [B,Tx,A], values [B,Tx,C], mask [B,Tx] or None, fert [B,Tx] (`coverage_fertility`), qproj [B,NQ,A],
    v [A], coverage_w [A], cov_in [B,Tx]: the sum of the weights of earlier steps, None for none.  Returns
    (contexts [B,NQ,C], weights [B,NQ,Tx], cov_out [B,Tx] = cov_in + the sum of the NQ steps' weights).  The
    weights are not differentiable; the gradient between calls flows through cov_out."""
    return _CoverageAttention.apply(keys, values, mask, fert, qproj, v, coverage_w, cov_in)


# ---------------------------------------------------------------------------
# Joint multi-source attention (attention.combination)
# ---------------------------------------------------------------------------
class _JointAttention(torch.autograd.Function):
    @staticmethod
    def forward(ctx, keys, values, mask, seg_ends, seg_bias, ckeys, cvalues, cand_bias, qproj, v):
        bsz, nq, a = qproj.shape
        tx = keys.size(1) if keys is not None else 0
        j = ckeys.size(2) if ckeys is not None else 0
        c = values.size(2) if values is not None else cvalues.size(3)
        keys, values, ckeys, cvalues = (t.contiguous() if t is not None else None
                                        for t in (keys, values, ckeys, cvalues))
        qproj = qproj.contiguous()
        mask_c = mask.contiguous() if mask is not None else None
        ends = (ctypes.c_int64 * max(len(seg_ends), 1))(*seg_ends)
        dev = qproj.device
        energies = torch.empty(bsz, nq, tx + j, device=dev, dtype=torch.float32)
        weights = torch.empty(bsz, nq, tx + j, device=dev, dtype=torch.float32)
        ctxv = torch.empty(bsz, nq, c, device=dev, dtype=torch.float32)
        call("nm_joint_attention_fwd", ptr(keys), ptr(values), ptr(mask_c), ctypes.addressof(ends), ptr(seg_bias),
             ptr(ckeys), ptr(cvalues), ptr(cand_bias), ptr(qproj), ptr(v), ptr(energies), ptr(weights), ptr(ctxv),
             bsz, tx, len(seg_ends), j, nq, a, c, lib.stream())
        ctx.save_for_backward(keys, values, mask_c, ckeys, cvalues, qproj, v, energies, weights)
        ctx.seg_ends = tuple(seg_ends)
        ctx.sinks = (_sink(v), _sink(seg_bias) if seg_bias is not None else None,
                     _sink(cand_bias) if cand_bias is not None else None)
        ctx.bias_shapes = (None if seg_bias is None else seg_bias.shape, None if cand_bias is None else cand_bias.shape)
        ctx.mark_non_differentiable(weights)
        return ctxv, weights

    @staticmethod
    def backward(ctx, dctx, _dweights):
        keys, values, mask, ckeys, cvalues, qproj, v, energies, weights = ctx.saved_tensors
        bsz, nq, a = qproj.shape
        tx, j, c = energies.size(2) - (ckeys.size(2) if ckeys is not None else 0), \
            (ckeys.size(2) if ckeys is not None else 0), dctx.size(2)
        dev = qproj.device
        dctx = dctx.contiguous()
        ends = (ctypes.c_int64 * max(len(ctx.seg_ends), 1))(*ctx.seg_ends)
        dkeys = torch.empty_like(keys) if keys is not None else None
        dvalues = torch.empty_like(values) if values is not None else None
        dckeys = torch.empty_like(ckeys) if ckeys is not None else None
        dcvalues = torch.empty_like(cvalues) if cvalues is not None else None
        dq = torch.empty_like(qproj)
        sv, ss, sc = ctx.sinks
        seg_shape, cand_shape = ctx.bias_shapes
        dv = sv if sv is not None else torch.zeros(a, device=dev, dtype=torch.float32)
        dseg = ss if ss is not None else (torch.zeros(seg_shape, device=dev, dtype=torch.float32)
                                          if seg_shape is not None else None)
        dcand = sc if sc is not None else (torch.zeros(cand_shape, device=dev, dtype=torch.float32)
                                           if cand_shape is not None else None)
        work = torch.empty(bsz * nq * (tx + j) + bsz * a + bsz * (len(ctx.seg_ends) + j), device=dev,
                           dtype=torch.float32)
        call("nm_joint_attention_bwd", ptr(keys), ptr(values), ptr(mask), ctypes.addressof(ends), ptr(ckeys),
             ptr(cvalues), ptr(qproj), ptr(v), ptr(energies), ptr(weights), ptr(dctx), ptr(dkeys), ptr(dvalues),
             ptr(dq), ptr(dckeys), ptr(dcvalues), ptr(dv), ptr(dseg), ptr(dcand), ptr(work),
             bsz, tx, len(ctx.seg_ends), j, nq, a, c, lib.stream())
        return (dkeys, dvalues, None, None, None if ss is not None else dseg, dckeys, dcvalues,
                None if sc is not None else dcand, dq, None if sv is not None else dv)


def joint_attention(keys: Optional[torch.Tensor], values: Optional[torch.Tensor], mask: Optional[torch.Tensor],
                    seg_ends: Sequence[int], seg_bias: Optional[torch.Tensor], ckeys: Optional[torch.Tensor],
                    cvalues: Optional[torch.Tensor], cand_bias: Optional[torch.Tensor], qproj: torch.Tensor,
                    v: torch.Tensor) -> Tuple[torch.Tensor, torch.Tensor]:
    """One softmax over shared keys in segments and per-query candidates (attention/combination.py:240-321 flat,
    :394-463 hierarchical) for all query steps at once.

    keys [B,Tx,A], values [B,Tx,C], mask [B,Tx] or None, seg_ends: the cumulative ends of the S segments of Tx,
    seg_bias [S] (one energy bias per segment), ckeys [B,NQ,J,A], cvalues [B,NQ,J,C], cand_bias [J],
    qproj [B,NQ,A], v [A].  With Tx = 0 the shared arguments are None (and seg_ends empty); with J = 0 the
    candidate ones.  Returns (contexts [B,NQ,C], weights [B,NQ,Tx+J])."""
    return _JointAttention.apply(keys, values, mask, list(seg_ends), seg_bias, ckeys, cvalues, cand_bias, qproj, v)


# ---------------------------------------------------------------------------
# K5/K6 vocabulary projection + cross-entropy
# ---------------------------------------------------------------------------
class _SmoothingTerm(torch.autograd.Function):
    """logit[m, target[m]] - mean_v logit[m, v] for logits = x @ W + b (+ -1e9 on the <unk> column) without
    materialising them: label smoothing adds `eps` times this to the plain cross-entropy
    (xent_smoothed = lse - (1 - eps) * logit_t - eps * mean_v logit = xent + eps * (logit_t - mean_v logit)).
    Host-level torch arithmetic on [M, K] tensors (a gather of M weight columns and a mean column); the
    weight / bias gradients are accumulated into the arena's gradient buffer like every other op's."""

    @staticmethod
    def forward(ctx, x, w, b, targets, unk_index, trans_w):
        vocab = w.size(0) if trans_w else w.size(1)
        cols = w.index_select(0, targets) if trans_w else w.index_select(1, targets).t()
        wmean = w.mean(0 if trans_w else 1)
        value = (x * cols).sum(1) - x @ wmean
        if b is not None:
            value = value + b.index_select(0, targets) - b.mean()
        if unk_index >= 0:
            value = value - 1e9 * (targets == unk_index).to(value.dtype) + 1e9 / vocab
        ctx.save_for_backward(x, cols, wmean, targets)
        ctx.cfg = (vocab, trans_w, b is not None, w.shape)
        ctx.sinks = (_sink(w), _sink(b) if b is not None else None)
        return value

    @staticmethod
    def backward(ctx, g):
        x, cols, wmean, targets = ctx.saved_tensors
        vocab, trans_w, has_bias, w_shape = ctx.cfg
        w_sink, b_sink = ctx.sinks
        dx = g.unsqueeze(1) * (cols - wmean) if ctx.needs_input_grad[0] else None
        gx = x * g.unsqueeze(1)                                    # [M, K]
        dw = w_sink if w_sink is not None else torch.zeros(w_shape, device=x.device, dtype=torch.float32)
        if trans_w:                                                 # W is [V, K]
            dw.index_add_(0, targets, gx)
            dw.sub_((gx.sum(0) / vocab).unsqueeze(0))
        else:                                                       # W is [K, V]
            dw.index_add_(1, targets, gx.t().contiguous())
            dw.sub_((gx.sum(0) / vocab).unsqueeze(1))
        db = None
        if has_bias:
            db = b_sink if b_sink is not None else torch.zeros(vocab, device=x.device, dtype=torch.float32)
            db.index_add_(0, targets, g)
            db.sub_(g.sum() / vocab)
        return (dx, None if w_sink is not None else dw, None if (b_sink is not None or not has_bias) else db,
                None, None, None)


def smoothing_term(x: torch.Tensor, w: torch.Tensor, b: Optional[torch.Tensor], targets: torch.Tensor,
                   unk_index: int = -1, trans_w: bool = False) -> torch.Tensor:
    return _SmoothingTerm.apply(x, w, b, targets, unk_index, trans_w)


# SMs the fp16 [dW; db] product of the vocabulary projection takes on the weight-gradient stream.  It runs one
# persistent CTA per SM it is given; on all of them it holds back the backward chain issued behind it.  En-de bench
# step on an H100 80GB HBM3 at a 700 W power limit (two runs each): 36 SMs 11.07-11.11 ms, 48 SMs 11.04-11.06 ms,
# 64 SMs 11.09-11.12 ms, all 132 SMs 11.14-11.17 ms.
_DW16_CTAS = 48


def _pad8(n: int) -> int:
    return (n + 7) // 8 * 8


class _LogitsXent16(torch.autograd.Function):
    """The fp16-operand variant of _LogitsXent for W stored [K,V] with the bias right behind it in the
    gradient buffer (the layout the decoders declare).  Same results within TF32-class rounding (fp16
    has TF32's 10 mantissa bits; the operands here are O(1): activations after tanh, U(-0.5, 0.5)-scale
    weights, and (softmax - onehot) in [-1, 1]).

        logits = X16 [M,K] . WT16 [V,K]^T                  forward, and the recompute of the backward
        P16    = half((softmax - onehot) * mask) [M,V]      written ONCE, row-major (0.8 GB at the bench shape,
                                                            against 1.6 GB fp32 written once and read twice)
        dX     = P16 . W16 [K,V]^T * upstream[m]            K-major x K-major
        dW,db  = [X * u, u]16^T . P16 * max|upstream|       both operands MN-major (TMA-loaded as stored,
                                                            read transposed by wgmma): no transposed copy of P
    The upstream per-row gradient u = upstream / max|upstream| rides in the fp16 copy of X for dW and in
    the fp32 epilogue for dX, so P itself stays unnormalised."""

    @staticmethod
    def forward(ctx, x, w, b, targets, weights, unk_index, keep_logits):
        x2 = x.reshape(-1, x.shape[-1])
        x2, ldx = _rows(x2)
        m, k = x2.shape
        v = w.size(1)
        dev = x.device
        kpad = _pad8(k)
        targets = targets.reshape(-1).contiguous()
        weights = weights.reshape(-1).contiguous()
        w2, ldw = _rows(w)
        x16 = torch.empty(m, kpad, device=dev, dtype=torch.float16)
        call("nm_cast_f16", ptr(x2), ldx, ptr(x16), kpad, m, k, None, 0, 0, lib.stream())
        wt16 = torch.empty(v, kpad, device=dev, dtype=torch.float16)
        call("nm_cast_f16", ptr(w2), ldw, ptr(wt16), kpad, k, v, None, 1, 0, lib.stream())
        lse = torch.empty(m, device=dev, dtype=torch.float32)
        xent = torch.empty(m, device=dev, dtype=torch.float32)
        argmax = torch.empty(m, device=dev, dtype=torch.int64)
        logits = torch.empty(m, v, device=dev, dtype=torch.float32) if keep_logits else None
        part = torch.empty(lib.load().nm_logits_xent_scratch(m, v), device=dev, dtype=torch.float32)
        call("nm_logits_xent_fwd16", ptr(x16), kpad, ptr(wt16), kpad, ptr(b), unk_index, ptr(targets),
             ptr(weights), ptr(lse), ptr(xent), ptr(argmax), ptr(part), ptr(logits), v, m, v, k,
             lib.stream())
        ctx.save_for_backward(x2, w2, b, targets, weights, lse, x16, wt16)
        ctx.cfg = (unk_index, x.shape)
        ctx.sinks = (_sink(w), _sink(b) if b is not None else None)
        ctx.mark_non_differentiable(lse, argmax)
        if keep_logits:
            ctx.mark_non_differentiable(logits)
        return xent, lse, argmax, logits

    @staticmethod
    def backward(ctx, dxent, _dlse, _dargmax, _dlogits):
        x2, w2, b, targets, weights, lse, x16, wt16 = ctx.saved_tensors
        unk_index, in_shape = ctx.cfg
        m, k = x2.shape
        v = w2.size(1)
        dev = x2.device
        kpad, vpad = _pad8(k), _pad8(v)
        _, ldx = _rows(x2)
        _, ldw = _rows(w2)
        # (softmax - onehot) * mask in fp16, row-major; values in [-1, 1]
        dl16 = torch.empty(m, vpad, device=dev, dtype=torch.float16)
        call("nm_logits_xent_bwd16", ptr(x16), kpad, ptr(wt16), kpad, ptr(b), unk_index, ptr(targets),
             ptr(weights), ptr(lse), ptr(dl16), vpad, m, v, k, lib.stream())
        upstream = dxent.reshape(-1).to(torch.float32).contiguous()    # per-row factor, applied in fp32
        dx = None
        if ctx.needs_input_grad[0]:
            w16 = torch.empty(k, vpad, device=dev, dtype=torch.float16)
            call("nm_cast_f16", ptr(w2), ldw, ptr(w16), vpad, k, v, None, 0, 0, lib.stream())
            dx = torch.empty(m, k, device=dev, dtype=torch.float32)
            call("nm_gemm_f16", m, k, v, ptr(dl16), vpad, ptr(w16), vpad, ptr(dx), k, None,
                 ptr(upstream), 0.0, 0, lib.stream())
            dx = dx.view(in_shape)
        w_sink, _b_sink = ctx.sinks
        # [dW; db] [K+1, V] += smax * [X * u, u]^T . P with u = upstream / smax: straight into the gradient
        # buffer (the weight rows, then the bias row)
        smax = upstream.abs().amax().clamp_min(1e-30).reshape(1)
        k1pad = _pad8(k + 1)
        xs16 = torch.empty(m, k1pad, device=dev, dtype=torch.float16)
        call("nm_cast_f16", ptr(x2), ldx, ptr(xs16), k1pad, m, k, ptr(upstream / smax), 0, 1, lib.stream())
        sink_aug = torch.as_strided(w_sink, (k + 1, v), (v, 1))

        def dw():
            args = (k + 1, v, m, ptr(xs16), k1pad, ptr(dl16), vpad, ptr(sink_aug), v, ptr(smax), 1.0)
            if _wg["open"]:   # beside the backward chain: on _DW16_CTAS SMs, the chain's kernels find SMs free
                call("nm_gemm_f16_tn_ctas", *args, _DW16_CTAS, lib.stream())
            else:
                call("nm_gemm_f16_tn", *args, lib.stream())
        _off_the_chain(dw, xs16, dl16, smax, sink_aug)
        return dx, None, None, None, None, None, None


class _LogitsXent(torch.autograd.Function):
    """xent[m] = (logsumexp(x@W+b) - (x@W+b)[target]) * weights[m]; also lse and argmax."""

    @staticmethod
    def forward(ctx, x, w, b, targets, weights, unk_index, trans_w, keep_logits):
        x2 = x.reshape(-1, x.shape[-1])
        x2, ldx = _rows(x2)
        m, k = x2.shape
        v = w.size(0) if trans_w else w.size(1)
        dev = x.device
        targets = targets.reshape(-1).contiguous()
        weights = weights.reshape(-1).contiguous()
        lse = torch.empty(m, device=dev, dtype=torch.float32)
        xent = torch.empty(m, device=dev, dtype=torch.float32)
        argmax = torch.empty(m, device=dev, dtype=torch.int64)
        w2, ldw = _rows(w)
        logits = torch.empty(m, v, device=dev, dtype=torch.float32) if keep_logits else None
        fused = _on_tensor_cores(False, trans_w, m, v, k, x2, ldx, w2, ldw, _GEMM_BACKEND)
        if fused:
            part = torch.empty(lib.load().nm_logits_xent_scratch(m, v), device=dev,
                               dtype=torch.float32)
            call("nm_logits_xent_fwd", ptr(x2), ldx, ptr(w2), ldw, int(trans_w), ptr(b), unk_index,
                 ptr(targets), ptr(weights), ptr(lse), ptr(xent), ptr(argmax), ptr(part),
                 ptr(logits), v, m, v, k, lib.stream())
        else:
            if logits is None:
                logits = torch.empty(m, v, device=dev, dtype=torch.float32)
            gemm(x2, w2, logits, trans_b=trans_w, bias=b)
            call("nm_xent_fwd", ptr(logits), unk_index, ptr(targets), ptr(weights), ptr(lse), ptr(xent),
                 ptr(argmax), m, v, v, lib.stream())
        ctx.save_for_backward(x2, w2, b, targets, weights, lse, None if fused else logits)
        ctx.cfg = (fused, unk_index, trans_w, x.shape)
        ctx.sinks = (_sink(w), _sink(b) if b is not None else None)
        ctx.mark_non_differentiable(lse, argmax)
        if keep_logits:
            ctx.mark_non_differentiable(logits)
            return xent, lse, argmax, logits
        return xent, lse, argmax, None

    @staticmethod
    def backward(ctx, dxent, _dlse, _dargmax, _dlogits):
        x2, w2, b, targets, weights, lse, logits = ctx.saved_tensors
        fused, unk_index, trans_w, in_shape = ctx.cfg
        m, k = x2.shape
        v = w2.size(0) if trans_w else w2.size(1)
        dev = x2.device
        # fold the upstream per-row gradient into the row weights (tiny [M] product)
        roww = torch.empty(m, device=dev, dtype=torch.float32)
        ones = torch.ones(1, device=dev, dtype=torch.float32)
        torch.mul(weights, dxent.reshape(-1), out=roww)
        if fused:
            dlogits = torch.empty(m, v, device=dev, dtype=torch.float32)
            _, ldx = _rows(x2)
            _, ldw = _rows(w2)
            call("nm_logits_xent_bwd", ptr(x2), ldx, ptr(w2), ldw, int(trans_w), ptr(b), unk_index,
                 ptr(targets), ptr(roww), ptr(lse), ptr(ones), ptr(dlogits), v, m, v, k, lib.stream())
        else:
            dlogits = logits  # in place
            call("nm_xent_bwd", ptr(logits), ptr(targets), ptr(roww), ptr(lse), ptr(ones),
                 ptr(dlogits), m, v, v, lib.stream())
        dx = dw = db = None
        if ctx.needs_input_grad[0]:
            dx = torch.empty(m, k, device=dev, dtype=torch.float32)
            gemm(dlogits, w2, dx, trans_b=not trans_w)
            dx = dx.view(in_shape)
        w_sink, b_sink = ctx.sinks
        want_w, want_b = ctx.needs_input_grad[1], b is not None and ctx.needs_input_grad[2]
        if want_w:
            if trans_w:   # w is [V,K]: dW = dlogits^T @ x
                dw = _weight_grad(dlogits, x2, True, False, w_sink, w2.shape)
            else:         # w is [K,V]: dW = x^T @ dlogits
                dw = _weight_grad(x2, dlogits, True, False, w_sink, w2.shape)
        if want_b:
            db = _bias_grad(dlogits, b_sink)
        return dx, dw, db, None, None, None, None, None


def logits_xent(x: torch.Tensor, w: torch.Tensor, b: Optional[torch.Tensor], targets: torch.Tensor,
                weights: torch.Tensor, unk_index: int = -1, trans_w: bool = False,
                keep_logits: bool = False):
    """Vocabulary projection + masked cross-entropy (decoders/autoregressive.py:288-316,450-459).

    Returns (xent [M], lse [M], argmax [M] int64, logits [M,V] or None)."""
    if (not trans_w and b is not None and _GEMM_BACKEND != lib.GEMM_SIMT
            and w.requires_grad and b.requires_grad):
        w_sink, b_sink = _sink(w), _sink(b)
        k, v = w.shape
        if (w_sink is not None and b_sink is not None and w_sink.is_contiguous()
                and b_sink.data_ptr() == w_sink.data_ptr() + 4 * k * v):
            return _LogitsXent16.apply(x, w, b, targets, weights, unk_index, keep_logits)
    return _LogitsXent.apply(x, w, b, targets, weights, unk_index, trans_w, keep_logits)


# ---------------------------------------------------------------------------
# K8 multi-head attention core
# ---------------------------------------------------------------------------
class _MHA(torch.autograd.Function):
    @staticmethod
    def forward(ctx, q, k, v, key_mask, causal, heads):
        bsz, tq, d = q.shape
        tk = k.size(1)
        dh = d // heads
        q, k, v = q.contiguous(), k.contiguous(), v.contiguous()
        mask_c = key_mask.contiguous() if key_mask is not None else None
        out = torch.empty_like(q)
        probs = torch.empty(bsz, heads, tq, tk, device=q.device, dtype=torch.float32)
        call("nm_mha_fwd", ptr(q), ptr(k), ptr(v), ptr(mask_c), int(causal), ptr(out), ptr(probs), bsz,
             tq, tk, heads, dh, lib.stream())
        ctx.save_for_backward(q, k, v, mask_c, probs)
        ctx.cfg = (causal, heads)
        ctx.mark_non_differentiable(probs)
        return out, probs

    @staticmethod
    def backward(ctx, dout, _dprobs):
        q, k, v, mask, probs = ctx.saved_tensors
        causal, heads = ctx.cfg
        bsz, tq, d = q.shape
        tk = k.size(1)
        dout = dout.contiguous()
        dq, dk, dv = torch.empty_like(q), torch.empty_like(k), torch.empty_like(v)
        work = torch.empty_like(probs)
        call("nm_mha_bwd", ptr(q), ptr(k), ptr(v), ptr(mask), int(causal), ptr(probs), ptr(dout),
             ptr(dq), ptr(dk), ptr(dv), ptr(work), bsz, tq, tk, heads, d // heads, lib.stream())
        return dq, dk, dv, None, None, None


class _MHADrop(torch.autograd.Function):
    """_MHA with attention-weight dropout: `drop_mask` [B, heads, Tq, Tk] holds 0 or 1/keep_prob.  Every
    shape _MHA takes: both kernel families of csrc/mha.cu apply the mask."""

    @staticmethod
    def forward(ctx, q, k, v, key_mask, causal, heads, drop_mask):
        bsz, tq, d = q.shape
        tk = k.size(1)
        q, k, v = q.contiguous(), k.contiguous(), v.contiguous()
        mask_c = key_mask.contiguous() if key_mask is not None else None
        drop_c = drop_mask.to(torch.float32).contiguous()
        out = torch.empty_like(q)
        probs = torch.empty(bsz, heads, tq, tk, device=q.device, dtype=torch.float32)
        call("nm_mha_fwd_drop", ptr(q), ptr(k), ptr(v), ptr(mask_c), int(causal), ptr(drop_c), ptr(out),
             ptr(probs), bsz, tq, tk, heads, d // heads, lib.stream())
        ctx.save_for_backward(q, k, v, mask_c, probs, drop_c)
        ctx.cfg = (causal, heads)
        ctx.mark_non_differentiable(probs)
        return out, probs

    @staticmethod
    def backward(ctx, dout, _dprobs):
        q, k, v, mask, probs, drop_c = ctx.saved_tensors
        causal, heads = ctx.cfg
        bsz, tq, d = q.shape
        tk = k.size(1)
        dout = dout.contiguous()
        dq, dk, dv = torch.empty_like(q), torch.empty_like(k), torch.empty_like(v)
        work = torch.empty_like(probs)
        call("nm_mha_bwd_drop", ptr(q), ptr(k), ptr(v), ptr(mask), int(causal), ptr(drop_c), ptr(probs),
             ptr(dout), ptr(dq), ptr(dk), ptr(dv), ptr(work), bsz, tq, tk, heads, d // heads, lib.stream())
        return dq, dk, dv, None, None, None, None


def _tma_operand(t: torch.Tensor) -> torch.Tensor:
    """t contiguous and starting on a 16-byte boundary, as a tensor map addresses it: a copy when a view starts
    elsewhere."""
    t = t.contiguous()
    return t if t.data_ptr() % 16 == 0 else t.clone()


class _MHATensorCore(torch.autograd.Function):
    """The attention core as batched wgmma products (csrc/mha_tc.cu): softmax and its backward in the GEMM
    epilogues, all (sentence, head) pairs in one launch per product.  TF32 operands."""

    @staticmethod
    def forward(ctx, q, k, v, key_mask, causal, heads, drop_mask):
        bsz, tq, d = q.shape
        tk = k.size(1)
        q, k, v = _tma_operand(q), _tma_operand(k), _tma_operand(v)
        mask_c = key_mask.contiguous() if key_mask is not None else None
        drop_c = drop_mask.to(torch.float32).contiguous() if drop_mask is not None else None
        tqp, tkp = (tq + 31) // 32 * 32, (tk + 31) // 32 * 32
        out = torch.empty_like(q)
        probs = torch.empty(bsz, heads, tqp, tkp, device=q.device, dtype=torch.float32)
        probs_drop = torch.empty_like(probs) if drop_c is not None else None
        call("nm_mha_tc_fwd", ptr(q), ptr(k), ptr(v), ptr(mask_c), int(causal), ptr(drop_c), ptr(out), ptr(probs),
             ptr(probs_drop), bsz, tq, tk, heads, d // heads, lib.stream())
        ctx.save_for_backward(q, k, v, mask_c, probs, probs_drop, drop_c)
        ctx.cfg = (causal, heads)
        weights = probs[:, :, :tq, :tk]
        ctx.mark_non_differentiable(weights)
        return out, weights

    @staticmethod
    def backward(ctx, dout, _dprobs):
        q, k, v, mask, probs, probs_drop, drop_c = ctx.saved_tensors
        causal, heads = ctx.cfg
        bsz, tq, d = q.shape
        tk = k.size(1)
        dout = _tma_operand(dout)
        dq, dk, dv = torch.empty_like(q), torch.empty_like(k), torch.empty_like(v)
        work = torch.empty_like(probs)
        call("nm_mha_tc_bwd", ptr(q), ptr(k), ptr(v), ptr(mask), int(causal), ptr(drop_c), ptr(probs),
             ptr(probs_drop), ptr(dout), ptr(dq), ptr(dk), ptr(dv), ptr(work), bsz, tq, tk, heads, d // heads,
             lib.stream())
        return dq, dk, dv, None, None, None, None


def _mha_on_tensor_cores(bsz: int, tq: int, tk: int, heads: int, dh: int) -> bool:
    """Tensor-core attention follows the GEMM backend ('simt' = the exact fp32 kernels everywhere); whole
    sequences only - the single-query steps of the decoding loops stay on the row kernels."""
    if _GEMM_BACKEND == lib.GEMM_SIMT or tq < 8:
        return False
    return bool(lib.load().nm_mha_tc_supported(bsz, tq, tk, heads, dh))


def mha_core(q: torch.Tensor, k: torch.Tensor, v: torch.Tensor, key_mask: Optional[torch.Tensor],
             causal: bool, heads: int, drop_mask: Optional[torch.Tensor] = None) -> Tuple[torch.Tensor, torch.Tensor]:
    """softmax(mask(q/sqrt(dh) k^T)) v per head (attention/scaled_dot_product.py:184-214).  With
    `drop_mask` ([B, heads, Tq, Tk], 0 or 1/keep_prob) the context is (softmax * drop_mask) v; the
    returned weights are the undropped softmax."""
    if q.is_cuda and _mha_on_tensor_cores(q.shape[0], q.shape[1], k.shape[1], heads, q.shape[2] // heads):
        return _MHATensorCore.apply(q, k, v, key_mask, causal, heads, drop_mask)
    if drop_mask is not None:
        return _MHADrop.apply(q, k, v, key_mask, causal, heads, drop_mask)
    return _MHA.apply(q, k, v, key_mask, causal, heads)


# ---------------------------------------------------------------------------
# non-differentiable helpers
# ---------------------------------------------------------------------------
def xent_rows(logits: torch.Tensor, targets: Optional[torch.Tensor] = None,
              weights: Optional[torch.Tensor] = None, want_argmax: bool = False, first_col: int = 0):
    """Row statistics of materialised logits [M, V] (contiguous rows) over columns first_col..V-1:
    (lse [M], weighted xent [M] or None without targets, first-index argmax [M] int64 relative to
    first_col or None).  One `nm_xent_fwd` launch; the column offset is pointer arithmetic with ld = V."""
    m, v = logits.shape
    dev = logits.device
    lse = torch.empty(m, device=dev, dtype=torch.float32)
    xent = torch.empty(m, device=dev, dtype=torch.float32) if targets is not None else None
    arg = torch.empty(m, device=dev, dtype=torch.int64) if want_argmax else None
    call("nm_xent_fwd", ptr(logits) + 4 * first_col, -1, ptr(targets), ptr(weights), ptr(lse), ptr(xent),
         ptr(arg), m, v - first_col, v, lib.stream())
    return lse, xent, arg


def log_softmax_from_lse(logits: torch.Tensor, lse: torch.Tensor) -> torch.Tensor:
    m, v = logits.shape
    out = torch.empty_like(logits)
    call("nm_log_softmax", ptr(logits), ptr(lse), ptr(out), m, v, logits.stride(0), lib.stream())
    return out


def beam_step(logprobs: torch.Tensor, logprob_sum: torch.Tensor, lengths: torch.Tensor,
              finished: torch.Tensor, alpha: float):
    """One BeamSearchDecoder step (beam_search_decoder.py:440-496).  Returns
    (scores, word_ids i64, beam_ids i32, logprob_sum', lengths' i32, finished' u8)."""
    bsz, k, v = logprobs.shape
    dev = logprobs.device
    scores = torch.empty(bsz, k, device=dev, dtype=torch.float32)
    words = torch.empty(bsz, k, device=dev, dtype=torch.int64)
    beams = torch.empty(bsz, k, device=dev, dtype=torch.int32)
    lsum = torch.empty(bsz, k, device=dev, dtype=torch.float32)
    lens = torch.empty(bsz, k, device=dev, dtype=torch.int32)
    fin = torch.empty(bsz, k, device=dev, dtype=torch.uint8)
    scratch = torch.empty(lib.load().nm_beam_scratch(bsz, k, v), device=dev, dtype=torch.int32)
    call("nm_beam_step", ptr(logprobs.contiguous()), ptr(logprob_sum.contiguous()),
         ptr(lengths.contiguous()), ptr(finished.contiguous()), float(alpha), ptr(scores), ptr(words),
         ptr(beams), ptr(lsum), ptr(lens), ptr(fin), ptr(scratch), bsz, k, v, lib.stream())
    return scores, words, beams, lsum, lens, fin


def beam_gather(x: torch.Tensor, beam_ids: torch.Tensor, bsz: int, k: int) -> torch.Tensor:
    """gather_flat (tf_utils.py:106-131) on a [B*k, ...] tensor."""
    x = x.contiguous()
    out = torch.empty_like(x)
    row_bytes = (x.numel() // (bsz * k)) * x.element_size()
    call("nm_beam_gather", ptr(x), ptr(beam_ids.contiguous()), ptr(out), bsz, k, row_bytes,
         lib.stream())
    return out


# ---------------------------------------------------------------------------
# K16 CTC loss and greedy CTC decoding
# ---------------------------------------------------------------------------
def _ctc_workspace_words(bsz: int, t: int, lmax: int) -> int:
    return bsz * t * (5 * lmax + 4) + bsz * (lmax + 4)      # the size nm_ctc_loss_fwd documents


class _CTCLoss(torch.autograd.Function):
    @staticmethod
    def forward(ctx, logits, frames, labels, label_lengths, merge_repeated):
        bsz, t, c = logits.shape
        lmax = labels.shape[1]
        words = _ctc_workspace_words(bsz, t, lmax)
        ws = torch.empty(words, device=logits.device, dtype=torch.float32)
        loss = torch.empty(bsz, device=logits.device, dtype=torch.float32)
        call("nm_ctc_loss_fwd", ptr(logits), ptr(frames), ptr(labels), ptr(label_lengths), int(merge_repeated),
             ptr(loss), ptr(ws), words, bsz, t, c, lmax, lib.stream())
        ctx.save_for_backward(logits, frames, labels, label_lengths, ws)
        ctx.merge = int(merge_repeated)
        return loss

    @staticmethod
    def backward(ctx, dloss):
        logits, frames, labels, label_lengths, ws = ctx.saved_tensors
        bsz, t, c = logits.shape
        dloss = _f32(dloss).contiguous()
        dlogits = torch.empty_like(logits)
        call("nm_ctc_loss_bwd", ptr(logits), ptr(frames), ptr(labels), ptr(label_lengths), ctx.merge, ptr(dloss),
             ptr(dlogits), ptr(ws), ws.numel(), bsz, t, c, labels.shape[1], lib.stream())
        return dlogits, None, None, None, None


def _ctc_inputs(logits: torch.Tensor, frames: torch.Tensor):
    if logits.dim() != 3:
        raise ValueError("CTC logits must be [batch, time, classes], got {}".format(tuple(logits.shape)))
    if frames.dtype != torch.int32 or frames.shape != (logits.shape[0],):
        raise ValueError("CTC frames must be int32 [batch]")
    return _f32(logits).contiguous(), frames.contiguous()


def ctc_loss(logits: torch.Tensor, frames: torch.Tensor, labels: torch.Tensor, label_lengths: torch.Tensor,
             merge_repeated: bool) -> torch.Tensor:
    """Per-sentence -log p(labels | logits) of tf.nn.ctc_loss(ignore_longer_outputs_than_inputs=True,
    ctc_merge_repeated=merge_repeated) (decoders/ctc_decoder.py:96-104).  logits [B, T, C] (blank = C-1),
    frames [B] int32, labels [B, Lmax] int64 (the first label_lengths[b] entries of row b; int32 lengths).
    Differentiable in the logits: the backward pass returns the dense dlogits."""
    logits, frames = _ctc_inputs(logits, frames)
    if labels.dtype != torch.int64 or labels.dim() != 2 or labels.shape[0] != logits.shape[0]:
        raise ValueError("CTC labels must be int64 [batch, max label length]")
    if label_lengths.dtype != torch.int32 or label_lengths.shape != (logits.shape[0],):
        raise ValueError("CTC label lengths must be int32 [batch]")
    return _CTCLoss.apply(logits, frames, labels.contiguous(), label_lengths.contiguous(), bool(merge_repeated))


def ctc_greedy_decode(logits: torch.Tensor, frames: torch.Tensor, merge_repeated: bool):
    """tf.nn.ctc_greedy_decoder (decoders/ctc_decoder.py:77-80) over batch-major logits [B, T, C]: returns
    (ids [B, T] int64 padded with </s>, lengths [B] int32)."""
    logits, frames = _ctc_inputs(logits.detach(), frames)
    bsz, t, c = logits.shape
    ids = torch.empty(bsz, t, device=logits.device, dtype=torch.int64)
    lengths = torch.empty(bsz, device=logits.device, dtype=torch.int32)
    call("nm_ctc_greedy_decode", ptr(logits), ptr(frames), int(merge_repeated), ptr(ids), ptr(lengths), bsz, t, c,
         lib.stream())
    return ids, lengths


# ---------------------------------------------------------------------------
# K17 rewards and sampling of the reinforcement-learning objectives
# ---------------------------------------------------------------------------
REWARD_MODES = {"bleu": 0, "gleu": 1}


def sentence_ngram_reward(references: torch.Tensor, hypotheses: torch.Tensor, mode: str) -> torch.Tensor:
    """Index-based sentence BLEU or GLEU (trainers/self_critical_objective.py:124-231) of time-major int64 token
    ids references [T_r, B] and hypotheses [T_h, B], any strides: [B] float32 on the device."""
    if references.dim() != 2 or hypotheses.dim() != 2 or references.shape[1] != hypotheses.shape[1]:
        raise ValueError("references and hypotheses must be [time, batch] with the same batch, got {} and {}"
                         .format(tuple(references.shape), tuple(hypotheses.shape)))
    if references.dtype != torch.int64 or hypotheses.dtype != torch.int64:
        raise ValueError("token ids must be int64")
    t_r, bsz = references.shape
    t_h = hypotheses.shape[0]
    reward = torch.empty(bsz, device=references.device, dtype=torch.float32)
    call("nm_sentence_ngram_reward", ptr(references), references.stride(0), references.stride(1), ptr(hypotheses),
         hypotheses.stride(0), hypotheses.stride(1), ptr(reward), t_r, t_h, bsz, REWARD_MODES[mode], lib.stream())
    return reward


def sample_logits_step(logits: torch.Tensor, temperature: float, finished: torch.Tensor, unk_index: int,
                       loop_step: int, sample_index: int):
    """One draw per row of logits [rows, V] (unit column stride) from softmax(logits / temperature), never column
    `unk_index`, then get_body's bookkeeping: symbols = draw * ~finished, finished |= symbols == </s>.  The
    random stream is the runtime's {seed, step} with (row, loop_step, sample_index) in the counter.
    Returns (symbols [rows] int64, finished [rows] bool)."""
    from neuralmonkey_b200 import runtime
    rows, v = logits.shape
    if logits.dtype != torch.float32 or logits.stride(1) != 1:
        raise ValueError("sample_logits_step needs fp32 logits with unit column stride")
    if finished.dtype != torch.bool or finished.shape != (rows,):
        raise ValueError("finished must be bool [rows]")
    symbols = torch.empty(rows, device=logits.device, dtype=torch.int64)
    finished_out = torch.empty(rows, device=logits.device, dtype=torch.bool)
    call("nm_sample_logits_step", ptr(logits), logits.stride(0), float(temperature), int(unk_index),
         ptr(finished.contiguous()), ptr(symbols), ptr(finished_out), ptr(runtime.dropout_state()), int(loop_step),
         int(sample_index), rows, v, lib.stream())
    return symbols, finished_out


# ---------------------------------------------------------------------------
# K12 frozen VGG stack primitives (forward only)
# ---------------------------------------------------------------------------
def conv3x3_bias_relu(x: torch.Tensor, w: torch.Tensor, b: torch.Tensor) -> torch.Tensor:
    """NHWC 3x3 SAME conv + bias + ReLU; w is HWIO (slim vgg_arg_scope)."""
    n, h, wd, cin = x.shape
    cout = w.shape[-1]
    x, w, b = _f32(x.detach()).contiguous(), _f32(w.detach()).contiguous(), _f32(b.detach())
    y = torch.empty(n, h, wd, cout, device=x.device, dtype=torch.float32)
    if _GEMM_BACKEND != lib.GEMM_SIMT and cout % 4 == 0:
        # tensor-core path: patch matrix (im2col) x filter matrix [9*Cin, Cout] through the wgmma
        # GEMM with the bias + ReLU epilogue; the output rows ARE the NHWC pixels.  The patch matrix
        # is built for a few images at a time so it stays below ~768 MB.
        k = 9 * cin
        ld = (k + 3) // 4 * 4
        per_image = h * wd * ld * 4
        chunk = max(1, min(n, (768 << 20) // per_image))
        cols = torch.zeros(chunk * h * wd, ld, device=x.device, dtype=torch.float32)
        w2 = w.view(k, cout)
        y2 = y.view(n * h * wd, cout)
        for n0 in range(0, n, chunk):
            nb = min(chunk, n - n0)
            call("nm_im2col3x3", ptr(x[n0:n0 + nb]), ptr(cols), nb, h, wd, cin, ld, lib.stream())
            gemm(cols[:nb * h * wd, :k], w2, y2[n0 * h * wd:(n0 + nb) * h * wd], bias=b, act="relu")
        return y
    call("nm_conv3x3_bias_relu_fwd", ptr(x), ptr(w), ptr(b), ptr(y), n, h, wd, cin, cout, lib.stream())
    return y


def maxpool2x2(x: torch.Tensor) -> torch.Tensor:
    n, h, wd, c = x.shape
    x = _f32(x.detach()).contiguous()
    y = torch.empty(n, h // 2, wd // 2, c, device=x.device, dtype=torch.float32)
    call("nm_maxpool2x2_fwd", ptr(x), ptr(y), n, h, wd, c, lib.stream())
    return y


def conv2d_bn_fwd(x: torch.Tensor, w: torch.Tensor, stride: int = 1, pads: Tuple[int, int] = (0, 0),
                  in_scale: Optional[torch.Tensor] = None, in_shift: Optional[torch.Tensor] = None,
                  out_scale: Optional[torch.Tensor] = None, out_shift: Optional[torch.Tensor] = None,
                  bias: Optional[torch.Tensor] = None, res: Optional[torch.Tensor] = None, res_stride: int = 1,
                  act: Optional[str] = None) -> torch.Tensor:
    """One frozen ResNet-v2 convolution (nm_conv2d_bn_fwd), forward only: NHWC x, HWIO w [k,k,Cin,Cout], `pads`
    (before, after) on both axes, then
        y = act(z + res[:, ::res_stride, ::res_stride]),  z = conv(A, w) * out_scale + out_shift  or  conv(A, w) + bias,
    A = relu(x * in_scale + in_shift) (0 in the padding) when in_scale is given, else x.  The exact fp32 kernels
    under the 'simt' GEMM backend, wgmma with TF32 operands otherwise."""
    if act not in (None, "relu"):
        raise ValueError("conv2d_bn_fwd: act must be None or 'relu'")
    n, h, wd, cin = x.shape
    k, cout = w.shape[0], w.shape[3]
    if tuple(w.shape[1:3]) != (k, cin):
        raise ValueError("conv2d_bn_fwd: filter {} does not fit input {}".format(tuple(w.shape), tuple(x.shape)))
    pt, pb = pads
    ho, wo = (h + pt + pb - k) // stride + 1, (wd + pt + pb - k) // stride + 1

    def vec(t):
        return None if t is None else _f32(t.detach()).contiguous()

    x, w = _f32(x.detach()).contiguous(), _f32(w.detach()).contiguous()
    res_h = res_w = 0
    if res is not None:
        res = vec(res)
        if res.shape[0] != n or res.shape[3] != cout:
            raise ValueError("conv2d_bn_fwd: residual {} does not fit output {}".format(
                tuple(res.shape), (n, ho, wo, cout)))
        res_h, res_w = res.shape[1], res.shape[2]
    vecs = [vec(t) for t in (in_scale, in_shift, out_scale, out_shift, bias)]   # alive until the call returns
    y = torch.empty(n, max(ho, 0), max(wo, 0), cout, device=x.device, dtype=torch.float32)
    call("nm_conv2d_bn_fwd", ptr(x), ptr(w), *[ptr(t) for t in vecs], ptr(res), res_h, res_w, res_stride, ptr(y), n,
         h, wd, cin, cout, k, stride, pt, pb, pt, pb, lib.NM_ACT[act], _conv_backend(), lib.stream())
    return y


# ---------------------------------------------------------------------------
# K12b trainable CNN layers (encoders/cnn_encoder.py): convolution, batch normalization, pooling
# ---------------------------------------------------------------------------
def conv_pads(k: int, padding: str) -> Tuple[int, int]:
    """(before, after) of one spatial axis at stride 1: TensorFlow's `same` puts the odd pixel after."""
    if padding == "valid":
        return 0, 0
    if padding == "same":
        return (k - 1) // 2, k - 1 - (k - 1) // 2
    raise ValueError("padding must be 'same' or 'valid', got {!r}".format(padding))


def _conv_backend() -> int:
    """The exact fp32 kernels under the 'simt' GEMM backend, wgmma with TF32 operands otherwise."""
    return lib.GEMM_SIMT if _GEMM_BACKEND == lib.GEMM_SIMT else lib.GEMM_AUTO


# the weight-gradient partials of one call: as many [k*k*Cin+1, Cout] slices as the kernel splits the pixel
# reduction into (nm_conv2d_wgrad_workspace), at most 64 MB, at least one slice
_WGRAD_WS_FLOATS = 16 << 20


def conv_wgrad_workspace(n, h, wd, cin, cout, k, pt, pb, backend) -> int:
    want = int(lib.load().nm_conv2d_wgrad_workspace(n, h, wd, cin, cout, k, pt, pb, pt, pb, backend))
    if want < 0:
        raise ValueError("conv2d: bad sizes {}".format((n, h, wd, cin, cout, k, pt, pb)))
    return max((k * k * cin + 1) * cout, min(_WGRAD_WS_FLOATS, want))


class _Conv2d(torch.autograd.Function):
    @staticmethod
    def forward(ctx, x, w, b, padding, act):
        n, h, wd, cin = x.shape
        k, cout = w.shape[0], w.shape[3]
        if w.shape[1] != k or w.shape[2] != cin:
            raise ValueError("conv2d: filter {} does not fit input {}".format(tuple(w.shape), tuple(x.shape)))
        pt, pb = conv_pads(k, padding)
        x = _f32(x).contiguous()
        w = _f32(w).contiguous()
        ho, wo = h + pt + pb - k + 1, wd + pt + pb - k + 1
        y = torch.empty(n, ho, wo, cout, device=x.device, dtype=torch.float32)
        backend = _conv_backend()
        call("nm_conv2d_fwd", ptr(x), ptr(w), ptr(b), ptr(y), n, h, wd, cin, cout, k, pt, pb, pt, pb, 0,
             lib.NM_ACT[act], backend, lib.stream())
        ctx.save_for_backward(x, w, y if act is not None else None)
        ctx.geom = (n, h, wd, cin, cout, k, pt, pb, backend, act)
        ctx.sinks = (_sink(w), _sink(b) if b is not None else None)
        ctx.has_bias = b is not None
        return y

    @staticmethod
    def backward(ctx, dy):
        x, w, y = ctx.saved_tensors
        n, h, wd, cin, cout, k, pt, pb, backend, act = ctx.geom
        dy = dy.contiguous()
        if act is not None:
            dpre = torch.empty_like(dy)
            call("nm_act_bwd", ptr(y), ptr(dy), ptr(dpre), dy.numel(), lib.NM_ACT[act], lib.stream())
            dy = dpre
        ho, wo = dy.shape[1], dy.shape[2]
        dx = None
        if ctx.needs_input_grad[0]:
            dx = torch.empty_like(x)
            call("nm_conv2d_fwd", ptr(dy), ptr(w), None, ptr(dx), n, ho, wo, cout, cin, k, k - 1 - pt, k - 1 - pb,
                 k - 1 - pt, k - 1 - pb, 1, 0, backend, lib.stream())
        w_sink, b_sink = ctx.sinks
        dw = w_sink if w_sink is not None else torch.zeros_like(w)
        db = None
        if ctx.has_bias:
            db = b_sink if b_sink is not None else torch.zeros(cout, device=x.device, dtype=torch.float32)
        ws = torch.empty(conv_wgrad_workspace(n, h, wd, cin, cout, k, pt, pb, backend), device=x.device,
                         dtype=torch.float32)
        call("nm_conv2d_wgrad", ptr(x), ptr(dy), ptr(dw), ptr(db), ptr(ws), ws.numel(), n, h, wd, cin, cout, k, pt,
             pb, pt, pb, backend, lib.stream())
        return (dx, None if w_sink is not None else dw,
                None if (b_sink is not None or not ctx.has_bias) else db, None, None)


def conv2d(x: torch.Tensor, w: torch.Tensor, b: Optional[torch.Tensor], padding: str,
           act: Optional[str] = None) -> torch.Tensor:
    """tf.layers.conv2d at stride 1: NHWC x, HWIO w, `same` or `valid` padding, act None or 'relu'."""
    if act not in (None, "relu"):
        raise ValueError("conv2d: act must be None or 'relu'")
    return _Conv2d.apply(x, w, b, padding, act)


def glu_conv_wgrad_workspace(bsz, t, f, k, backend) -> int:
    want = int(lib.load().nm_glu_conv1d_wgrad_workspace(bsz, t, f, k, backend))
    if want < 0:
        raise ValueError("conv1d_glu_residual: bad sizes {}".format((bsz, t, f, k)))
    return max((k * f + 1) * 2 * f, min(_WGRAD_WS_FLOATS, want))


class _Conv1dGluResidual(torch.autograd.Function):
    @staticmethod
    def forward(ctx, x, w, b):
        bsz, t, f = x.shape
        k = w.shape[0]
        if w.shape[1:] != (f, 2 * f) or tuple(b.shape) != (2 * f,):
            raise ValueError("conv1d_glu_residual: filter {} / bias {} do not fit input {}".format(
                tuple(w.shape), tuple(b.shape), tuple(x.shape)))
        x = _f32(x).contiguous()
        w = _f32(w).contiguous()
        b = _f32(b).contiguous()
        y = torch.empty_like(x)
        training = any(ctx.needs_input_grad)
        z = torch.empty(bsz, t, 2 * f, device=x.device, dtype=torch.float32) if training else None
        backend = _conv_backend()
        call("nm_glu_conv1d_fwd", ptr(x), ptr(w), ptr(b), ptr(y), ptr(z), bsz, t, f, k, backend, lib.stream())
        ctx.save_for_backward(x, w, z)
        ctx.geom = (bsz, t, f, k, backend)
        ctx.sinks = (_sink(w), _sink(b))
        return y

    @staticmethod
    def backward(ctx, dy):
        x, w, z = ctx.saved_tensors
        bsz, t, f, k, backend = ctx.geom
        dy = _f32(dy).contiguous()
        dz = torch.empty_like(z)
        call("nm_glu_conv1d_dz", ptr(dy), ptr(z), ptr(dz), bsz * t, f, lib.stream())
        dx = None
        if ctx.needs_input_grad[0]:
            dx = torch.empty_like(x)
            call("nm_glu_conv1d_dgrad", ptr(dz), ptr(w), ptr(dy), ptr(dx), bsz, t, f, k, backend, lib.stream())
        w_sink, b_sink = ctx.sinks
        if not (ctx.needs_input_grad[1] or ctx.needs_input_grad[2]):
            return dx, None, None
        dw = w_sink if w_sink is not None else torch.zeros_like(w)
        db = b_sink if b_sink is not None else torch.zeros(2 * f, device=x.device, dtype=torch.float32)
        ws = torch.empty(glu_conv_wgrad_workspace(bsz, t, f, k, backend), device=x.device, dtype=torch.float32)
        call("nm_glu_conv1d_wgrad", ptr(x), ptr(dz), ptr(dw), ptr(db), ptr(ws), ws.numel(), bsz, t, f, k, backend,
             lib.stream())
        return dx, None if w_sink is not None else dw, None if b_sink is not None else db


def conv1d_glu_residual(x: torch.Tensor, w: torch.Tensor, b: torch.Tensor) -> torch.Tensor:
    """One ConvS2S encoder layer: z = tf.nn.conv1d(x, w, 1, 'SAME') + b, y = z[..., :F] * sigmoid(z[..., F:]) + x.
    x [B,T,F], w [k,F,2F], b [2F].  The exact fp32 kernels under the 'simt' GEMM backend, wgmma with TF32 operands
    otherwise."""
    return _Conv1dGluResidual.apply(x, w, b)


# ---------------------------------------------------------------------------
# K22 character-level sentence encoder (encoders/sentence_cnn_encoder.py): the one-row convolution, the highway gate
# ---------------------------------------------------------------------------
def conv1d_wgrad_workspace(bsz, t, cin, cout, k, backend) -> int:
    want = int(lib.load().nm_conv1d_wgrad_workspace(bsz, t, cin, cout, k, backend))
    if want < 0:
        raise ValueError("conv1d: bad sizes {}".format((bsz, t, cin, cout, k)))
    return max((k * cin + 1) * cout, min(_WGRAD_WS_FLOATS, want))


class _Conv1d(torch.autograd.Function):
    @staticmethod
    def forward(ctx, x, w, b, act):
        bsz, t, cin = x.shape
        k, cout = w.shape[0], w.shape[2]
        if w.shape[1] != cin or (b is not None and tuple(b.shape) != (cout,)):
            raise ValueError("conv1d: filter {} / bias {} do not fit input {}".format(
                tuple(w.shape), None if b is None else tuple(b.shape), tuple(x.shape)))
        x = _f32(x).contiguous()
        w = _f32(w).contiguous()
        y = torch.empty(bsz, t, cout, device=x.device, dtype=torch.float32)
        backend = _conv_backend()
        call("nm_conv1d_fwd", ptr(x), ptr(w), ptr(b), ptr(y), bsz, t, cin, cout, k, lib.NM_ACT[act], backend,
             lib.stream())
        ctx.save_for_backward(x, w, y if act is not None else None)
        ctx.geom = (bsz, t, cin, cout, k, backend, act)
        ctx.sinks = (_sink(w), _sink(b) if b is not None else None)
        ctx.has_bias = b is not None
        return y

    @staticmethod
    def backward(ctx, dy):
        x, w, y = ctx.saved_tensors
        bsz, t, cin, cout, k, backend, act = ctx.geom
        dy = _f32(dy).contiguous()
        if act is not None:
            dpre = torch.empty_like(dy)
            call("nm_act_bwd", ptr(y), ptr(dy), ptr(dpre), dy.numel(), lib.NM_ACT[act], lib.stream())
            dy = dpre
        dx = None
        if ctx.needs_input_grad[0]:
            dx = torch.empty_like(x)
            call("nm_conv1d_dgrad", ptr(dy), ptr(w), ptr(dx), bsz, t, cin, cout, k, backend, lib.stream())
        w_sink, b_sink = ctx.sinks
        if not (ctx.needs_input_grad[1] or (ctx.has_bias and ctx.needs_input_grad[2])):
            return dx, None, None, None
        dw = w_sink if w_sink is not None else torch.zeros_like(w)
        db = None
        if ctx.has_bias:
            db = b_sink if b_sink is not None else torch.zeros(cout, device=x.device, dtype=torch.float32)
        ws = torch.empty(conv1d_wgrad_workspace(bsz, t, cin, cout, k, backend), device=x.device, dtype=torch.float32)
        call("nm_conv1d_wgrad", ptr(x), ptr(dy), ptr(dw), ptr(db), ptr(ws), ws.numel(), bsz, t, cin, cout, k, backend,
             lib.stream())
        return (dx, None if w_sink is not None else dw,
                None if (b_sink is not None or not ctx.has_bias) else db, None)


def conv1d(x: torch.Tensor, w: torch.Tensor, b: Optional[torch.Tensor], padding: str = "same",
           act: Optional[str] = None) -> torch.Tensor:
    """act(tf.nn.conv1d(x, w, 1, 'SAME') + b): x [B,T,Cin], w [k,Cin,Cout], b [Cout] or None, act None or 'relu'.
    The one-row kernels keep the sequence length, so `padding` is 'same' only.  The exact fp32 kernels under the
    'simt' GEMM backend, wgmma with TF32 operands otherwise."""
    if padding != "same":
        raise ValueError("conv1d: padding must be 'same', got {!r}".format(padding))
    if act not in (None, "relu"):
        raise ValueError("conv1d: act must be None or 'relu'")
    return _Conv1d.apply(x, w, b, act)


class _HighwayGate(torch.autograd.Function):
    @staticmethod
    def forward(ctx, zh, zt, x):
        if zh.shape != x.shape or zt.shape != x.shape:
            raise ValueError("highway_gate: shapes {}, {} and {} differ".format(
                tuple(zh.shape), tuple(zt.shape), tuple(x.shape)))
        zh, zt, x = (_f32(a).contiguous() for a in (zh, zt, x))
        y = torch.empty_like(x)
        call("nm_highway_fwd", ptr(zh), ptr(zt), ptr(x), ptr(y), x.numel(), lib.stream())
        ctx.save_for_backward(zh, zt, x)
        return y

    @staticmethod
    def backward(ctx, dy):
        zh, zt, x = ctx.saved_tensors
        dy = _f32(dy).contiguous()
        dzh, dzt, dx = torch.empty_like(x), torch.empty_like(x), torch.empty_like(x)
        call("nm_highway_bwd", ptr(dy), ptr(zh), ptr(zt), ptr(x), ptr(dzh), ptr(dzt), ptr(dx), x.numel(),
             lib.stream())
        return dzh, dzt, dx


def highway_gate(zh: torch.Tensor, zt: torch.Tensor, x: torch.Tensor) -> torch.Tensor:
    """relu(zh) * sigmoid(zt) + x * (1 - sigmoid(zt)) for the outputs zh, zt of a highway layer's two dense
    products; the backward gives both products' output gradients and the carry term of dx."""
    return _HighwayGate.apply(zh, zt, x)


BN_WS_DOUBLES_PER_CHANNEL = 130     # NM_BN_WS_DOUBLES_PER_CHANNEL


class _BatchNorm(torch.autograd.Function):
    @staticmethod
    def forward(ctx, x, gamma, beta, moving_mean, moving_var, training, relu, momentum, eps):
        c = x.shape[-1]
        x2 = _f32(x).contiguous()
        p = x2.numel() // c
        y = torch.empty_like(x2)
        mean = torch.empty(c, device=x.device, dtype=torch.float32)
        invstd = torch.empty(c, device=x.device, dtype=torch.float32)
        ws = torch.empty(BN_WS_DOUBLES_PER_CHANNEL * c, device=x.device, dtype=torch.float64)
        call("nm_batchnorm_fwd", ptr(x2), ptr(gamma), ptr(beta), ptr(y), ptr(moving_mean), ptr(moving_var), ptr(mean),
             ptr(invstd), ptr(ws), p, c, float(momentum), float(eps), int(training), int(relu), lib.stream())
        ctx.save_for_backward(x2, gamma, beta, mean, invstd)
        ctx.flags = (int(training), int(relu))
        ctx.sinks = (_sink(gamma), _sink(beta))
        return y

    @staticmethod
    def backward(ctx, dy):
        x2, gamma, beta, mean, invstd = ctx.saved_tensors
        training, relu = ctx.flags
        c = x2.shape[-1]
        p = x2.numel() // c
        dy = dy.contiguous()
        dx = torch.empty_like(x2)
        sg, sb = ctx.sinks
        dg = sg if sg is not None else torch.zeros(c, device=dy.device, dtype=torch.float32)
        db = sb if sb is not None else torch.zeros(c, device=dy.device, dtype=torch.float32)
        ws = torch.empty(BN_WS_DOUBLES_PER_CHANNEL * c, device=dy.device, dtype=torch.float64)
        call("nm_batchnorm_bwd", ptr(x2), ptr(dy), ptr(gamma), ptr(beta), ptr(mean), ptr(invstd), ptr(dx), ptr(dg),
             ptr(db), ptr(ws), p, c, training, relu, lib.stream())
        return (dx, None if sg is not None else dg, None if sb is not None else db,
                None, None, None, None, None, None)


def batch_norm(x: torch.Tensor, gamma: torch.Tensor, beta: torch.Tensor, moving_mean: torch.Tensor,
               moving_var: torch.Tensor, training: bool, relu: bool = False, momentum: float = 0.99,
               eps: float = 1e-3) -> torch.Tensor:
    """tf.layers.batch_normalization over the last axis (TF 1.x defaults), optionally followed by ReLU.  In
    training the moving statistics are updated in place (the UPDATE_OPS the reference's trainer runs)."""
    return _BatchNorm.apply(x, gamma, beta, moving_mean, moving_var, bool(training), bool(relu), momentum, eps)


def pool_out(size: int, k: int, stride: int, padding: str) -> int:
    if padding == "same":
        return -(-size // stride)
    return (size - k) // stride + 1


class _Pool2d(torch.autograd.Function):
    @staticmethod
    def forward(ctx, x, k, stride, padding, is_max):
        n, h, wd, c = x.shape
        x = _f32(x).contiguous()
        y = torch.empty(n, pool_out(h, k, stride, padding), pool_out(wd, k, stride, padding), c, device=x.device,
                        dtype=torch.float32)
        same = int(padding == "same")
        call("nm_pool2d_fwd", ptr(x), ptr(y), n, h, wd, c, k, stride, same, int(is_max), lib.stream())
        ctx.save_for_backward(x)
        ctx.geom = (k, stride, same, int(is_max))
        return y

    @staticmethod
    def backward(ctx, dy):
        (x,) = ctx.saved_tensors
        k, stride, same, is_max = ctx.geom
        n, h, wd, c = x.shape
        dx = torch.empty_like(x)
        call("nm_pool2d_bwd", ptr(x), ptr(dy.contiguous()), ptr(dx), n, h, wd, c, k, stride, same, is_max,
             lib.stream())
        return dx, None, None, None, None


def pool2d(x: torch.Tensor, k: int, stride: int, padding: str, kind: str) -> torch.Tensor:
    """tf.layers.max_pooling2d (kind 'max') / average_pooling2d ('avg') over NHWC x."""
    if padding not in ("same", "valid"):
        raise ValueError("padding must be 'same' or 'valid', got {!r}".format(padding))
    if kind not in ("max", "avg"):
        raise ValueError("pooling kind must be 'max' or 'avg'")
    return _Pool2d.apply(x, int(k), int(stride), padding, kind == "max")


# ---------------------------------------------------------------------------
# K18 sentence classification and regression (csrc/classify.cu): pooling over time, self-attentive pooling,
# the Kim-CNN convolution + max over time, the squared-error loss
# ---------------------------------------------------------------------------
def _mask_or_none(mask: Optional[torch.Tensor], b: int, t: int) -> Optional[torch.Tensor]:
    if mask is None:
        return None
    if tuple(mask.shape) != (b, t):
        raise ValueError("mask must be [{}, {}], got {}".format(b, t, tuple(mask.shape)))
    return _f32(mask).contiguous()


def _check_mask_sum(mask: Optional[torch.Tensor]) -> None:
    """The reference's tf.assert_greater(reduce_sum(mask), 0.5) before its max pooling (encoders/pooling.py:53)."""
    if mask is not None and float(mask.sum()) <= 0.5:
        raise ValueError("max pooling over a batch without a single valid position (mask sum <= 0.5)")


class _SeqMaxPool(torch.autograd.Function):
    @staticmethod
    def forward(ctx, x, mask):
        b, t, d = x.shape
        x = _f32(x).contiguous()
        y = torch.empty(b, d, device=x.device, dtype=torch.float32)
        call("nm_seq_max_pool_fwd", ptr(x), ptr(mask), ptr(y), b, t, t, d, 0, lib.stream())
        ctx.save_for_backward(x, mask)
        return y

    @staticmethod
    def backward(ctx, dy):
        x, mask = ctx.saved_tensors
        b, t, d = x.shape
        dx = torch.empty_like(x)
        call("nm_seq_max_pool_bwd", ptr(x), ptr(mask), ptr(dy.contiguous()), ptr(dx), b, t, t, d, b * t, 0,
             lib.stream())
        return dx, None


def seq_max_pool(x: torch.Tensor, mask: Optional[torch.Tensor]) -> torch.Tensor:
    """reduce_max(x*m + 1e-15*(1-m), axis=1) of [B,T,D] x (SequenceMaxPooling); the gradient is split equally
    among tied maxima, as TF's is."""
    m = _mask_or_none(mask, x.shape[0], x.shape[1])
    _check_mask_sum(m)
    return _SeqMaxPool.apply(x, m)


class _SeqMeanPool(torch.autograd.Function):
    @staticmethod
    def forward(ctx, x, mask):
        b, t, d = x.shape
        x = _f32(x).contiguous()
        y = torch.empty(b, d, device=x.device, dtype=torch.float32)
        call("nm_seq_mean_pool_fwd", ptr(x), ptr(mask), ptr(y), b, t, d, lib.stream())
        ctx.save_for_backward(mask)
        ctx.shape = (b, t, d)
        return y

    @staticmethod
    def backward(ctx, dy):
        (mask,) = ctx.saved_tensors
        b, t, d = ctx.shape
        dx = torch.empty(b, t, d, device=dy.device, dtype=torch.float32)
        call("nm_seq_mean_pool_bwd", ptr(mask), ptr(dy.contiguous()), ptr(dx), b, t, d, lib.stream())
        return dx, None


def seq_mean_pool(x: torch.Tensor, mask: Optional[torch.Tensor]) -> torch.Tensor:
    """sum_t(x*m) / (sum_t m + 1e-8) of [B,T,D] x (SequenceAveragePooling)."""
    return _SeqMeanPool.apply(x, _mask_or_none(mask, x.shape[0], x.shape[1]))


class _AttentivePool(torch.autograd.Function):
    @staticmethod
    def forward(ctx, energies, mask, states):
        b, t, r = energies.shape
        d = states.shape[2]
        energies, states = _f32(energies).contiguous(), _f32(states).contiguous()
        weights = torch.empty(b, t, r, device=states.device, dtype=torch.float32)
        out = torch.empty(b, r, d, device=states.device, dtype=torch.float32)
        call("nm_attentive_pool_fwd", ptr(energies), ptr(mask), ptr(states), ptr(weights), ptr(out), b, t, r, d,
             lib.stream())
        ctx.save_for_backward(energies, mask, states, weights)
        return weights, out

    @staticmethod
    def backward(ctx, dweights, dout):
        energies, mask, states, weights = ctx.saved_tensors
        b, t, r = energies.shape
        d = states.shape[2]
        if dout is None:
            dout = torch.zeros(b, r, d, device=states.device, dtype=torch.float32)
        de, ds = torch.empty_like(energies), torch.empty_like(states)
        call("nm_attentive_pool_bwd", ptr(energies), ptr(mask), ptr(states), ptr(weights), ptr(dout.contiguous()),
             ptr(None if dweights is None else dweights.contiguous()), ptr(de), ptr(ds), b, t, r, d, lib.stream())
        return de, None, ds


def attentive_pool(energies: torch.Tensor, mask: Optional[torch.Tensor],
                   states: torch.Tensor) -> Tuple[torch.Tensor, torch.Tensor]:
    """The self-attentive pooling of AttentiveEncoder after its dense layers: energies [B,T,R], states [B,T,D] ->
    (weights [B,T,R]: softmax over all T, times the mask, renormalised with +1e-8; weights^T . states [B,R,D])."""
    if energies.dim() != 3 or states.dim() != 3 or energies.shape[:2] != states.shape[:2]:
        raise ValueError("energies [B,T,R] and states [B,T,D] must agree on B and T, got {} and {}".format(
            tuple(energies.shape), tuple(states.shape)))
    return _AttentivePool.apply(energies, _mask_or_none(mask, energies.shape[0], energies.shape[1]), states)


class _Conv1dMaxPool(torch.autograd.Function):
    """y[m] = sum_j x_flat[m+j] . w[j] + bias over the M = B*T-w+1 rows of the flattened batch: one nm_gemm per
    filter tap over a row-shifted view of x (K = E each), accumulated in place (beta = 1).  The windows that cross a
    sentence boundary are computed and never read.  The ReLU is folded into the max over time (max(relu(y)) =
    relu(max(y)), and the ReLU gradient at the tied positions)."""

    @staticmethod
    def forward(ctx, x, w, bias):
        b, t, e = x.shape
        width, _, f = w.shape
        x2 = _f32(x).contiguous().view(b * t, e)
        m = b * t - width + 1
        y = torch.empty(m, f, device=x.device, dtype=torch.float32)
        for j in range(width):
            gemm(x2[j:j + m], w[j], y, bias=bias if j == 0 else None, beta=0.0 if j == 0 else 1.0)
        out = torch.empty(b, f, device=x.device, dtype=torch.float32)
        call("nm_seq_max_pool_fwd", ptr(y), None, ptr(out), b, t - width + 1, t, f, 1, lib.stream())
        ctx.save_for_backward(x2, w, y)
        ctx.shape = (b, t, e, width, f)
        ctx.sinks = (_sink(w), _sink(bias))
        return out

    @staticmethod
    def backward(ctx, dout):
        x2, w, y = ctx.saved_tensors
        b, t, e, width, f = ctx.shape
        m = y.shape[0]
        dy = torch.empty_like(y)
        call("nm_seq_max_pool_bwd", ptr(y), None, ptr(dout.contiguous()), ptr(dy), b, t - width + 1, t, f, m, 1,
             lib.stream())
        w_sink, b_sink = ctx.sinks
        dw = None if w_sink is not None else torch.empty_like(w)
        for j in range(width):
            if w_sink is not None:
                gemm(x2[j:j + m], dy, w_sink[j], trans_a=True, beta=1.0)
            else:
                gemm(x2[j:j + m], dy, dw[j], trans_a=True)
        db = _bias_grad(dy, b_sink)
        dx = torch.zeros(b * t, e, device=y.device, dtype=torch.float32)
        for j in range(width):
            gemm(dy, w[j], dx[j:j + m], trans_b=True, beta=1.0)
        return dx.view(b, t, e), dw, db


def conv1d_max_pool(x: torch.Tensor, w: torch.Tensor, bias: torch.Tensor) -> torch.Tensor:
    """reduce_max(relu(conv1d(x, w, VALID) + bias), axis=1) of the Kim-CNN sentence encoder: x [B,T,E],
    w [width,E,F], bias [F] -> [B,F].  A batch shorter than the filter is refused (TF would reduce over an empty
    axis)."""
    b, t, e = x.shape
    if w.dim() != 3 or w.shape[1] != e or bias.shape != (w.shape[2],):
        raise ValueError("conv1d_max_pool: filter {} and bias {} do not fit inputs of width {}".format(
            tuple(w.shape), tuple(bias.shape), e))
    if t < w.shape[0]:
        raise ValueError("the batch is {} positions long, shorter than the filter width {}: the max over time "
                         "would run over no window".format(t, w.shape[0]))
    return _Conv1dMaxPool.apply(x, w, bias)


class _SquaredError(torch.autograd.Function):
    @staticmethod
    def forward(ctx, pred, target):
        b, dim = pred.shape
        pred, target = _f32(pred).contiguous(), _f32(target).contiguous()
        loss = torch.empty((), device=pred.device, dtype=torch.float32)
        call("nm_squared_error_fwd", ptr(pred), ptr(target), ptr(loss), b, dim, lib.stream())
        ctx.save_for_backward(pred, target)
        return loss

    @staticmethod
    def backward(ctx, dloss):
        pred, target = ctx.saved_tensors
        b, dim = pred.shape
        dpred = torch.empty_like(pred)
        call("nm_squared_error_bwd", ptr(pred), ptr(target), ptr(dloss.contiguous()), ptr(dpred), b, dim,
             lib.stream())
        return dpred, None


def squared_error(pred: torch.Tensor, target: torch.Tensor) -> torch.Tensor:
    """mean((pred [B,dim] - target[:, None])^2), the SequenceRegressor cost."""
    if pred.dim() != 2 or target.shape != (pred.shape[0],):
        raise ValueError("squared_error: predictions [B, dim] and targets [B], got {} and {}".format(
            tuple(pred.shape), tuple(target.shape)))
    return _SquaredError.apply(pred, target)


# ---------------------------------------------------------------------------
# K20 speech features
# ---------------------------------------------------------------------------
SPEECH_KINDS = {"mfcc": 0, "fbank": 1, "logfbank": 2, "ssc": 3}   # NM_SPEECH_* of include/nmb200.h


def speech_frame_count(samples: int, frame_len: int, frame_step: int) -> int:
    """Frames of python_speech_features' framesig: one when the signal fits in a frame, else enough frames at
    `frame_step` to cover it, the last one zero-padded."""
    if samples <= frame_len:
        return 1
    return 1 + -(-(samples - frame_len) // frame_step)


def speech_features(signal: torch.Tensor, window: torch.Tensor, frame_step: int, nfft: int, preemph: float,
                    fbank: torch.Tensor, fb_first: torch.Tensor, fb_last: torch.Tensor, kind: str, rate: float,
                    numcep: int = 13, ceplifter: float = 0.0, append_energy: bool = False, delta_order: int = 0,
                    delta_window: int = 2) -> torch.Tensor:
    """Speech features of one utterance (processors/speech.py): the `kind` features of python_speech_features
    0.6.1 over the fp64 device signal [samples], framed by the fp64 window [frame_len] every `frame_step` samples,
    followed by `delta_order` orders of deltas.  fbank [nfilt, nfft/2+1] fp64 is the filterbank, fb_first /
    fb_last [nfilt] int32 its nonzero bin ranges.  Returns [frames, width * (1 + delta_order)] fp64."""
    for name, t, dtype in (("signal", signal, torch.float64), ("window", window, torch.float64),
                           ("fbank", fbank, torch.float64), ("fb_first", fb_first, torch.int32),
                           ("fb_last", fb_last, torch.int32)):
        if t.dtype != dtype or not t.is_contiguous():
            raise ValueError("speech_features: {} must be a contiguous {} tensor".format(name, dtype))
    nfilt = fbank.shape[0]
    if fbank.dim() != 2 or fbank.shape[1] != nfft // 2 + 1 or fb_first.shape != (nfilt,) or fb_last.shape != (nfilt,):
        raise ValueError("speech_features: filterbank [nfilt, nfft/2+1] and bin ranges [nfilt] expected")
    frame_len = window.numel()
    frames = speech_frame_count(signal.numel(), frame_len, frame_step)
    width = min(numcep, nfilt) if kind == "mfcc" else nfilt
    stride = width * (1 + delta_order)
    out = torch.empty(frames, stride, device=signal.device, dtype=torch.float64)
    call("nm_speech_features", ptr(signal), signal.numel(), ptr(window), frame_len, frame_step, nfft, float(preemph),
         ptr(fbank), ptr(fb_first), ptr(fb_last), nfilt, SPEECH_KINDS[kind], numcep, float(ceplifter),
         int(append_energy), float(rate), ptr(out), frames, stride, lib.stream())
    for block in range(delta_order):
        call("nm_speech_deltas", ptr(out), frames, width, stride, block, delta_window, lib.stream())
    return out
