"""CPU stand-ins for `neuralmonkey_b200.ops` - TEST INFRASTRUCTURE ONLY.

The product has no CPU execution path (ops call the CUDA library and fail loudly without it).  To check
the HOST side of the model parts without a GPU - which tensors they feed to which operation, variable
names, teacher forcing, loop bookkeeping, the step-wise variants - the `cpu_model` fixture of
tests/test_host_model_cpu.py swaps every `ops.<name>` the model parts call for the function of the same
name and signature below, written with the oracle's arithmetic, and points `runtime.device()` at the CPU.
Nothing outside tests/ imports this module; the kernels themselves are tested in tests/test_gpu_*.py."""
import math
from typing import Optional

import torch

from oracle import nm_oracle as O

_ACT = {None: lambda x: x, "tanh": torch.tanh, "relu": torch.relu, "sigmoid": torch.sigmoid}


def linear(x, w, b=None, act=None):
    y = x @ w
    if b is not None:
        y = y + b
    return _ACT[act](y)


def embed(ids, table, mask=None):
    out = table[ids]
    return out if mask is None else out * mask.unsqueeze(-1)


def maxout(z):
    size = z.shape[-1] // 2
    return torch.maximum(z[..., :size], z[..., size:])


def layer_norm(x, gamma, beta, eps=1e-6):
    return O.layer_norm(x, gamma, beta, eps)


def gru_layer(x, gates_kernel, gates_bias, cand_kernel, cand_bias, h0=None, lengths=None, reverse=False,
              drop_mask=None, sm_budget=0):
    full = torch.full((x.shape[0],), x.shape[1], dtype=torch.int64)
    lens = full if lengths is None else lengths.to(torch.int64)
    inputs = O.reverse_sequence(x, lens) if reverse else x
    if drop_mask is None:
        raw, final = O.dynamic_gru(inputs, None if lengths is None else lens, gates_kernel, gates_bias,
                                   cand_kernel, cand_bias, h0)
        if reverse:
            raw = O.reverse_sequence(raw, lens)
        return raw, final, raw
    # with a dropout mask the state handed to the next step is the DROPPED output (the reference's decoder
    # feeds `prev_rnn_output = dropout(cell_output)` back: decoders/decoder.py:330-349), as in nm_gru_seq_fwd
    assert not reverse and lengths is None
    h = h0 if h0 is not None else x.new_zeros(x.shape[0], cand_kernel.shape[1])
    raws, dropped = [], []
    for t in range(x.shape[1]):
        new = O.gru_cell(x[:, t], h, gates_kernel, gates_bias, cand_kernel, cand_bias)
        h = new * drop_mask[:, t]
        raws.append(new)
        dropped.append(h)
    return torch.stack(dropped, 1), h, torch.stack(raws, 1)


def bahdanau_attention(keys, values, mask, qproj, v, bias):
    energies = (v * torch.tanh(keys.unsqueeze(1) + qproj.unsqueeze(2))).sum(-1) + bias
    weights = torch.softmax(energies, dim=-1)
    if mask is not None:
        weights = weights * mask.unsqueeze(1)
        weights = weights / (weights.sum(-1, keepdim=True) + 1e-8)
    return torch.einsum("bqt,btc->bqc", weights, values), weights


def logits_xent(x, w, b, targets, weights, unk_index=-1, trans_w=False, keep_logits=False):
    logits = x @ (w.t() if trans_w else w)
    if b is not None:
        logits = logits + b
    if unk_index >= 0:
        pen = torch.zeros(logits.shape[-1], dtype=logits.dtype)
        pen[unk_index] = -1e9
        logits = logits + pen
    lse = torch.logsumexp(logits, dim=-1)
    xent = (lse - logits.gather(1, targets.unsqueeze(1)).squeeze(1)) * weights
    return xent, lse, torch.argmax(logits, dim=-1), (logits if keep_logits else None)


def log_softmax_from_lse(logits, lse):
    return logits - lse.unsqueeze(-1)


def mha_core(q, k, v, key_mask, causal, heads, drop_mask=None):
    bsz, tq, dim = q.shape
    tk, dh = k.shape[1], dim // heads

    def split(x):
        return x.reshape(bsz, x.shape[1], heads, dh).transpose(1, 2)
    energies = split(q) @ split(k).transpose(-1, -2) / math.sqrt(dh)
    if causal:      # mask_future: tf.where(lower triangle, e, -1e9)
        tri = torch.tril(torch.ones(tq, tk, dtype=torch.bool))
        energies = torch.where(tri, energies, torch.full_like(energies, -1e9))
    if key_mask is not None:
        m = key_mask.unsqueeze(1).unsqueeze(1)
        energies = energies * m + (1.0 - m) * -1e9
    weights = torch.softmax(energies, dim=-1)
    applied = weights if drop_mask is None else weights * drop_mask
    return (applied @ split(v)).transpose(1, 2).reshape(bsz, tq, dim), weights


def beam_step(logprobs, logprob_sum, lengths, finished, alpha):
    scores, words, beams, lsum, lens, fin = O.beam_step(logprobs, logprob_sum, lengths.to(torch.int32),
                                                        finished.to(torch.bool), alpha)
    return scores, words, beams, lsum, lens, fin.to(torch.uint8)


def beam_gather(x, beam_ids, bsz, k):
    flat = (torch.arange(bsz).unsqueeze(1) * k + beam_ids.to(torch.int64)).reshape(-1)
    return x[flat]


def conv3x3_bias_relu(x, w, b):
    y = torch.nn.functional.conv2d(x.permute(0, 3, 1, 2), w.permute(3, 2, 0, 1), b, padding=1)   # NHWC x HWIO
    return torch.relu(y).permute(0, 2, 3, 1).contiguous()


def maxpool2x2(x):
    return torch.nn.functional.max_pool2d(x.permute(0, 3, 1, 2), 2, 2).permute(0, 2, 3, 1).contiguous()


def xent_rows(logits, targets=None, weights=None, want_argmax=False, first_col=0):
    part = logits[:, first_col:]
    lse = torch.logsumexp(part, dim=-1)
    xent = None
    if targets is not None:
        xent = (lse - part.gather(1, targets.unsqueeze(1)).squeeze(1)) * weights
    return lse, xent, (torch.argmax(part, dim=-1) if want_argmax else None)


def adam_kernel(trainer, grad_scale, denominator, lr_t, lr_t_dev):
    """Stand-in for GenericTrainer._adam_kernel (`nm_clip_adam_step`) over the arena's gradient buffer
    (the stand-in ops leave their gradients in `.grad`; the trainer folds those in).  Same order as the
    kernel: scale, add the L1 / L2 terms of the regularised variables, clip per tensor, TF-Adam."""
    from neuralmonkey_b200 import runtime
    arena, opt = runtime.arena(), trainer.optimizer
    scale = float(grad_scale) / (float(denominator) if denominator is not None else 1.0)
    if not hasattr(trainer, "_l1l2_buf"):
        trainer._l1l2_buf = torch.zeros(2)
    adam_m, adam_v = arena.optimizer_slot(opt)
    l1 = l2 = 0.0
    with torch.no_grad():
        for name in trainer.var_list:                 # with var_scopes: only the variables in scope
            var = arena.get(name)
            grad = arena.grad(name) * scale           # the trainer folded the autograd gradients in
            if O.is_regularizable(name):
                l1 += float(var.abs().sum())
                l2 += float((var ** 2).sum())
                grad = grad + trainer.l1_weight * torch.sign(var) + 2.0 * trainer.l2_weight * var
            if trainer.clip_norm:
                grad = O.clip_by_norm(grad, float(trainer.clip_norm))
            info = arena.variables[name]
            m = adam_m[info.offset:info.offset + var.numel()].view(var.shape)
            v = adam_v[info.offset:info.offset + var.numel()].view(var.shape)
            m.mul_(opt.beta1).add_(grad, alpha=1 - opt.beta1)
            v.mul_(opt.beta2).addcmul_(grad, grad, value=1 - opt.beta2)
            var.sub_((float(lr_t_dev) if lr_t_dev is not None else lr_t) * m / (v.sqrt() + opt.epsilon))
    trainer._l1l2_buf[0], trainer._l1l2_buf[1] = l1, l2


def nematus_gru_gate(state_gates, input_gates, state_cand, input_cand, state):
    gates = torch.sigmoid(state_gates + input_gates)
    size = state.shape[1]
    reset, update = gates[:, :size], gates[:, size:]
    cand = torch.tanh(state_cand * reset + input_cand)
    return update * state + (1.0 - update) * cand


def lstm_gate(z, c):
    i, j, f, o = z.chunk(4, dim=1)
    new_c = torch.sigmoid(f + 1.0) * c + torch.sigmoid(i) * torch.tanh(j)
    return new_c, torch.sigmoid(o) * torch.tanh(new_c)


def gru_bilayer(x, lengths, cell_fw, cell_bw):
    out_fw, fin_fw, _ = gru_layer(x, *cell_fw, lengths=lengths, reverse=False)
    out_bw, fin_bw, _ = gru_layer(x, *cell_bw, lengths=lengths, reverse=True)
    return out_fw, fin_fw, out_bw, fin_bw


STAND_INS = ("gru_bilayer", "nematus_gru_gate", "lstm_gate", "xent_rows", "conv3x3_bias_relu", "maxpool2x2", "linear", "embed", "maxout", "layer_norm", "gru_layer", "bahdanau_attention", "logits_xent",
             "log_softmax_from_lse", "mha_core", "beam_step", "beam_gather")
