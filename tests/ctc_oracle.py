"""fp64 torch restatement of the CTC operations of decoders/ctc_decoder.py - TEST INFRASTRUCTURE ONLY.

TF 1.12's ctc_loss (ctc_loss_calculator: the forward variables of the extended label, `ctc_merge_repeated`,
`ignore_longer_outputs_than_inputs=True`) and ctc_greedy_decoder (first index of the row maximum, blank dropped,
repeats merged), written independently of the kernels: the loss is the forward recursion alone and its gradient
comes from autograd, not from the alpha-beta occupancy formula the kernel uses."""
from typing import List, Tuple

import torch

END = 2


def _required_frames(labels: List[int], merge: bool) -> int:
    return len(labels) + (sum(1 for a, b in zip(labels, labels[1:]) if a == b) if merge else 0)


def _sentence_logp(logp: torch.Tensor, labels: List[int], merge: bool) -> torch.Tensor:
    """log p(labels | frames) for one sentence's log-probabilities [f, C] (blank = C-1)."""
    blank = logp.shape[1] - 1
    ext = [blank]
    for lab in labels:
        ext += [lab, blank]
    n = len(ext)
    idx = torch.tensor(ext, dtype=torch.int64)
    self_ok = torch.tensor([merge or c == blank for c in ext])
    skip_ok = torch.tensor([s >= 2 and ext[s] != blank and not (merge and ext[s] == ext[s - 2]) for s in range(n)])
    # "log 0" is a large finite negative: a logsumexp over nothing but -inf has a NaN gradient
    neg = torch.tensor(-1e30, dtype=logp.dtype)
    alpha = torch.full((n,), -1e30, dtype=logp.dtype)
    alpha = torch.where(torch.arange(n) <= 1, logp[0, idx], alpha)
    for t in range(1, logp.shape[0]):
        stay = torch.where(self_ok, alpha, neg)
        step = torch.cat([neg.reshape(1), alpha[:-1]])
        skip = torch.where(skip_ok, torch.cat([neg.expand(2), alpha[:-2]])[:n], neg)
        alpha = torch.logsumexp(torch.stack([stay, step, skip]), dim=0) + logp[t, idx]
    return torch.logsumexp(alpha[-2:], dim=0) if n > 1 else alpha[0]


def ctc_loss(logits: torch.Tensor, frames, labels, label_lengths, merge: bool) -> torch.Tensor:
    """Per-sentence -log p of batch-major logits [B, T, C]; 0 where no alignment fits in the frames (or there
    are none).  Differentiable in `logits`."""
    logits = logits.to(torch.float64)
    out = []
    for b in range(logits.shape[0]):
        f = max(0, min(int(frames[b]), logits.shape[1]))
        lab = [int(x) for x in labels[b][:int(label_lengths[b])]]
        if f == 0 or _required_frames(lab, merge) > f:
            out.append(torch.zeros((), dtype=torch.float64))
            continue
        logp = torch.log_softmax(logits[b, :f], dim=-1)
        out.append(-_sentence_logp(logp, lab, merge))
    return torch.stack(out)


def ctc_greedy_decode(logits: torch.Tensor, frames, merge: bool) -> Tuple[torch.Tensor, torch.Tensor]:
    """(ids [B, T] int64 padded with </s>, lengths [B] int32) as the greedy kernel writes them."""
    bsz, t_max, c = logits.shape
    blank = c - 1
    ids = torch.full((bsz, t_max), END, dtype=torch.int64)
    lengths = torch.zeros(bsz, dtype=torch.int32)
    best = torch.argmax(logits, dim=-1)          # first maximal index, as TF's RowMax
    for b in range(bsz):
        f = max(0, min(int(frames[b]), t_max))
        prev, seq = -1, []
        for t in range(f):
            k = int(best[b, t])
            if k != blank and not (merge and k == prev):
                seq.append(k)
            prev = k
        ids[b, :len(seq)] = torch.tensor(seq, dtype=torch.int64)
        lengths[b] = len(seq)
    return ids, lengths


def ctc_decoder(params, name: str, states: torch.Tensor, frames, labels, label_lengths, merge_outputs: bool):
    """The CTCDecoder head over encoder states [B, T, D]: the projection (ctc_decoder.py:121-150), the summed
    loss (:96-104) and the time-major greedy decoding padded with </s> (:73-88)."""
    logits = states.to(torch.float64) @ params[name + "/state_to_word_W"] + params[name + "/state_to_word_b"]
    losses = ctc_loss(logits, frames, labels, label_lengths, merge_outputs)
    ids, lengths = ctc_greedy_decode(logits.detach(), frames, merge_outputs)
    longest = int(lengths.max()) if lengths.numel() else 0
    return {"logits": logits, "losses": losses, "cost": losses.sum(), "decoded": ids[:, :longest].t()}
