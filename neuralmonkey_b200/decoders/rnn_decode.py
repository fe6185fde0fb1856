"""Run-time decoding of the RNN attention decoder on the fused step kernel.

A greedy / beam step of `Decoder` (reference: decoders/decoder.py:279-358 inside the while_loop of
decoders/autoregressive.py:442-562, wrapped by decoders/beam_search_decoder.py:394-556) is THREE launches
of libnmb200 and no torch arithmetic:

    nm_attn_decoder_step_fwd   embedding row, GRU cell, query projection, Bahdanau attention, deep output
    nm_decode_logits_step      wgmma vocabulary GEMM with softmax partials  +  combine kernel doing the
                               argmax / `* unfinished` / `finished |= </s>` bookkeeping

(beam search adds the two kernels of nm_beam_step_logits, which reads the logits and their logsumexp
directly; the re-ordering of the recurrent state by the selected beams is an index the step kernel
follows while loading, and the token history is re-built once at the end by nm_beam_backtrack).
All state lives in static buffers owned by this object, so the steps are captured into CUDA graphs in
chunks of `CHUNK` steps and replayed; the host looks at the device-side "hypotheses still unfinished"
counters once per chunk and trims the histories to the step the reference loop would have stopped at.

Used by `Decoder` (greedy) and `BeamSearchDecoder` (RNN parent) when the decoder has the default
structure: GRU cell, no conditional GRU, exactly one feed-forward `Attention`, dense or maxout output.
"""
from typing import Any, Dict, Optional

import torch

from neuralmonkey_b200 import lib, ops, runtime
from neuralmonkey_b200.lib import call, ptr
from neuralmonkey_b200.vocabulary import START_TOKEN_INDEX


def supported(decoder) -> bool:
    """The fused step covers the decoder the five target configs build (SURVEY.md 8(a) a6)."""
    from neuralmonkey_b200.attention.feed_forward import Attention
    from neuralmonkey_b200.decoders.output_projection import _Maxout, _Nonlinear
    if getattr(decoder, "_stepwise", True) or getattr(decoder, "_rnn_cell_str", "") != "GRU":
        return False
    if len(decoder.attentions) != 1 or type(decoder.attentions[0]) is not Attention:
        return False
    if not isinstance(decoder.output_projection, (_Maxout, _Nonlinear)):
        return False
    return runtime.device().type == "cuda"


class _Graphs:
    """CUDA graphs of step chunks, keyed by (kind, chunk index)."""

    def __init__(self) -> None:
        self.graphs = {}   # type: Dict[Any, torch.cuda.CUDAGraph]

    def run(self, key, fn) -> None:
        graph = self.graphs.get(key)
        if graph is None:
            graph = torch.cuda.CUDAGraph()
            with torch.cuda.graph(graph, capture_error_mode="thread_local"):
                fn()
            self.graphs[key] = graph
        graph.replay()


class RNNDecodeEngine:
    CHUNK = 16           # steps per captured graph / per look at the "unfinished" counters
    GRAPH_AFTER = 2      # a shape is captured the second time it is decoded; one-offs run eagerly

    def __init__(self, decoder) -> None:
        self.dec = decoder
        self.att = decoder.attentions[0]
        self.bufs = {}     # type: Dict[Any, Dict[str, torch.Tensor]]
        self.graphs = {}   # type: Dict[Any, _Graphs]
        self.seen = {}     # type: Dict[Any, int]
        self.use_cuda_graph = True

    # -- parameters (views into the arena: stable addresses) ------------------------------------
    def _weights(self) -> Dict[str, Any]:
        from neuralmonkey_b200.decoders.output_projection import _Maxout
        from neuralmonkey_b200.encoders.recurrent import gru_cell_tensors
        dec, att = self.dec, self.att
        wg, bg, wc, bc = gru_cell_tensors(dec, dec._CELL_SCOPE)
        proj = dec.output_projection
        if isinstance(proj, _Maxout):
            pre = "attention_decoder/MaxoutProjection/MaxoutProjection/"
            wo, bo, act, maxout = dec.var(pre + "kernel"), dec.var(pre + "bias"), 0, 1
        else:
            wo, bo = dec.var("attention_decoder/dense/kernel"), dec.var("attention_decoder/dense/bias")
            act, maxout = lib.NM_ACT[proj.activation], 0
        return dict(wg=wg, bg=bg, wc=wc, bc=bc, wq=att.var("Attention/attn_query_projection"),
                    bq=att.var("attn_projection_bias"), v=att.var("attn_similarity_v"),
                    ab=att.var("attn_bias"), wo=wo, bo=bo, act=act, maxout=maxout,
                    table=dec.embedding_matrix, w=dec.decoding_w, b=dec.decoding_b)

    def _dims(self) -> Dict[str, int]:
        dec, att = self.dec, self.att
        return dict(E=dec.embedding_size, H=dec.rnn_size, A=att.state_size, C=att.context_vector_size,
                    O=dec.output_dimension, V=len(dec.vocabulary))

    # -- static buffers ------------------------------------------------------------------------------
    def _buffers(self, key, rows: int, nb: int, tx: int, steps: int, beam: int) -> Dict[str, torch.Tensor]:
        if key in self.bufs:
            return self.bufs[key]
        while len(self.bufs) >= 4:                      # bounded: every entry holds its histories
            old = next(iter(self.bufs))
            self.bufs.pop(old)
            self.graphs.pop(old, None)
        d, dev = self._dims(), runtime.device()
        f32, i64, i32, u8 = torch.float32, torch.int64, torch.int32, torch.uint8

        def z(shape, dtype=f32):
            return torch.zeros(shape, device=dev, dtype=dtype)

        b = dict(keys=z((nb, tx, d["A"])), values=z((nb, tx, d["C"])), mask=z((nb, tx)),
                 h0=z((rows, d["H"])), start=torch.full((rows,), START_TOKEN_INDEX, device=dev, dtype=i64),
                 counts=z((steps + 1,), i32),
                 part=z((lib.load().nm_logits_xent_scratch(rows, d["V"]),)))
        if beam:
            b.update(h=z((2, rows, d["H"])), out=z((rows, d["O"])), logits=z((rows, d["V"])), lse=z((rows,)),
                     first=z((rows,), i64), words=z((steps, rows), i64), parents=z((steps, rows), i32),
                     lsum=z((2, rows)), lens=z((2, rows), i32), fin=z((2, rows), u8), scores=z((rows,)),
                     scratch=z((lib.load().nm_beam_scratch(nb, beam, d["V"]),), i32),
                     tokens=z((steps + 1, rows), i64))
        else:
            b.update(h=z((steps, rows, d["H"])), out=z((steps, rows, d["O"])), ctx=z((steps, rows, d["C"])),
                     att_w=z((steps, rows, tx)), lse=z((steps, rows)), argmax=z((steps, rows), i64),
                     symbols=z((steps, rows), i64), maskh=z((steps, rows), u8), fin=z((rows,), u8),
                     xent=z((steps, rows)), gold=z((steps, rows), i64), goldw=z((steps, rows)),
                     logits1=None)
        self.bufs[key] = b
        self.graphs[key] = _Graphs()
        return b

    def _load_encoder(self, b: Dict[str, torch.Tensor], rows_per_sentence: int) -> None:
        dec, att = self.dec, self.att
        b["keys"].copy_(att.hidden_features)
        b["values"].copy_(att.attention_states)
        mask = att.attention_mask
        if mask is None:
            b["mask"].fill_(1.0)
        else:
            b["mask"].copy_(mask)
        self._has_mask = mask is not None
        h0 = dec.initial_state
        b["h0"].copy_(h0 if rows_per_sentence == 1 else h0.repeat_interleave(rows_per_sentence, 0))

    def _step_kernel(self, w, d, b, symbols, h_prev, parent, h_out, ctx_out, w_out, out, rows, group, tx):
        call("nm_attn_decoder_step_fwd", ptr(symbols), ptr(w["table"]), None, ptr(h_prev), ptr(parent),
             ptr(w["wg"]), ptr(w["bg"]), ptr(w["wc"]), ptr(w["bc"]), ptr(w["wq"]), ptr(w["bq"]), ptr(w["v"]),
             ptr(w["ab"]), ptr(b["keys"]), ptr(b["values"]), ptr(b["mask"]) if self._has_mask else None,
             ptr(w["wo"]), ptr(w["bo"]), None, ptr(h_out), ptr(ctx_out), ptr(w_out), ptr(out),
             rows, group, d["E"], d["H"], d["A"], d["C"], tx, d["O"], w["act"], w["maxout"], lib.stream())

    def _logits_kernel(self, w, d, x, rows, fin_in=None, targets=None, weights=None, lse=None, argmax=None,
                       xent=None, sym_out=None, fin_out=None, mask_out=None, count=None, part=None,
                       logits=None) -> None:
        dec = self.dec
        trans = int(dec._w_transposed)
        wmat = w["w"]
        call("nm_decode_logits_step", ptr(x), x.stride(0), ptr(wmat), wmat.stride(0), trans, ptr(w["b"]),
             dec._unk_index, ptr(fin_in), ptr(targets), ptr(weights), ptr(lse), ptr(argmax), ptr(xent),
             ptr(sym_out), ptr(fin_out), ptr(mask_out), ptr(count), ptr(part), ptr(logits), d["V"], rows,
             d["V"], d["O"], ops.gemm_backend(), lib.stream())

    def _tc_logits(self, rows: int, d: Dict[str, int]) -> bool:
        """Whether the vocabulary projection of a step runs on the tensor cores (else: exact fp32 CUDA
        cores into a materialised [rows, V] buffer)."""
        dec = self.dec
        wmat = dec.decoding_w
        return (ops.gemm_backend() != lib.GEMM_SIMT and
                lib.load().nm_gemm_uses_tc(0, int(dec._w_transposed), rows, d["V"], d["O"], d["O"],
                                           wmat.stride(0), d["V"]) == 1 and wmat.data_ptr() % 16 == 0)

    def _run_chunks(self, key, kind: str, steps: int, first_step: int, step_fn, counts: torch.Tensor) -> int:
        """Issue steps first_step..steps-1 in chunks; returns how many steps the reference loop runs:
        it stops after the first step that leaves no hypothesis unfinished."""
        self.seen[key] = self.seen.get(key, 0) + 1
        graphs = self.graphs[key] if (self.use_cuda_graph and self.seen[key] >= self.GRAPH_AFTER) else None
        t = first_step
        while t < steps:
            end = min(steps, t + self.CHUNK)

            def chunk(t0=t, t1=end):
                for s in range(t0, t1):
                    step_fn(s)
            if graphs is not None:
                graphs.run((kind, t, end), chunk)
            else:
                chunk()
            # one small device->host copy per chunk (pinned staging, no torch arithmetic on the device)
            host = self._counts_host(counts.numel())
            host[t:end].copy_(counts[t:end], non_blocking=True)
            torch.cuda.current_stream().synchronize()
            for s in range(t, end):
                if int(host[s]) == 0:
                    return s + 1
            t = end
        return steps

    def _counts_host(self, n: int) -> torch.Tensor:
        buf = self.__dict__.get("_counts_pinned")
        if buf is None or buf.numel() < n:
            buf = torch.zeros(max(n, 256), dtype=torch.int32).pin_memory()
            self.__dict__["_counts_pinned"] = buf
        return buf

    # -- greedy decoding ------------------------------------------------------------------------------
    @torch.no_grad()
    def greedy(self, max_steps: int, gold: Optional[torch.Tensor] = None,
               gold_mask: Optional[torch.Tensor] = None) -> Dict[str, torch.Tensor]:
        """decoding_loop(train_mode=False) (autoregressive.py:532-562).  gold / gold_mask ([time, batch],
        optional): the references, for the runtime cross-entropies.  Histories are time-major."""
        dec = self.dec
        rows, d = dec.batch_size, self._dims()
        tx = self.att.hidden_features.shape[1]
        key = ("greedy", rows, tx, max_steps)
        b = self._buffers(key, rows, rows, tx, max_steps, 0)
        w = self._weights()
        self._load_encoder(b, 1)
        b["fin"].zero_()
        b["counts"].zero_()
        gsteps = 0
        if gold is not None:
            gsteps = min(int(gold.shape[0]), max_steps)
            b["gold"][:gsteps].copy_(gold[:gsteps])
            b["goldw"][:gsteps].copy_(gold_mask[:gsteps].to(torch.float32))
        use_tc = self._tc_logits(rows, d)
        if not use_tc and b["logits1"] is None:
            b["logits1"] = torch.zeros(rows, d["V"], device=runtime.device())

        def step(t: int) -> None:
            self._step_kernel(w, d, b, b["start"] if t == 0 else b["symbols"][t - 1],
                              b["h0"] if t == 0 else b["h"][t - 1], None, b["h"][t], b["ctx"][t],
                              b["att_w"][t], b["out"][t], rows, 1, tx)
            has_gold = t < gsteps
            self._logits_kernel(w, d, b["out"][t], rows, fin_in=b["fin"],
                                targets=b["gold"][t] if has_gold else None,
                                weights=b["goldw"][t] if has_gold else None, lse=b["lse"][t],
                                argmax=b["argmax"][t], xent=b["xent"][t] if has_gold else None,
                                sym_out=b["symbols"][t], fin_out=b["fin"], mask_out=b["maskh"][t],
                                count=b["counts"][t:t + 1], part=b["part"],
                                logits=None if use_tc else b["logits1"])

        kind = ("g", gsteps, use_tc, self._has_mask)
        n = self._run_chunks(key, kind, max_steps, 0, step, b["counts"])
        return dict(steps=n, symbols=b["symbols"][:n].clone(), argmax=b["argmax"][:n].clone(),
                    mask=b["maskh"][:n].to(torch.bool), lse=b["lse"][:n].clone(),
                    output_states=b["out"][:n].clone(), rnn_outputs=b["h"][:n].clone(),
                    contexts=b["ctx"][:n].clone(), weights=b["att_w"][:n].clone(),
                    xent=b["xent"][:min(n, gsteps)].clone() if gsteps else None,
                    finished=b["fin"].to(torch.bool))

    # -- beam search -------------------------------------------------------------------------------------
    @torch.no_grad()
    def beam(self, beam_size: int, max_steps: int, alpha: float) -> Dict[str, Any]:
        """BeamSearchDecoder.outputs (beam_search_decoder.py:167-191, 218-556) around this decoder."""
        dec = self.dec
        nb, k, d = dec.batch_size, beam_size, self._dims()
        rows = nb * k
        tx = self.att.hidden_features.shape[1]
        key = ("beam", nb, k, tx, max_steps)
        b = self._buffers(key, rows, nb, tx, max_steps, k)
        w = self._weights()
        self._load_encoder(b, k)
        use_tc = self._tc_logits(rows, d)
        b["counts"].zero_()
        b["counts"][0] = 1                    # slot 0 is the initial decoder step, not a search step
        b["fin"].zero_()
        b["lens"].zero_()
        b["lsum"][0].fill_(-1e9)              # logprob_sum = [0, -INF, ...] (beam_search_decoder.py:283-295)
        b["lsum"][0].view(nb, k)[:, 0] = 0.0
        b["scores"].zero_()
        # the initial step (get_initial_loop_state :218-328): every hypothesis of a sentence is the same row
        self._step_kernel(w, d, b, b["start"], b["h0"], None, b["h"][0], None, None, b["out"], rows, k, tx)
        self._logits_kernel(w, d, b["out"], rows, lse=b["lse"], argmax=b["first"], part=b["part"],
                            logits=b["logits"])

        def step(t: int) -> None:               # search step t = 1 .. max_steps
            p, q = (t - 1) & 1, t & 1
            call("nm_beam_step_logits", ptr(b["logits"]), ptr(b["lse"]), ptr(b["lsum"][p]), ptr(b["lens"][p]),
                 ptr(b["fin"][p]), float(alpha), ptr(b["scores"]), ptr(b["words"][t - 1]),
                 ptr(b["parents"][t - 1]), ptr(b["lsum"][q]), ptr(b["lens"][q]), ptr(b["fin"][q]),
                 ptr(b["counts"][t:t + 1]), ptr(b["scratch"]), nb, k, d["V"], lib.stream())
            self._step_kernel(w, d, b, b["words"][t - 1], b["h"][p], b["parents"][t - 1], b["h"][q], None, None,
                              b["out"], rows, k, tx)
            self._logits_kernel(w, d, b["out"], rows, lse=b["lse"], part=b["part"], logits=b["logits"])

        kind = ("b", use_tc, self._has_mask)
        last = self._run_chunks(key, kind, max_steps + 1, 1, step, b["counts"]) - 1   # search steps the loop ran
        call("nm_beam_backtrack", ptr(b["first"]), ptr(b["words"]), ptr(b["parents"]), ptr(b["tokens"]), nb, k,
             last, lib.stream())
        q = last & 1
        # steps issued past the stopping step are idempotent on (scores, logprob_sum, lengths, finished):
        # finished hypotheses only extend with <pad> at log-probability 0 (beam_search_decoder.py:440-456)
        return dict(steps=last, scores=b["scores"].view(nb, k).clone(),
                    token_ids=b["tokens"][:last + 1].view(last + 1, nb, k).clone(),
                    logprob_sum=b["lsum"][q].view(nb, k).clone(), lengths=b["lens"][q].view(nb, k).clone(),
                    finished=b["fin"][q].view(nb, k).to(torch.bool), logits=b["logits"].view(nb, k, -1),
                    lse=b["lse"].view(nb, k))
