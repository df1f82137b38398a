"""Mistral-7B / Qwen2 decoder prefill (+ greedy or sampled decode) on libvl2 kernels.

Arithmetic of HF MistralModel / Qwen2Model (HF:mistral/modeling_mistral.py:35-48,51-82,122-239,262-470;
HF:qwen2/modeling_qwen2.py:187-246): RMSNorm -> fused QKV GEMM (+bias for Qwen2) -> RoPE -> causal GQA flash attention
-> o_proj(+residual) -> RMSNorm -> gate/up GEMM with SwiGLU epilogue -> down_proj(+residual) -> norm -> lm_head.
Weights are repacked once: q/k/v concatenated, gate/up rows interleaved so SwiGLU happens inside the GEMM tile, and the
RMSNorm gains multiplied into the weight columns: the per-layer norms cost no kernel (row statistics are produced by
the residual GEMM epilogues, the 1/rms factor is applied in the consuming GEMM's epilogue)."""
from __future__ import annotations

import os
from typing import Dict, List, Optional

import torch

from .. import _lib, ops


class DecoderEngine:
    def __init__(self, config):
        self.config = config
        self.H = config.hidden_size
        self.Hq = config.num_attention_heads
        self.Hkv = config.num_key_value_heads
        self.D = config.hidden_size // config.num_attention_heads
        self.I = config.intermediate_size
        self.eps = config.rms_norm_eps
        self.dtype = getattr(config, "storage_dtype", torch.bfloat16)      # bf16 or fp16 (selects the library build)
        self.layers: List[Dict[str, torch.Tensor]] = []
        self.w: Dict[str, torch.Tensor] = {}
        self.is_loaded = False
        self.kv: List[torch.Tensor] = []   # per layer [S_max, (Hq+2Hkv)*D] fused qkv rows (K,V columns = cache)
        self.kv_len = 0
        self._graphed = None
        self._decode_graph = None   # (graph, tok_dev, pos_dev, logits, stage) of the captured greedy single-token step
        self._decode_graph_sampled = None   # the same step ending in vl2_sample_token instead of the arg-max
        # the greedy and sampled steps with vl2_process_logits in front of the token choice (captured on first use only)
        self._decode_graph_processed = self._decode_graph_sampled_processed = None
        # the four steps above, also recording their rows for generate(output_scores / output_logits), keyed by
        # (sampled, processed) and captured on first use only
        self._decode_graphs_recorded: Dict[tuple, tuple] = {}
        self._decode_bufs = None    # (tok_dev, pos_dev, stage, gen_buf, step_dev): device state the graphs share
        self._decode_log = None     # (device id buffer, device step counter) the graphs append their tokens to
        self._decode_hist = None    # new token 0 followed by the id log (gen_buf is its view from index 1)
        self._sample_params = None  # device vl2_sample_params the sampled graph reads (values copied in when armed)
        self._process_params = None  # device vl2_logits_process_params block the processed graphs read (copied when armed)
        self._process_tables = None  # the ops.logits_process_params tensor whose tables the armed block points into
        self._record_params = None  # device vl2_score_record_params block the recording graphs read (copied when armed)
        self._armed = None          # the graph decode_graph_begin armed last
        self._decode_read = 0
        self.graph_decode = False
        self.decode_pdl = os.environ.get("VL2_DECODE_PDL", "0") == "1"   # PDL edges inside the decode graph
        # MB of o_proj + gate/up weights pulled into L2 on a forked graph branch while the attention phase runs
        # (HBM is idle there); 0 disables the fork
        self.decode_prefetch_mb = float(os.environ.get("VL2_DECODE_PREFETCH_MB", "0"))
        self._side_stream = None

    def enable_cuda_graphs(self, on: bool = True):
        """Graph the cache-less last-position prefill (the bench / first-token path)."""
        from ..graphs import GraphedStage
        self._graphed = GraphedStage(lambda e: self._prefill_last(e)) if on else None
        self.graph_decode = on
        self._drop_decode_graphs()
        return self

    def _drop_decode_graphs(self) -> None:
        """Forget the captured decode steps: they hold the addresses of the KV cache they were captured on."""
        self._decode_graph = self._decode_graph_sampled = self._decode_bufs = self._armed = None
        self._decode_graph_processed = self._decode_graph_sampled_processed = None
        self._decode_graphs_recorded = {}

    def _prefill_last(self, embeds: torch.Tensor) -> torch.Tensor:
        return self.prefill(embeds, all_logits=False, keep_cache=False, _no_graph=True)[0]

    def load_state_dict(self, sd: Dict[str, torch.Tensor], device) -> "DecoderEngine":
        dev = torch.device(device)
        bf = lambda t: t.to(device=dev, dtype=self.dtype).contiguous()
        f32 = lambda t: t.to(device=dev, dtype=torch.float32).contiguous()
        self.layers = []
        # RoPE runs in the epilogue of the fused QKV GEMM on ADJACENT column pairs: permute the q / k weight rows (and
        # biases) so that the partners (i, i + D/2) of a head come out as columns (2i, 2i+1).  q.k is invariant under the
        # permutation (same one for q and k), v is untouched, so attention and the KV cache consume the rows as they are.
        nqk = (self.Hq + self.Hkv) * self.D
        qk_perm = torch.cat([ops.rope_interleave_rows(self.Hq + self.Hkv, self.D),
                             torch.arange(nqk, nqk + self.Hkv * self.D)]).to(dev)
        for i in range(self.config.num_hidden_layers):
            p = f"model.layers.{i}."
            names = ("q_proj", "k_proj", "v_proj")
            # RMSNorm gains are folded into the columns of the weight that consumes the normalised activations:
            # rmsnorm(x; g) W^T = rstd(x) * (x (W * g)^T); rstd is applied per row in the GEMM epilogue.
            g1 = sd[p + "input_layernorm.weight"].to(device=dev, dtype=torch.float32)
            g2 = sd[p + "post_attention_layernorm.weight"].to(device=dev, dtype=torch.float32)
            wqkv = torch.cat([sd[p + f"self_attn.{n}.weight"] for n in names], 0).to(device=dev, dtype=torch.float32)
            wqkv = wqkv[qk_perm]          # RoPE partners of every q / k head become adjacent output columns
            wgu = torch.stack([sd[p + "mlp.gate_proj.weight"], sd[p + "mlp.up_proj.weight"]], 1).reshape(
                2 * self.I, self.H).to(device=dev, dtype=torch.float32)
            L = {
                "wqkv": (wqkv * g1[None, :]).to(self.dtype).contiguous(),
                "wo": bf(sd[p + "self_attn.o_proj.weight"]),
                "wgu": (wgu * g2[None, :]).to(self.dtype).contiguous(),
                "wd": bf(sd[p + "mlp.down_proj.weight"]),
            }
            del wqkv, wgu
            if p + "self_attn.q_proj.bias" in sd:
                L["bqkv"] = f32(torch.cat([sd[p + f"self_attn.{n}.bias"] for n in names], 0).to(dev)[qk_perm])
            self.layers.append(L)
        self.w = {"embed": bf(sd["model.embed_tokens.weight"]), "norm": bf(sd["model.norm.weight"]),
                  # final-norm gain folded into the lm_head columns (the GEMV / GEMM epilogue applies 1/rms itself)
                  "lm_head": (sd["lm_head.weight"].to(device=dev, dtype=torch.float32)
                                * sd["model.norm.weight"].to(device=dev, dtype=torch.float32)[None, :]
                                ).to(self.dtype).contiguous(),
                  "ones": torch.ones((self.H,), device=dev, dtype=self.dtype)}
        inv = 1.0 / (self.config.rope_theta ** (torch.arange(0, self.D, 2, dtype=torch.int64).float() / self.D))
        self.w["inv_freq"] = inv.to(dev)
        # one table for every position the model can see (8 MB at 32768 x 64): captured graphs keep its address
        self._rope_tab = ops.rope_table(int(getattr(self.config, "max_position_embeddings", 32768) or 32768), self.D,
                                        self.config.rope_theta, dev, self.dtype)
        self.device = dev
        self.is_loaded = True
        return self

    @property
    def embed_tokens(self) -> torch.Tensor:
        return self.w["embed"]

    def rope_table(self, n_pos: int) -> torch.Tensor:
        """Packed bf16 (cos, sin) of every (position, frequency), built once at load."""
        if self._rope_tab.shape[0] < n_pos:
            raise ValueError(f"sequence of {n_pos} positions exceeds max_position_embeddings ({self._rope_tab.shape[0]})")
        return self._rope_tab

    # ---- prefill ---------------------------------------------------------------------------------------------
    def _layer(self, L, x: torch.Tensor, S: int, pos0: int, qkv_out: Optional[torch.Tensor], ss_x: torch.Tensor):
        """One decoder layer.  ss_x [S, parts]: partial sums of squares of the incoming residual stream's rows.
        Returns (outgoing stream, its partial sums of squares [S, H/32] written by the down_proj epilogue)."""
        Hq, Hkv, D = self.Hq, self.Hkv, self.D
        # RMSNorm scale, bias and RoPE all happen in this GEMM's epilogue; K / V land in the cache layout directly
        qkv = ops.gemm(x, L["wqkv"], bias=L.get("bqkv"), out=qkv_out, rms_in=ss_x, rms_eps=self.eps,
                       rope=(self.rope_table(pos0 + S), pos0, D, (Hq + Hkv) * D))
        o = ops.attention(qkv[:, : Hq * D], qkv[:, Hq * D: (Hq + Hkv) * D], qkv[:, (Hq + Hkv) * D:], B=1, S=S, Hq=Hq,
                          Hkv=Hkv, D=D, causal=True, scale=D ** -0.5)
        ss_mid = torch.empty((S, self.H // 32), device=x.device, dtype=torch.float32)
        x = ops.gemm(o, L["wo"], residual=x, sumsq_out=ss_mid)                      # stats of the mid-layer stream
        h = ops.gemm(x, L["wgu"], act=ops.ACT_SWIGLU, rms_in=ss_mid, rms_eps=self.eps)
        ss_out = torch.empty((S, self.H // 32), device=x.device, dtype=torch.float32)
        x = ops.gemm(h, L["wd"], residual=x, sumsq_out=ss_out)                      # stats for the next layer
        return x, ss_out

    def prefill(self, embeds: torch.Tensor, all_logits: bool = False, keep_cache: bool = False,
                max_len: Optional[int] = None, _no_graph: bool = False, tap=None):
        """embeds [S,H] bf16 -> (logits fp32 [S,V] or [1,V], final hidden [S,H] or None when graph-replayed).
        `tap(layer_index, stream)` (parity checks only) sees the residual stream after every layer; it forces the
        eager path."""
        if not self.is_loaded:
            raise RuntimeError("DecoderEngine: weights not loaded")
        if self._graphed is not None and not _no_graph and not all_logits and not keep_cache and tap is None:
            return self._graphed(embeds.contiguous()), None
        S = embeds.shape[0]
        x = embeds
        if keep_cache:
            self._ensure_cache(max_len or S, x.device)
            self.kv_len = S
        ss_x = ops.row_sumsq(x)
        for i, L in enumerate(self.layers):
            x, ss_x = self._layer(L, x, S, 0, self.kv[i][:S] if keep_cache else None, ss_x)
            if tap is not None:
                tap(i, x)
        if all_logits:
            logits = ops.gemm(x, self.w["lm_head"], out_dtype=torch.float32, rms_in=ss_x, rms_eps=self.eps)
        else:
            logits = ops.gemv(x[S - 1:].contiguous(), self.w["lm_head"], rms_eps=self.eps, out_dtype=torch.float32)
        return logits, x

    def _ensure_cache(self, cap: int, device) -> None:
        """The per-layer fused-row cache is allocated once and reused (a captured decode graph holds its addresses)."""
        if self.kv and self.kv[0].shape[0] >= cap and self.kv[0].device == torch.device(device):
            return
        cap = (cap + 255) // 256 * 256
        width = (self.Hq + 2 * self.Hkv) * self.D
        self.kv = [torch.empty((cap, width), device=device, dtype=self.dtype) for _ in self.layers]
        self._drop_decode_graphs()

    # ---- KV-cache decode (one token) -----------------------------------------------------------------------
    def decode_step(self, x: torch.Tensor) -> torch.Tensor:
        """x [1,H] bf16 (embedding of the newest token) -> logits fp32 [1,V]; appends K/V at position kv_len.
        Every linear layer is a weight-streaming GEMV with the RMSNorm in front of it fused (vl2_gemv_bf16), attention
        is the split-KV vl2_attention_decode."""
        if not self.kv:
            raise RuntimeError("decode_step needs prefill(keep_cache=True) first")
        pos = self.kv_len
        if pos >= self.kv[0].shape[0]:
            raise RuntimeError(f"KV cache full ({pos} positions)")
        Hq, Hkv, D = self.Hq, self.Hkv, self.D
        for i, L in enumerate(self.layers):
            cache = self.kv[i]
            row = cache[pos:pos + 1]
            ops.gemv(x, L["wqkv"], bias=L.get("bqkv"), out=row, rms_eps=self.eps)
            ops.rope_inplace(row, 1, Hq, Hkv, D, 0, Hq * D, pos, self.w["inv_freq"], interleaved=True)
            o = ops.attention_decode(row[0, : Hq * D], cache[:, Hq * D: (Hq + Hkv) * D], cache[:, (Hq + Hkv) * D:],
                                     n_pos=pos + 1, Hq=Hq, Hkv=Hkv, D=D, scale=D ** -0.5)
            x = ops.gemv(o, L["wo"], residual=x)
            h = ops.gemv(x, L["wgu"], act=ops.ACT_SWIGLU, rms_eps=self.eps)
            x = ops.gemv(h, L["wd"], residual=x)
        self.kv_len = pos + 1
        return ops.gemv(x, self.w["lm_head"], rms_eps=self.eps, out_dtype=torch.float32)

    # ---- the same step as ONE CUDA graph ---------------------------------------------------------------------
    def _decode_body(self, tok_dev: torch.Tensor, pos_dev: torch.Tensor, stage: torch.Tensor, log=None,
                     sampler: Optional[torch.Tensor] = None, processor: Optional[torch.Tensor] = None,
                     recorder: Optional[torch.Tensor] = None) -> torch.Tensor:
        """Single-token step whose position and token live in device memory: embeds *tok_dev, appends K/V at *pos_dev,
        writes argmax(logits) back to tok_dev and increments pos_dev, so one captured graph serves every token.
        `sampler` (a device vl2_sample_params block, needs `log`): the new token is drawn by vl2_sample_token with
        counter *step_dev + 1 instead - the n-th new token of a generate() call uses counter n, token 0 came from the
        prefill.  `processor` (a device vl2_logits_process_params block, needs `log`): vl2_process_logits edits the
        logits first, with the history _decode_hist[0 .. *step_dev + 1) = new tokens 0 .. n - 1.  `recorder` (a device
        vl2_score_record_params block, needs `log`): the raw logits row goes to slot n = *step_dev + 1 of its logits
        buffer before the processors edit it, and the row the token is chosen from (processed; warped by the scored
        sampler when sampling) to slot n of its scores buffer."""
        Hq, Hkv, D = self.Hq, self.Hkv, self.D
        x = torch.index_select(self.w["embed"], 0, tok_dev)
        o = torch.empty((1, Hq * D), device=x.device, dtype=self.dtype)
        for i, L in enumerate(self.layers):
            cache = self.kv[i]
            ops.gemv(x, L["wqkv"], bias=L.get("bqkv"), out=stage, rms_eps=self.eps)
            joined = None
            if self.decode_prefetch_mb > 0:       # fork: weight prefetch into L2 next to the attention phase
                main = torch.cuda.current_stream()
                if self._side_stream is None:
                    self._side_stream = torch.cuda.Stream(device=x.device)
                fork = torch.cuda.Event()
                fork.record(main)
                self._side_stream.wait_event(fork)
                with torch.cuda.stream(self._side_stream):
                    budget = int(self.decode_prefetch_mb * 1e6)
                    n_wo = L["wo"].numel() * 2
                    ops.l2_prefetch(L["wo"], min(budget, n_wo))
                    if budget > n_wo:
                        ops.l2_prefetch(L["wgu"], budget - n_wo)
                    joined = torch.cuda.Event()
                    joined.record(self._side_stream)
            ops.decode_rope_append(stage, cache, pos_dev, Hq, Hkv, D, self.w["inv_freq"], interleaved=True)
            ops.attention_decode_dyn(stage[0, : Hq * D], cache[:, Hq * D: (Hq + Hkv) * D], cache[:, (Hq + Hkv) * D:],
                                     pos_dev, Hq=Hq, Hkv=Hkv, D=D, scale=D ** -0.5, out=o)
            if joined is not None:
                torch.cuda.current_stream().wait_event(joined)
            x = ops.gemv(o, L["wo"], residual=x)
            h = ops.gemv(x, L["wgu"], act=ops.ACT_SWIGLU, rms_eps=self.eps)
            x = ops.gemv(h, L["wd"], residual=x)
        logits = ops.gemv(x, self.w["lm_head"], rms_eps=self.eps, out_dtype=torch.float32)
        if recorder is not None:
            ops.record_rows(logits, recorder, _lib.RECORD_LOGITS, log[1], 1, self.dtype)
        if processor is not None:
            ops.process_logits(logits, processor, self._decode_hist, log[1], 1, self.dtype)
        if sampler is None:
            if recorder is not None:
                ops.record_rows(logits, recorder, _lib.RECORD_SCORES, log[1], 1, self.dtype)
            tok_dev.copy_(torch.argmax(logits, dim=1))
        else:
            ops.sample_token(logits, sampler, log[1], 1, tok_dev, self.dtype, record=recorder)
        pos_dev.add_(1)
        if log is not None:          # device-side log of the generated ids: the host reads it in chunks, not per token
            gen_buf, step_dev = log
            gen_buf.scatter_(0, step_dev, tok_dev)
            step_dev.add_(1)
        return logits

    def _capture_decode(self, sampler: Optional[torch.Tensor], processor: Optional[torch.Tensor] = None,
                        recorder: Optional[torch.Tensor] = None):
        """Capture the single-token step (greedy, or sampled with the parameter block `sampler`; with the processor
        block `processor`, the logits processors first; with the record block `recorder`, recording its rows) on the
        shared buffers."""
        dev = self.kv[0].device
        if self._decode_bufs is None:
            self._decode_hist = torch.zeros((self.kv[0].shape[0] + 2,), device=dev, dtype=torch.int64)
            self._decode_bufs = (torch.zeros((1,), device=dev, dtype=torch.int64),
                                 torch.zeros((1,), device=dev, dtype=torch.int32),
                                 torch.empty((1, (self.Hq + 2 * self.Hkv) * self.D), device=dev, dtype=self.dtype),
                                 self._decode_hist[1:],
                                 torch.zeros((1,), device=dev, dtype=torch.int64))
            self._decode_log = self._decode_bufs[3:]
        tok_dev, pos_dev, stage, _, step_dev = self._decode_bufs
        log = self._decode_log
        scratch_pos = self.kv[0].shape[0] - 1     # warm-up writes land in the last cache row (rewritten when reached)
        side = torch.cuda.Stream(device=dev)
        side.wait_stream(torch.cuda.current_stream())
        with torch.cuda.stream(side):
            for _ in range(2):
                pos_dev.fill_(scratch_pos)
                step_dev.zero_()
                with ops.pdl(self.decode_pdl):
                    self._decode_body(tok_dev, pos_dev, stage, log, sampler, processor, recorder)
        torch.cuda.current_stream().wait_stream(side)
        graph = torch.cuda.CUDAGraph()
        with torch.cuda.graph(graph), ops.pdl(self.decode_pdl):
            logits = self._decode_body(tok_dev, pos_dev, stage, log, sampler, processor, recorder)
        return (graph, tok_dev, pos_dev, logits, stage)

    def decode_graph_begin(self, first_token: int, sampling: Optional[torch.Tensor] = None,
                           processing: Optional[torch.Tensor] = None, recording: Optional[torch.Tensor] = None) -> None:
        """Arm the graph-replayed decode loop after prefill(keep_cache=True): token := first_token, pos := kv_len.
        `sampling`: an ops.sampling_params block - arm the sampled graph (captured once, then reused for every parameter
        setting) instead of the greedy one.  `processing`: an ops.logits_process_params tensor - arm the variant of that
        graph with the logits processors (also captured once; the tensor is kept alive while armed).
        `recording`: an ops.score_record_params block - arm the recording variant of that graph (captured once per
        variant): step n writes its rows to slot n of the block's buffers, which must stay alive while armed."""
        if not self.kv:
            raise RuntimeError("decode_graph_begin needs prefill(keep_cache=True) first")
        dev = self.kv[0].device
        proc = None
        if processing is not None:
            if self._process_params is None or self._process_params.device != dev:
                self._process_params = torch.zeros((ops.PROCESS_HEADER_WORDS,), device=dev, dtype=torch.int64)
            self._process_params.copy_(processing[:ops.PROCESS_HEADER_WORDS])
            self._process_tables = processing
            proc = self._process_params
        if recording is not None:
            self._arm_recording(recording, sampling, proc)
        elif sampling is None:
            if proc is None:
                if self._decode_graph is None:
                    self._decode_graph = self._capture_decode(None)
                self._armed = self._decode_graph
            else:
                if self._decode_graph_processed is None:
                    self._decode_graph_processed = self._capture_decode(None, proc)
                self._armed = self._decode_graph_processed
        else:
            if self._sample_params is None or self._sample_params.device != dev:
                self._sample_params = torch.zeros((3,), device=dev, dtype=torch.int64)
            self._sample_params.copy_(sampling)
            if proc is None:
                if self._decode_graph_sampled is None:
                    self._decode_graph_sampled = self._capture_decode(self._sample_params)
                self._armed = self._decode_graph_sampled
            else:
                if self._decode_graph_sampled_processed is None:
                    self._decode_graph_sampled_processed = self._capture_decode(self._sample_params, proc)
                self._armed = self._decode_graph_sampled_processed
        _, tok_dev, pos_dev, _, _ = self._armed
        tok_dev.fill_(int(first_token))
        self._decode_hist[0].fill_(int(first_token))
        pos_dev.fill_(self.kv_len)
        self._decode_log[1].zero_()
        self._decode_read = 0

    def _arm_recording(self, recording: torch.Tensor, sampling: Optional[torch.Tensor], proc: Optional[torch.Tensor]):
        """Arm the recording graph for (sampled, processed), capturing it on first use.  The capture's warm-up steps run
        with a cleared block, so they write into no caller's buffer."""
        dev = self.kv[0].device
        if self._record_params is None or self._record_params.device != dev:
            self._record_params = torch.zeros((ops.SCORE_RECORD_WORDS,), device=dev, dtype=torch.int64)
        if sampling is not None:
            if self._sample_params is None or self._sample_params.device != dev:
                self._sample_params = torch.zeros((3,), device=dev, dtype=torch.int64)
            self._sample_params.copy_(sampling)
        key = (sampling is not None, proc is not None)
        if key not in self._decode_graphs_recorded:
            self._record_params.zero_()
            self._decode_graphs_recorded[key] = self._capture_decode(
                self._sample_params if sampling is not None else None, proc, self._record_params)
        self._record_params.copy_(recording)
        self._armed = self._decode_graphs_recorded[key]

    def decode_graph_run(self, k: int) -> None:
        """Enqueue k token steps back to back (no host round trip in between: each replay embeds the token the previous one
        left in device memory and logs its own token into the device-side id buffer)."""
        graph = self._armed[0]
        if self.kv_len + k > self.kv[0].shape[0]:
            raise RuntimeError(f"KV cache full ({self.kv_len} + {k} positions)")
        for _ in range(k):
            graph.replay()
        self.kv_len += k

    def decode_graph_tokens(self, k: int) -> list:
        """The next k logged token ids (one device->host copy, one synchronisation for the whole chunk)."""
        a = self._decode_read
        self._decode_read = a + k
        return self._decode_log[0][a:a + k].tolist()

    def decode_graph_step(self) -> torch.Tensor:
        """Replay one token; returns the device int64[1] holding the NEW token (the arg-max, or the draw when armed with
        sampling); the greedy graph's logits stay in its static buffer (`decode_graph_logits`)."""
        graph, tok_dev, _, _, _ = self._armed
        if self.kv_len >= self.kv[0].shape[0]:
            raise RuntimeError(f"KV cache full ({self.kv_len} positions)")
        graph.replay()
        self.kv_len += 1
        return tok_dev

    def shared_seed(self, seed: int) -> int:
        """The sampling seed every rank decoding this sequence uses (a single-GPU engine: its own)."""
        return seed

    @property
    def decode_graph_logits(self) -> torch.Tensor:
        return self._decode_graph[3]
