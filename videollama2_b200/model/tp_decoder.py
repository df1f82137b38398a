"""Tensor-parallel decoder for the 72B configuration (BASELINE.json configs[4]: VideoLLaMA2-72B = Qwen2-72B backbone, 8 GPUs).

The reference has no tensor parallelism: its only multi-GPU loading is `device_map="auto"` (videollama2/model/__init__.py:48,54,
layer-wise placement by accelerate); 150 GB of bf16 weights need the 8 GPUs of a box either way.  This engine shards every
decoder layer Megatron-style over the ranks of one process group (SURVEY.md §8e):

    QKV        column-parallel   rank r owns q heads [r Hq/G, (r+1) Hq/G) and kv heads [r Hkv/G, (r+1) Hkv/G)  (+ their biases)
    attention  local             causal GQA over the rank's own heads: no communication
    o_proj     row-parallel      partial [S, H] per rank  -> all-reduce (sum) -> + residual
    gate / up  column-parallel   I/G columns each, SwiGLU in the GEMM epilogue
    down_proj  row-parallel      partial [S, H]           -> all-reduce (sum) -> + residual
    lm_head    vocab-parallel    V/G logits per rank      -> all-gather

Per layer that is the single-GPU engine's kernels on 1/G of the weights plus two all-reduces of [S, H] bf16.  The residual is
added by rank 0's GEMM epilogue (its partial carries x), so the reduced tensor IS the new residual stream; RMSNorm stays folded
into the consuming GEMMs, its row statistics are recomputed after each all-reduce.  Collective: NCCL (NVLS on NVSwitch) through
torch.distributed; the all-reduce is the only data-path exchange of the decoder.  Host logic is backend-agnostic (gloo CPU tests
of the partitioning); the kernels need CUDA."""
from __future__ import annotations

from typing import Dict, List, Optional

import torch
import torch.distributed as dist

from .. import ops
from .decoder import DecoderEngine


def shard_plan(config, rank: int, world: int) -> dict:
    """Which rows / columns of every decoder weight rank `rank` of `world` owns (pure index arithmetic)."""
    Hq, Hkv = config.num_attention_heads, config.num_key_value_heads
    D = config.hidden_size // Hq
    I, V = config.intermediate_size, config.vocab_size
    if Hq % world or Hkv % world or I % world or V % world:
        raise ValueError(f"tensor parallel degree {world} must divide heads ({Hq}/{Hkv}), intermediate ({I}) and vocab ({V})")
    if (I // world) % 8:
        raise ValueError(f"intermediate_size / {world} = {I // world} must be a multiple of 8 (16-byte rows)")
    hq, hkv, il, vl = Hq // world, Hkv // world, I // world, V // world
    return {
        "Hq": hq, "Hkv": hkv, "D": D, "I": il, "V": vl,
        "q_rows": (rank * hq * D, (rank + 1) * hq * D),          # rows of q_proj.weight / bias
        "kv_rows": (rank * hkv * D, (rank + 1) * hkv * D),       # rows of k_proj / v_proj
        "o_cols": (rank * hq * D, (rank + 1) * hq * D),          # columns of o_proj.weight
        "i_rows": (rank * il, (rank + 1) * il),                  # rows of gate / up, columns of down
        "v_rows": (rank * vl, (rank + 1) * vl),                  # rows of lm_head
    }


def shard_layer(sd: Dict[str, torch.Tensor], prefix: str, plan: dict) -> Dict[str, torch.Tensor]:
    """HF-named tensors of one decoder layer -> this rank's slices under the same names (so that the single-GPU repacking
    code can consume them unchanged)."""
    a, b = plan["q_rows"]
    c, d = plan["kv_rows"]
    e, f = plan["i_rows"]
    out = {
        prefix + "self_attn.q_proj.weight": sd[prefix + "self_attn.q_proj.weight"][a:b],
        prefix + "self_attn.k_proj.weight": sd[prefix + "self_attn.k_proj.weight"][c:d],
        prefix + "self_attn.v_proj.weight": sd[prefix + "self_attn.v_proj.weight"][c:d],
        prefix + "self_attn.o_proj.weight": sd[prefix + "self_attn.o_proj.weight"][:, plan["o_cols"][0]:plan["o_cols"][1]],
        prefix + "mlp.gate_proj.weight": sd[prefix + "mlp.gate_proj.weight"][e:f],
        prefix + "mlp.up_proj.weight": sd[prefix + "mlp.up_proj.weight"][e:f],
        prefix + "mlp.down_proj.weight": sd[prefix + "mlp.down_proj.weight"][:, e:f],
        prefix + "input_layernorm.weight": sd[prefix + "input_layernorm.weight"],
        prefix + "post_attention_layernorm.weight": sd[prefix + "post_attention_layernorm.weight"],
    }
    if prefix + "self_attn.q_proj.bias" in sd:
        out[prefix + "self_attn.q_proj.bias"] = sd[prefix + "self_attn.q_proj.bias"][a:b]
        out[prefix + "self_attn.k_proj.bias"] = sd[prefix + "self_attn.k_proj.bias"][c:d]
        out[prefix + "self_attn.v_proj.bias"] = sd[prefix + "self_attn.v_proj.bias"][c:d]
    return out


def shard_state_dict(sd: Dict[str, torch.Tensor], config, rank: int, world: int) -> Dict[str, torch.Tensor]:
    """Full HF decoder state dict -> the tensors rank `rank` loads (embedding and final norm replicated)."""
    plan = shard_plan(config, rank, world)
    out = {"model.embed_tokens.weight": sd["model.embed_tokens.weight"], "model.norm.weight": sd["model.norm.weight"],
           "lm_head.weight": sd["lm_head.weight"][plan["v_rows"][0]:plan["v_rows"][1]]}
    for i in range(config.num_hidden_layers):
        out.update(shard_layer(sd, f"model.layers.{i}.", plan))
    return out


class _LocalConfig:
    """The per-rank view of the decoder geometry: local head / intermediate / vocab counts, global hidden size."""

    def __init__(self, config, plan):
        self.__dict__.update({k: getattr(config, k) for k in ("hidden_size", "num_hidden_layers", "rms_norm_eps", "rope_theta")})
        self.max_position_embeddings = getattr(config, "max_position_embeddings", 32768)
        self.storage_dtype = getattr(config, "storage_dtype", torch.bfloat16)
        self.num_attention_heads = plan["Hq"]
        self.num_key_value_heads = plan["Hkv"]
        self.intermediate_size = plan["I"]
        self.vocab_size = plan["V"]
        self.head_dim = plan["D"]


class TPDecoderEngine(DecoderEngine):
    """DecoderEngine whose linear layers are sharded over `group`; call surface of DecoderEngine (prefill / decode_step).
    Every rank passes the SAME embeds and receives the SAME logits."""

    def __init__(self, config, group=None):
        self.group = group
        self.rank = dist.get_rank(group)
        self.world = dist.get_world_size(group)
        self.full_config = config
        self.plan = shard_plan(config, self.rank, self.world)
        super().__init__(_LocalConfig(config, self.plan))
        self.D = self.plan["D"]                      # head width comes from the GLOBAL geometry (hidden / all heads)
        self.graph_decode = False                    # collectives run eagerly between kernels
        self._nvls = None

    def load_state_dict(self, sd: Dict[str, torch.Tensor], device, presharded: bool = False) -> "TPDecoderEngine":
        """`sd`: the full HF-named state dict (sliced here), or with presharded=True this rank's slices already."""
        local = sd if presharded else shard_state_dict(sd, self.full_config, self.rank, self.world)
        return super().load_state_dict(local, device)

    # ---- collectives ---------------------------------------------------------------------------------------------
    def enable_nvls_all_reduce(self, max_rows: int, use_multicast: bool = True, inswitch_reduce: bool = False):
        """Route the prefill all-reduces through the library's own kernel (parallel.NvlsAllReduce: reduction over peer memory +
        RMSNorm statistics + NVSwitch broadcast in one launch) instead of NCCL + a statistics kernel.  The row-parallel GEMMs then
        write their partials straight into the symmetric buffer."""
        from ..parallel import NvlsAllReduce
        self._nvls = NvlsAllReduce(max_rows, self.H, self.device, self.group, use_multicast, inswitch_reduce, self.dtype) \
            if self.world > 1 else None
        return self

    def _all_reduce(self, part: torch.Tensor) -> torch.Tensor:
        """Sum of the ranks' partial [S, H] tensors, in place (rank 0's partial already carries the residual)."""
        if self.world > 1:
            dist.all_reduce(part, op=dist.ReduceOp.SUM, group=self.group)
        return part

    def _reduce_stats(self, gemm_into):
        """Run a row-parallel GEMM (`gemm_into(out)` writes the partial) and return (reduced stream, its row sums of squares)."""
        nv = getattr(self, "_nvls", None)
        S = self._cur_rows
        if nv is not None and S <= nv.max_rows:
            gemm_into(nv.part[:S])
            return nv.reduce(S)
        x = self._all_reduce(gemm_into(None))
        return x, ops.row_sumsq(x)

    def _gather_logits(self, local: torch.Tensor) -> torch.Tensor:
        """[rows, V/G] per rank -> [rows, V] (vocab shards are contiguous row ranges of lm_head)."""
        if self.world == 1:
            return local
        parts = [torch.empty_like(local) for _ in range(self.world)]
        dist.all_gather(parts, local.contiguous(), group=self.group)
        return torch.cat(parts, dim=-1)

    def shared_seed(self, seed: int) -> int:
        """The first rank's sampling seed, on every rank of the group: the ranks then draw the same token from the identical
        gathered logits, whatever state their own generators are in."""
        if self.world == 1:
            return seed
        dev = self.device if dist.get_backend(self.group) == "nccl" else torch.device("cpu")
        t = torch.tensor([seed], dtype=torch.int64, device=dev)
        src = dist.get_global_rank(self.group, 0) if self.group is not None else 0
        dist.broadcast(t, src=src, group=self.group)
        return int(t.item())

    # ---- one layer -------------------------------------------------------------------------------------------------
    def _layer(self, L, x: torch.Tensor, S: int, pos0: int, qkv_out: Optional[torch.Tensor], ss_x: torch.Tensor):
        Hq, Hkv, D = self.Hq, self.Hkv, self.D
        res = x if self.rank == 0 else None          # the residual enters the sum exactly once
        qkv = ops.gemm(x, L["wqkv"], bias=L.get("bqkv"), out=qkv_out, rms_in=ss_x, rms_eps=self.eps,
                       rope=(self.rope_table(pos0 + S), pos0, D, (Hq + Hkv) * D))
        o = ops.attention(qkv[:, : Hq * D], qkv[:, Hq * D: (Hq + Hkv) * D], qkv[:, (Hq + Hkv) * D:], B=1, S=S, Hq=Hq,
                          Hkv=Hkv, D=D, causal=True, scale=D ** -0.5)
        self._cur_rows = S
        x, ss = self._reduce_stats(lambda out: ops.gemm(o, L["wo"], residual=res, out=out))
        h = ops.gemm(x, L["wgu"], act=ops.ACT_SWIGLU, rms_in=ss, rms_eps=self.eps)
        res2 = x if self.rank == 0 else None
        return self._reduce_stats(lambda out: ops.gemm(h, L["wd"], residual=res2, out=out))

    def prefill(self, embeds: torch.Tensor, all_logits: bool = False, keep_cache: bool = False,
                max_len: Optional[int] = None, _no_graph: bool = False, tap=None):
        logits, x = super().prefill(embeds, all_logits=all_logits, keep_cache=keep_cache, max_len=max_len, _no_graph=True,
                                    tap=tap)
        return self._gather_logits(logits), x

    # ---- single-token decode (eager: one GEMV per shard + a [1, H] all-reduce after o_proj and down_proj) ------------------
    def decode_step(self, x: torch.Tensor) -> torch.Tensor:
        if not self.kv:
            raise RuntimeError("decode_step needs prefill(keep_cache=True) first")
        pos = self.kv_len
        if pos >= self.kv[0].shape[0]:
            raise RuntimeError(f"KV cache full ({pos} positions)")
        Hq, Hkv, D = self.Hq, self.Hkv, self.D
        for i, L in enumerate(self.layers):
            cache = self.kv[i]
            row = cache[pos:pos + 1]
            res = x if self.rank == 0 else None
            ops.gemv(x, L["wqkv"], bias=L.get("bqkv"), out=row, rms_eps=self.eps)
            ops.rope_inplace(row, 1, Hq, Hkv, D, 0, Hq * D, pos, self.w["inv_freq"], interleaved=True)
            o = ops.attention_decode(row[0, : Hq * D], cache[:, Hq * D: (Hq + Hkv) * D], cache[:, (Hq + Hkv) * D:],
                                     n_pos=pos + 1, Hq=Hq, Hkv=Hkv, D=D, scale=D ** -0.5)
            x = self._all_reduce(ops.gemv(o, L["wo"], residual=res))
            h = ops.gemv(x, L["wgu"], act=ops.ACT_SWIGLU, rms_eps=self.eps)
            x = self._all_reduce(ops.gemv(h, L["wd"], residual=res if res is None else x))
        self.kv_len = pos + 1
        return self._gather_logits(ops.gemv(x, self.w["lm_head"], rms_eps=self.eps, out_dtype=torch.float32))
