"""CLIP / SigLIP ViT towers on libvl2 kernels — same class surface as the reference's CLIPVisionTower and
SiglipVisionTower (videollama2/model/encoder.py:12-81, 84-151), arithmetic of HF CLIPVisionModel
(HF:clip/modeling_clip.py:202-218,282-385,647-696) and HF SiglipVisionModel (HF:siglip/modeling_siglip.py).

Only the layers that feed `hidden_states[select_layer]` are executed (select_layer = -2 -> 23 of 24; the reference runs
the 24th layer and post_layernorm and throws the result away)."""
from __future__ import annotations

import os
from typing import Dict, List, Optional

import torch

from .. import ops
from .config import VisionConfig

_PFX = "vision_tower.vision_model."


class _ImageProcessorInfo:
    """Carries the fields of CLIPImageProcessor the callers read (crop/size/mean/std); preprocessing itself is CPU I/O."""

    def __init__(self, size: int):
        self.crop_size = {"height": size, "width": size}
        self.size = {"shortest_edge": size}
        self.image_mean = [0.48145466, 0.4578275, 0.40821073]
        self.image_std = [0.26862954, 0.26130258, 0.27577711]


class CLIPVisionTower:
    def __init__(self, vision_tower: str, args, vision_config: Optional[VisionConfig] = None, load_pretrained=False):
        self.is_loaded = False
        self.vision_tower_name = vision_tower
        self.select_layer = args.mm_vision_select_layer
        self.select_feature = getattr(args, "mm_vision_select_feature", "patch")
        if self.select_feature not in ("patch", "cls_patch"):
            raise ValueError(f"Unexpected select feature: {self.select_feature}")
        if vision_config is None:
            vision_config = getattr(args, "vision_config", None) or VisionConfig.from_dir(vision_tower)
        self._config = vision_config
        self._dtype = getattr(args, "storage_dtype", torch.bfloat16)       # bf16 or fp16 (selects the library build)
        self.image_processor = _ImageProcessorInfo(vision_config.image_size)
        self._device = torch.device("cpu")
        self.w: Dict[str, torch.Tensor] = {}
        self.layers: List[Dict[str, torch.Tensor]] = []
        self._graphed = None

    def enable_cuda_graphs(self, on: bool = True):
        """Replay the tower as one CUDA graph per input shape (see videollama2_b200/graphs.py)."""
        from ..graphs import GraphedStage
        self._graphed = GraphedStage(self._features) if on else None
        return self

    # ---- weights -------------------------------------------------------------------------------------------
    @property
    def n_used_layers(self) -> int:
        L = self._config.num_hidden_layers
        n = L + 1 + self.select_layer if self.select_layer < 0 else self.select_layer
        if not 0 <= n <= L:
            raise ValueError(f"select_layer {self.select_layer} out of range for {L} layers")
        return n

    def load_state_dict(self, sd: Dict[str, torch.Tensor], device, prefix: str = _PFX) -> "CLIPVisionTower":
        """Repack HF-named CLIP weights once: fused QKV [3C,C], fp32 biases, patch conv as [C, Kpad] GEMM weight."""
        c = self._config
        dev = torch.device(device)
        bf = lambda t: t.to(device=dev, dtype=self._dtype).contiguous()
        f32 = lambda t: t.to(device=dev, dtype=torch.float32).contiguous()
        K = 3 * c.patch_size * c.patch_size
        self.kpad = (K + 63) // 64 * 64
        wp = torch.zeros((c.hidden_size, self.kpad), dtype=self._dtype, device=dev)
        wp[:, :K] = bf(sd[prefix + "embeddings.patch_embedding.weight"]).reshape(c.hidden_size, K)
        self.w = {
            "patch": wp,
            "cls": bf(sd[prefix + "embeddings.class_embedding"]),
            "pos": bf(sd[prefix + "embeddings.position_embedding.weight"]),
            "pre_g": bf(sd[prefix + "pre_layrnorm.weight"]), "pre_b": bf(sd[prefix + "pre_layrnorm.bias"]),
        }
        self._load_layers(sd, prefix, dev)
        self._device = dev
        self.is_loaded = True
        return self

    # ---- forward -------------------------------------------------------------------------------------------
    def hidden_states(self, images: torch.Tensor, last_out: Optional[torch.Tensor] = None, bcast_ptrs=None,
                      mc_ptr: int = 0) -> torch.Tensor:
        """[F,3,H,W] bf16 -> residual stream after the selected layer, [F, np+1, C].
        `last_out` ([F*(np+1), C] view, e.g. this rank's rows of a symmetric-memory gather buffer) receives the final
        GEMM's output; `bcast_ptrs` / `mc_ptr` make that GEMM's epilogue also store every tile into the peers' buffers
        (NVLink P2P) or an NVSwitch multicast address: the all-gather of visual tokens fused into the last ViT GEMM."""
        c = self._config
        Fn = images.shape[0]
        C = c.hidden_size
        H = c.num_attention_heads
        D = C // H
        S = self.num_patches + 1
        if self.fused_embed and self.kpad <= 640 and c.patch_size % 2 == 0 and C % 32 == 0:
            # one implicit-GEMM launch: gather patches -> wgmma conv -> + position -> class row -> pre-LayerNorm
            x = ops.patch_embed(images.contiguous(), self.w["patch"], self.w["pos"], c.patch_size, cls=self.w["cls"],
                                gamma=self.w["pre_g"], beta=self.w["pre_b"], eps=c.layer_norm_eps)
        else:
            A = ops.patch_im2col(images.contiguous(), c.patch_size, self.kpad)
            patch = ops.gemm(A, self.w["patch"])
            x = ops.clip_embed_finish(patch, self.w["cls"], self.w["pos"], self.w["pre_g"], self.w["pre_b"], Fn,
                                      c.layer_norm_eps)
        x = self._encoder(x, Fn, S, last_out, bcast_ptrs, mc_ptr, None)
        return x.view(Fn, S, C)

    _ACT = ops.ACT_QUICK_GELU

    # LayerNorms folded into the GEMMs that consume them (VL2_VIT_FOLD_LN=1): gamma goes into the weight columns, beta into
    # the bias, and the row statistics (sum, sum of squares) come out of the epilogue of the GEMM that produced the residual
    # stream - 2 launches and 2 round trips of the stream fewer per layer.  Parity-tested, but OFF by default: the K = 1024 tower
    # GEMMs are epilogue-bound, so the extra epilogue work can cost more than the 46 stand-alone LayerNorm launches it
    # removes (not measured on the H100).
    fold_layernorm = os.environ.get("VL2_VIT_FOLD_LN", "0") == "1"
    # embeddings as ONE implicit-GEMM kernel (vl2_patch_embed); VL2_VIT_FUSED_EMBED=0 -> explicit im2col + GEMM + finish
    fused_embed = os.environ.get("VL2_VIT_FUSED_EMBED", "1") != "0"

    def _encoder(self, x: torch.Tensor, Fn: int, S: int, last_out=None, bcast_ptrs=None, mc_ptr: int = 0,
                 stats=None) -> torch.Tensor:
        """Pre-LN transformer layers shared by both towers: LN -> fused QKV GEMM -> attention -> out_proj(+residual)
        -> LN -> fc1(+activation) -> fc2(+residual).  `stats` = (row sums, row sums of squares) of x for the folded form."""
        c = self._config
        C = c.hidden_size
        H = c.num_attention_heads
        D = C // H
        if self.fold_layernorm and self.layers and C % 32 == 0 and "wqkv_f" in self.layers[0]:
            return self._encoder_folded(x, Fn, S, last_out, bcast_ptrs, mc_ptr, stats)
        for li, L in enumerate(self.layers):
            last = li == len(self.layers) - 1
            y = ops.layernorm(x, L["ln1_g"], L["ln1_b"], c.layer_norm_eps)
            qkv = ops.gemm(y, L["wqkv"], bias=L["bqkv"])
            o = ops.attention(qkv[:, :C], qkv[:, C:2 * C], qkv[:, 2 * C:], B=Fn, S=S, Hq=H, Hkv=H, D=D, causal=False,
                              scale=D ** -0.5)
            x = ops.gemm(o, L["wo"], bias=L["bo"], residual=x)
            y = ops.layernorm(x, L["ln2_g"], L["ln2_b"], c.layer_norm_eps)
            h = ops.gemm(y, L["w1"], bias=L["b1"], act=self._ACT)
            if last and (last_out is not None or bcast_ptrs or mc_ptr):
                x = ops.gemm(h, L["w2"], bias=L["b2"], residual=x, out=last_out, bcast_ptrs=bcast_ptrs, mc_ptr=mc_ptr)
            else:
                x = ops.gemm(h, L["w2"], bias=L["b2"], residual=x)
        return x

    def _encoder_folded(self, x, Fn, S, last_out, bcast_ptrs, mc_ptr, stats):
        c = self._config
        C = c.hidden_size
        H = c.num_attention_heads
        D = C // H
        eps = c.layer_norm_eps
        M = x.shape[0]
        if stats is None:
            stats = ops.row_stats(x)
        new_stats = lambda: (torch.empty((M, C // 32), device=x.device, dtype=torch.float32),
                             torch.empty((M, C // 32), device=x.device, dtype=torch.float32))
        for li, L in enumerate(self.layers):
            last = li == len(self.layers) - 1
            qkv = ops.gemm(x, L["wqkv_f"], bias=L["bqkv_f"], ln_in=stats, ln_colsum=L["cqkv"], rms_eps=eps)
            o = ops.attention(qkv[:, :C], qkv[:, C:2 * C], qkv[:, 2 * C:], B=Fn, S=S, Hq=H, Hkv=H, D=D, causal=False,
                              scale=D ** -0.5)
            mid = new_stats()
            x = ops.gemm(o, L["wo"], bias=L["bo"], residual=x, rowsum_out=mid[0], sumsq_out=mid[1])
            h = ops.gemm(x, L["w1_f"], bias=L["b1_f"], act=self._ACT, ln_in=mid, ln_colsum=L["c1"], rms_eps=eps)
            if last:
                kw = {}
                if last_out is not None or bcast_ptrs or mc_ptr:
                    kw = dict(out=last_out, bcast_ptrs=bcast_ptrs, mc_ptr=mc_ptr)
                x = ops.gemm(h, L["w2"], bias=L["b2"], residual=x, **kw)
            else:
                stats = new_stats()
                x = ops.gemm(h, L["w2"], bias=L["b2"], residual=x, rowsum_out=stats[0], sumsq_out=stats[1])
        return x

    def _load_layers(self, sd, prefix, dev):
        bf = lambda t: t.to(device=dev, dtype=self._dtype).contiguous()
        f32 = lambda t: t.to(device=dev, dtype=torch.float32).contiguous()

        def fold(w, b, g, beta):
            """LN(x; g, beta) w^T + b  ->  (w * g as bf16, its fp32 row sums, b + w beta)."""
            wf = w.to(device=dev, dtype=torch.float32)
            wg = (wf * g.to(device=dev, dtype=torch.float32)[None, :]).to(self._dtype).contiguous()
            return wg, wg.float().sum(1).contiguous(), (b.to(device=dev, dtype=torch.float32)
                                                        + wf @ beta.to(device=dev, dtype=torch.float32)).contiguous()

        self.layers = []
        for i in range(self.n_used_layers):
            p = f"{prefix}encoder.layers.{i}."
            wqkv = torch.cat([sd[p + f"self_attn.{n}.weight"] for n in ("q_proj", "k_proj", "v_proj")], 0)
            bqkv = torch.cat([sd[p + f"self_attn.{n}.bias"] for n in ("q_proj", "k_proj", "v_proj")], 0)
            folded = {}
            if self.fold_layernorm:
                wq, cq, bq = fold(wqkv, bqkv, sd[p + "layer_norm1.weight"], sd[p + "layer_norm1.bias"])
                w1, c1, b1 = fold(sd[p + "mlp.fc1.weight"], sd[p + "mlp.fc1.bias"], sd[p + "layer_norm2.weight"],
                                  sd[p + "layer_norm2.bias"])
                folded = {"wqkv_f": wq, "cqkv": cq, "bqkv_f": bq, "w1_f": w1, "c1": c1, "b1_f": b1}
            self.layers.append({
                **folded,
                "ln1_g": bf(sd[p + "layer_norm1.weight"]), "ln1_b": bf(sd[p + "layer_norm1.bias"]),
                "ln2_g": bf(sd[p + "layer_norm2.weight"]), "ln2_b": bf(sd[p + "layer_norm2.bias"]),
                "wqkv": bf(torch.cat([sd[p + f"self_attn.{n}.weight"] for n in ("q_proj", "k_proj", "v_proj")], 0)),
                "bqkv": f32(torch.cat([sd[p + f"self_attn.{n}.bias"] for n in ("q_proj", "k_proj", "v_proj")], 0)),
                "wo": bf(sd[p + "self_attn.out_proj.weight"]), "bo": f32(sd[p + "self_attn.out_proj.bias"]),
                "w1": bf(sd[p + "mlp.fc1.weight"]), "b1": f32(sd[p + "mlp.fc1.bias"]),
                "w2": bf(sd[p + "mlp.fc2.weight"]), "b2": f32(sd[p + "mlp.fc2.bias"]),
            })

    def feature_select(self, hidden: torch.Tensor) -> torch.Tensor:
        if self.select_feature == "patch":
            return hidden[:, 1:]
        return hidden

    @torch.no_grad()
    def forward(self, images):
        if not self.is_loaded:
            raise RuntimeError("CLIPVisionTower: weights not loaded")
        if type(images) is list:
            return [self.forward(im.unsqueeze(0)) for im in images]
        if not images.is_cuda:
            raise ops._lib.Vl2Error("CLIPVisionTower needs CUDA tensors (no CPU fallback)")
        dt = images.dtype
        x = images.to(self._dtype).contiguous()
        feats = self._graphed(x) if self._graphed is not None else self._features(x)
        return feats.to(dt)

    def _features(self, images: torch.Tensor) -> torch.Tensor:
        return self.feature_select(self.hidden_states(images)).contiguous()

    __call__ = forward

    # ---- properties of the reference class (encoder.py:55-81) -----------------------------------------------
    @property
    def dtype(self):
        return self._dtype

    @property
    def device(self):
        return self._device

    @property
    def config(self):
        return self._config

    @property
    def hidden_size(self):
        return self._config.hidden_size

    @property
    def num_patches(self):
        return (self._config.image_size // self._config.patch_size) ** 2

    @property
    def seq_len(self):
        """Rows per frame of the residual stream (class token + patches)."""
        return self.num_patches + 1

    @property
    def num_patches_per_side(self):
        return self._config.image_size // self._config.patch_size

    @property
    def image_size(self):
        return self._config.image_size


class _SiglipProcessorInfo:
    """Fields of SiglipImageProcessor the callers read (mm_utils.py:132-202 / __init__.py:60-96)."""

    def __init__(self, size: int):
        self.size = {"height": size, "width": size}
        self.crop_size = {"height": size, "width": size}
        self.image_mean = [0.5, 0.5, 0.5]
        self.image_std = [0.5, 0.5, 0.5]


class SiglipVisionTower(CLIPVisionTower):
    """SigLIP ViT (so400m/14@384 in VideoLLaMA2.1): no class token, no pre-LN, patch conv WITH bias, learned position
    table over the patches, gelu-tanh MLP, LayerNorm eps 1e-6, head_dim 72 (encoder.py:84-151).  `feature_select` keeps
    every token (encoder.py:103-109); post_layernorm and the attention-pooling head never feed hidden_states[-2]."""

    _ACT = ops.ACT_GELU_TANH

    def __init__(self, vision_tower: str, args, vision_config: Optional[VisionConfig] = None, load_pretrained=False):
        super().__init__(vision_tower, args, vision_config=vision_config, load_pretrained=load_pretrained)
        if self.select_feature != "patch":
            raise ValueError(f"Unexpected select feature: {self.select_feature}")
        self.image_processor = _SiglipProcessorInfo(self._config.image_size)
        self._pos_rows: Dict[int, torch.Tensor] = {}

    def load_state_dict(self, sd: Dict[str, torch.Tensor], device, prefix: str = _PFX) -> "SiglipVisionTower":
        c = self._config
        dev = torch.device(device)
        K = 3 * c.patch_size * c.patch_size
        self.kpad = (K + 63) // 64 * 64
        wp = torch.zeros((c.hidden_size, self.kpad), dtype=self._dtype, device=dev)
        wp[:, :K] = sd[prefix + "embeddings.patch_embedding.weight"].to(device=dev, dtype=self._dtype).reshape(c.hidden_size, K)
        self.w = {
            "patch": wp,
            "patch_b": sd[prefix + "embeddings.patch_embedding.bias"].to(device=dev, dtype=torch.float32).contiguous(),
            "pos": sd[prefix + "embeddings.position_embedding.weight"].to(device=dev, dtype=self._dtype).contiguous(),
        }
        self._pos_rows = {}
        self._load_layers(sd, prefix, dev)
        self._device = dev
        self.is_loaded = True
        return self

    def hidden_states(self, images: torch.Tensor, last_out: Optional[torch.Tensor] = None, bcast_ptrs=None,
                      mc_ptr: int = 0) -> torch.Tensor:
        """[F,3,H,W] bf16 -> residual stream after the selected layer, [F, np, C].  The embedding is ONE implicit-GEMM
        launch (vl2_patch_embed: patches gathered from the frames, conv on wgmma, + bias + position rows in the epilogue);
        the explicit form (im2col + GEMM with the position table as residual operand) remains for the folded-LN variant."""
        c = self._config
        Fn = images.shape[0]
        S = self.num_patches
        if self.fused_embed and not self.fold_layernorm and self.kpad <= 640 and c.patch_size % 2 == 0 and c.hidden_size % 32 == 0:
            x = ops.patch_embed(images.contiguous(), self.w["patch"], self.w["pos"], c.patch_size, bias=self.w["patch_b"])
            x = self._encoder(x, Fn, S, last_out, bcast_ptrs, mc_ptr, None)
            return x.view(Fn, S, c.hidden_size)
        pos = self._pos_rows.get(Fn)
        if pos is None:
            pos = self.w["pos"].repeat(Fn, 1).contiguous()
            self._pos_rows[Fn] = pos
        A = ops.patch_im2col(images.contiguous(), c.patch_size, self.kpad)
        stats = None
        if self.fold_layernorm and self.layers and c.hidden_size % 32 == 0:
            M = A.shape[0]
            stats = (torch.empty((M, c.hidden_size // 32), device=A.device, dtype=torch.float32),
                     torch.empty((M, c.hidden_size // 32), device=A.device, dtype=torch.float32))
            x = ops.gemm(A, self.w["patch"], bias=self.w["patch_b"], residual=pos, rowsum_out=stats[0], sumsq_out=stats[1])
        else:
            x = ops.gemm(A, self.w["patch"], bias=self.w["patch_b"], residual=pos)
        x = self._encoder(x, Fn, S, last_out, bcast_ptrs, mc_ptr, stats)
        return x.view(Fn, S, c.hidden_size)

    def feature_select(self, hidden: torch.Tensor) -> torch.Tensor:
        return hidden

    @property
    def seq_len(self):
        return self.num_patches


def build_vision_tower(vision_tower_cfg, **kwargs):
    """encoder.py:154-164: 'clip' / 'siglip' in the tower name pick the class; an in-memory vision_config decides by its
    model_type."""
    vision_tower = getattr(vision_tower_cfg, "mm_vision_tower", getattr(vision_tower_cfg, "vision_tower", None))
    if vision_tower is None:
        raise ValueError("Unknown vision tower: None")
    vc = getattr(vision_tower_cfg, "vision_config", None)
    if vc is not None and "siglip" in getattr(vc, "model_type", ""):
        return SiglipVisionTower(vision_tower, args=vision_tower_cfg, **kwargs)
    if "clip" in vision_tower.lower() or vc is not None:
        return CLIPVisionTower(vision_tower, args=vision_tower_cfg, **kwargs)
    if "siglip" in vision_tower.lower():
        return SiglipVisionTower(vision_tower, args=vision_tower_cfg, **kwargs)
    raise ValueError(f"Unknown vision tower: {vision_tower}")
