"""STC connector on libvl2 kernels — same class surface as videollama2/model/projector.py:133-238
(STCConnector, STCConnectorV35, build_vision_projector, load_mm_projector).

Everything is channels-last: the ViT output [F, 576, C] *is* [F,24,24,C], so the reference's `b d t h w` rearranges
(projector.py:196-213) disappear.  RegStage 1x1 convs, the Conv3d (after a tap-gather) and the readout MLP are
vl2_gemm_bf16 calls; LayerNorm+SiLU, depthwise 3x3, SE squeeze/excite are fused row kernels (SURVEY.md Appendix B)."""
from __future__ import annotations

import os
import re
from typing import Dict, List, Optional

import torch

from .. import ops

_REGSTAGE_LN_EPS = 1e-5  # timm LayerNormAct2d default (norm_layer=LayerNorm2d is mapped to it inside ConvNormAct)


def load_mm_projector(model_path, cache_dir=None, token=None):
    """projector.py:49-63 — local files only (no hub access in this engine)."""
    path = os.path.join(model_path, "mm_projector.bin")
    if not os.path.exists(path):
        raise FileNotFoundError(f"{path} not found (hub download is not supported; pass a local directory)")
    weights = torch.load(path, map_location="cpu")
    return {k: v.to(torch.float16) for k, v in weights.items()}


class STCConnector:
    """Temporal Convolutional Vision-Language Connector (projector.py:133-215)."""

    padding = 1

    def __init__(self, config, downsample=(2, 2, 2), depth=4, mlp_depth=2):
        if tuple(downsample) != (2, 2, 2):
            raise NotImplementedError("STCConnector engine supports downsample=(2,2,2) only")
        if mlp_depth != 2:
            raise NotImplementedError("STCConnector engine supports mlp_depth=2 only")
        self.encoder_hidden_size = config.mm_hidden_size
        self.hidden_size = config.hidden_size
        self.output_hidden_size = config.hidden_size
        self.depth = depth
        self.mlp_depth = mlp_depth
        self.downsample = tuple(downsample)
        self.eps = _REGSTAGE_LN_EPS
        self.dtype = getattr(config, "storage_dtype", torch.bfloat16)      # bf16 or fp16 (selects the library build)
        self.s1_dtype = self.dtype
        self.blocks: Dict[str, List[Dict[str, torch.Tensor]]] = {"s1": [], "s2": []}
        self.w: Dict[str, torch.Tensor] = {}
        self.is_loaded = False
        self._graphed = None
        self._graphed_s1 = None
        self._graphed_tail = None

    def enable_cuda_graphs(self, on: bool = True):
        from ..graphs import GraphedStage
        self._graphed = GraphedStage(lambda x: self._forward_one(x, None)) if on else None
        # the two halves the frame-parallel path runs on either side of its all-gather (parallel.FrameParallel)
        self._graphed_s1 = GraphedStage(self.run_s1) if on else None
        self._graphed_tail = GraphedStage(lambda a: self.run_readout(self.run_s2(self.run_sampler(a)), None)) if on else None
        return self

    # ---- weights -------------------------------------------------------------------------------------------
    def load_state_dict(self, sd: Dict[str, torch.Tensor], device, prefix: str = "") -> "STCConnector":
        dev = torch.device(device)
        bf = lambda t: t.to(device=dev, dtype=self.dtype).contiguous()
        f32 = lambda t: t.to(device=dev, dtype=torch.float32).contiguous()
        C = self.hidden_size
        for stage in ("s1", "s2"):
            self.blocks[stage] = []
            for b in range(1, self.depth + 1):
                p = f"{prefix}{stage}.b{b}."
                w1 = sd[p + "conv1.conv.weight"]
                blk = {
                    "w1": bf(w1.reshape(w1.shape[0], w1.shape[1])),
                    "g1": bf(sd[p + "conv1.bn.weight"]), "b1": bf(sd[p + "conv1.bn.bias"]),
                    "wd": bf(sd[p + "conv2.conv.weight"].reshape(C, 9).t()),           # [9, C]: tap-major
                    "g2": bf(sd[p + "conv2.bn.weight"]), "b2": bf(sd[p + "conv2.bn.bias"]),
                    "f1": bf(sd[p + "se.fc1.weight"].reshape(-1, C)), "f1b": f32(sd[p + "se.fc1.bias"]),
                    "f2": bf(sd[p + "se.fc2.weight"].reshape(C, -1)), "f2b": f32(sd[p + "se.fc2.bias"]),
                    "w3": bf(sd[p + "conv3.conv.weight"].reshape(C, C)),
                    "g3": bf(sd[p + "conv3.bn.weight"]), "b3": bf(sd[p + "conv3.bn.bias"]),
                }
                if p + "downsample.conv.weight" in sd:
                    ws = sd[p + "downsample.conv.weight"]
                    blk.update({"ws": bf(ws.reshape(ws.shape[0], ws.shape[1])),
                                "gs": bf(sd[p + "downsample.bn.weight"]), "bs": bf(sd[p + "downsample.bn.bias"])})
                self.blocks[stage].append(blk)
        wc = sd[prefix + "sampler.0.weight"]                                             # [C, C, 2, 2, 2]
        self.w = {
            "wc": bf(wc.permute(0, 2, 3, 4, 1).reshape(C, 8 * C)),                       # K index = tap*C + cin
            "bc": f32(sd[prefix + "sampler.0.bias"]),
            "r0": bf(sd[prefix + "readout.0.weight"]), "r0b": f32(sd[prefix + "readout.0.bias"]),
            "r2": bf(sd[prefix + "readout.2.weight"]), "r2b": f32(sd[prefix + "readout.2.bias"]),
        }
        self.is_loaded = True
        return self

    # ---- forward -------------------------------------------------------------------------------------------
    def _block(self, blk, x: torch.Tensor) -> torch.Tensor:
        """timm regnet.Bottleneck (1x1 -> LN+SiLU -> dw3x3 -> LN+SiLU -> SE -> 1x1 -> LN -> +shortcut -> SiLU); x [F,H,W,Cin]."""
        Fn, H, W, cin = x.shape
        C = self.hidden_size
        x2 = x.view(-1, cin)
        y = ops.gemm(x2, blk["w1"])
        y = ops.layernorm(y, blk["g1"], blk["b1"], self.eps, act=ops.ACT_SILU)
        y, pooled = ops.dwconv3x3_ln_silu(y.view(Fn, H, W, C), blk["wd"], blk["g2"], blk["b2"], self.eps)
        s = ops.gemm_skinny(pooled, blk["f1"], bias=blk["f1b"], act=ops.ACT_SILU)
        s = ops.gemm_skinny(s, blk["f2"], bias=blk["f2b"], act=ops.ACT_SIGMOID)
        ops.se_scale(y, s)
        z = ops.gemm(y.view(-1, C), blk["w3"])
        if "ws" in blk:
            r = ops.layernorm(ops.gemm(x2, blk["ws"]), blk["gs"], blk["bs"], self.eps)
        else:
            r = x2
        out = ops.layernorm(z, blk["g3"], blk["b3"], self.eps, act=ops.ACT_SILU, residual=r)
        return out.view(Fn, H, W, C)

    def run_s1(self, x: torch.Tensor) -> torch.Tensor:
        """[T,H,W,Cin] -> [T,H,W,C]: first RegStage, per frame (frames are the batch; SE pools per frame)."""
        for blk in self.blocks["s1"]:
            x = self._block(blk, x)
        return x

    def run_sampler(self, x: torch.Tensor) -> torch.Tensor:
        """[T,H,W,C] -> [T',H',W',C]: Conv3d(k=s=2, padding) + SiLU as an implicit GEMM (projector.py:164-174)."""
        T, H, W, C = x.shape
        p = self.padding
        To, Ho, Wo = (T + 2 * p - 2) // 2 + 1, (H + 2 * p - 2) // 2 + 1, (W + 2 * p - 2) // 2 + 1
        if Wo <= 16 and Ho <= 16 and C % 64 == 0 and ((W % 2 == 0 and H % 2 == 0) or p == 0):
            # implicit GEMM: the TMA producer of vl2_gemm_bf16 gathers the taps from x itself (no im2col matrix)
            return ops.conv3d_k2s2(x.contiguous(), self.w["wc"], bias=self.w["bc"], act=ops.ACT_SILU, pad=p).view(To, Ho, Wo, C)
        A = ops.conv3d_im2col(x.contiguous(), p)       # frames beyond 16 x 16 output positions: explicit tap gather
        return ops.gemm(A, self.w["wc"], bias=self.w["bc"], act=ops.ACT_SILU).view(To, Ho, Wo, C)

    def run_s2(self, y: torch.Tensor) -> torch.Tensor:
        for blk in self.blocks["s2"]:
            y = self._block(blk, y)
        return y

    def run_readout(self, y: torch.Tensor, out: Optional[torch.Tensor] = None) -> torch.Tensor:
        """[..., C] -> [(t h w), C]: Linear -> GELU(erf) -> Linear (projector.py:125-130); may write into `out`."""
        C = self.hidden_size
        h = ops.gemm(y.reshape(-1, C), self.w["r0"], bias=self.w["r0b"], act=ops.ACT_GELU_ERF)
        return ops.gemm(h, self.w["r2"], bias=self.w["r2b"], out=out)

    def _forward_one(self, x: torch.Tensor, out: Optional[torch.Tensor]) -> torch.Tensor:
        """x: [T, H, W, Cin] (one video) -> [T'*H'*W', C]; the last GEMM can write straight into `out`."""
        return self.run_readout(self.run_s2(self.run_sampler(self.run_s1(x))), out)

    def forward_s1(self, x: torch.Tensor) -> torch.Tensor:
        """[f,H,W,Cin] -> [f,H,W,C]: the per-frame half of the connector (first RegStage) on any subset of frames."""
        if not self.is_loaded:
            raise RuntimeError("STCConnector: weights not loaded")
        x = x.to(self.dtype).contiguous()
        g = getattr(self, "_graphed_s1", None)
        return g(x) if g is not None else self.run_s1(x)

    def forward_from_s1(self, a: torch.Tensor) -> torch.Tensor:
        """[b,T,H,W,C] (first-RegStage output of every frame) -> [b, l', D]: Conv3d sampler + s2 + readout."""
        b = a.size(0)
        out = torch.empty((b, self.num_output_tokens(a.size(1), a.size(2)), self.output_hidden_size), device=a.device,
                          dtype=self.dtype)
        g = getattr(self, "_graphed_tail", None)
        for i in range(b):
            if g is not None:
                out[i].copy_(g(a[i].contiguous()))
            else:
                self.run_readout(self.run_s2(self.run_sampler(a[i].contiguous())), out[i])
        return out

    def num_output_tokens(self, t: int, hw: int) -> int:
        p = self.padding
        return ((t + 2 * p - 2) // 2 + 1) * ((hw + 2 * p - 2) // 2 + 1) ** 2

    def forward(self, x: torch.Tensor, out: Optional[torch.Tensor] = None) -> torch.Tensor:
        """x: [b, t, l, d] or [b, t, h, w, d]  ->  [b, l', D]   (projector.py:189-215)."""
        if not self.is_loaded:
            raise RuntimeError("STCConnector: weights not loaded")
        if not x.is_cuda:
            raise ops._lib.Vl2Error("STCConnector needs CUDA tensors (no CPU fallback)")
        dt = x.dtype
        if x.ndim == 4:
            hw = int(x.size(2) ** 0.5)
            x = x.reshape(x.size(0), x.size(1), hw, hw, x.size(3))
        elif x.ndim != 5:
            raise ValueError(f"STCConnector expects a 4-D or 5-D input, got {x.ndim}-D")
        x = x.to(self.dtype).contiguous()
        b = x.size(0)
        n = self.num_output_tokens(x.size(1), x.size(2))
        if self._graphed is not None and b == 1 and out is None:
            # one video, graph replay: hand out the graph's own output buffer (valid until the next call with this shape;
            # the splice copies it into inputs_embeds right away) instead of staging it through another tensor
            return self._graphed(x[0]).unsqueeze(0).to(dt)
        if out is None:
            out = torch.empty((b, n, self.output_hidden_size), device=x.device, dtype=self.dtype)
        for i in range(b):
            if self._graphed is not None:
                out[i].copy_(self._graphed(x[i]))
            else:
                self._forward_one(x[i], out[i])
        return out.to(dt)

    __call__ = forward


class STCConnectorV35(STCConnector):
    """projector.py:225-238: same connector with an un-padded Conv3d."""
    padding = 0


def build_vision_projector(config, delay_load=False, **kwargs):
    """projector.py:95-122.  This engine implements the STC family; the ablation variants are not on the hot path."""
    projector_type = getattr(config, "mm_projector_type", "linear")
    if projector_type == "stc_connector":
        return STCConnector(config)
    if projector_type == "stc_connector_v35":
        return STCConnectorV35(config)
    if projector_type in ("linear", "identity", "stp_connector", "spatial_conv", "spatial_pool") or \
            re.match(r"^mlp(\d+)x_gelu$", projector_type):
        raise NotImplementedError(f"projector type {projector_type} is not implemented in this engine")
    raise ValueError(f"Unknown projector type: {projector_type}")
