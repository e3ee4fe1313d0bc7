"""Drop-in `MoGeModel` for the MoGe-2 inference hot path, backed by libmoge_b200.so (hand-written sm_90a CUDA).

Mirrors the public surface of /root/reference/moge/model/v2.py:
  __init__ kwargs (v2.py:30-57), from_pretrained (v2.py:76-107), .to/.eval/.half, .device/.dtype (v2.py:59-65),
  forward(image, num_tokens) -> {'points','normal','mask','metric_scale'} (v2.py:138-192),
  infer(image, num_tokens, resolution_level, force_projection, apply_mask, fov_x, use_fp16)
      -> {'points','intrinsics','depth','mask','normal'} (v2.py:194-303),
and, with no reference counterpart, infer_many(images, ...) over a list of images of different sizes (one encoder pass per call).
This file holds the MoGe-2 config, its engine hooks (token grid, output heads, group struct, post-processing) and the public
signatures; the forward path itself (engine calls, chunking, packing, the bodies of forward / infer / infer_many) is EngineModel's
in _engine.py.  Host logic only: tensor allocation and checkpoint I/O use PyTorch, every arithmetic step of the path runs in the
C-ABI library.  There is no CPU / eager fallback.
"""
from __future__ import annotations

import warnings
from numbers import Number
from typing import Any, Dict, List, Optional, Union

import ctypes as C
import torch

from .. import capi
from ..configs import backbone_dims, token_grid
from ._engine import EngineModel


class _HeadMarker:
    """Truthy placeholder so that `hasattr(model, 'normal_head')` works like on the reference module (app.py:260)."""

    def __init__(self, cfg):
        self.config = cfg

    def __repr__(self):
        return f"<moge_b200 decoder stack {self.config}>"


class MoGeModel(EngineModel):
    _strict_load = False            # the reference's from_pretrained loads with strict=False (v2.py:105)
    _fp32_pass_error = (
        "moge_b200: use_fp16=False (full-fp32 network pass) is not provided; the engine computes with 16-bit "
        "tensor-core operands, fp32 accumulation, an fp32 residual stream and fp32 post-processing (outputs within "
        "1e-3 of the fp32 reference, see DESIGN.md).  Call infer(..., use_fp16=True).")

    def __init__(self,
                 encoder: Dict[str, Any],
                 neck: Dict[str, Any],
                 points_head: Dict[str, Any] = None,
                 mask_head: Dict[str, Any] = None,
                 normal_head: Dict[str, Any] = None,
                 scale_head: Dict[str, Any] = None,
                 remap_output: str = 'linear',
                 num_tokens_range: List[int] = [1200, 3600],
                 **deprecated_kwargs):
        if deprecated_kwargs:
            warnings.warn(f"The following deprecated/invalid arguments are ignored: {deprecated_kwargs}")
        if remap_output not in capi.REMAP:
            raise ValueError(f"Invalid remap output type: {remap_output}")
        backbone_dims(encoder["backbone"])          # validates the backbone name
        self.remap_output = remap_output
        self.num_tokens_range = list(num_tokens_range)
        self.model_config = dict(encoder=encoder, neck=neck, points_head=points_head, mask_head=mask_head,
                                 normal_head=normal_head, scale_head=scale_head, remap_output=remap_output,
                                 num_tokens_range=list(num_tokens_range))
        self.encoder = _HeadMarker(encoder)
        self.neck = _HeadMarker(neck)
        for name, cfg in (("points_head", points_head), ("mask_head", mask_head), ("normal_head", normal_head),
                          ("scale_head", scale_head)):
            if cfg is not None:
                setattr(self, name, _HeadMarker(cfg))
        super().__init__()

    # ------------------------------------------------------------------ nn.Module-like plumbing
    @property
    def onnx_compatible_mode(self) -> bool:
        return False

    @onnx_compatible_mode.setter
    def onnx_compatible_mode(self, value: bool):
        if value:
            raise NotImplementedError("onnx_compatible_mode changes the resize/pos-embed numerics (modules.py:121, "
                                      "vision_transformer.py:192) and is not provided by the engine")

    def init_weights(self):
        raise NotImplementedError("training-only (v2.py:109-110)")

    def enable_gradient_checkpointing(self):
        raise NotImplementedError("training-only (v2.py:112-117)")

    def enable_pytorch_native_sdpa(self):
        pass    # attention always runs in the engine's own kernel

    def _expected_keys(self) -> List[str]:
        from ..synthetic import expected_keys
        return expected_keys(self.model_config)

    # ------------------------------------------------------------------ engine hooks (EngineModel runs the forward path)
    _group_t = capi.Group
    _c_workspace_bytes_groups = "moge_engine_workspace_bytes_groups"
    _c_forward_groups = "moge_engine_forward_groups"
    _output_names = ("points", "normal", "mask", "metric_scale")

    def _create_engine(self, handle: C.c_void_p):
        cfg = capi.make_config(self.model_config, self._compute_code())
        capi.check(capi.lib().moge_engine_create(C.byref(cfg), self._device.index, C.byref(handle)))

    def _geometry(self, H: int, W: int, num_tokens):
        """((h, w) token grid, token rows per image) of an H x W image at `num_tokens`, truncated to an int."""
        h, w = token_grid(H, W, int(num_tokens))
        return (h, w), h * w + 1

    def _alloc_outputs(self, B: int, H: int, W: int):
        """fp32 (points, normal, mask_prob, metric_scale) buffers for B images of H x W, absent heads as None."""
        dev = self._device
        points = torch.empty(B, H, W, 3, dtype=torch.float32, device=dev) if hasattr(self, "points_head") else None
        normal = torch.empty(B, H, W, 3, dtype=torch.float32, device=dev) if hasattr(self, "normal_head") else None
        mask = torch.empty(B, H, W, dtype=torch.float32, device=dev) if hasattr(self, "mask_head") else None
        scale = torch.empty(B, dtype=torch.float32, device=dev) if hasattr(self, "scale_head") else None
        return points, normal, mask, scale

    def _fill_group(self, g: capi.Group, geom, outputs):
        g.h, g.w = geom
        g.points, g.normal, g.mask_prob, g.metric_scale = (capi.ptr(t) for t in outputs)

    def _postprocess(self, outputs, aspect_ratio, fov_x, apply_mask, force_projection) -> Dict[str, torch.Tensor]:
        """K18 + K19 of infer() (v2.py:246-298) on the raw forward outputs of one shape group; all on the device."""
        points, normal, mask, metric_scale = outputs
        dev = self._device
        some = points if points is not None else (normal if normal is not None else mask)
        B, H, W = some.shape[0], some.shape[1], some.shape[2]
        L = capi.lib()
        ret: Dict[str, torch.Tensor] = {}
        with torch.cuda.device(dev):
            stream = capi.current_stream()
            if points is not None:
                focal = torch.empty(B, dtype=torch.float32, device=dev)
                shift = torch.empty(B, dtype=torch.float32, device=dev)
                focal_in = self._focal_in(fov_x, aspect_ratio, B)
                capi.check(L.moge_recover_focal_shift(points.data_ptr(), capi.ptr(mask), None, B, H, W,
                                                      capi.ptr(focal_in), focal.data_ptr(), shift.data_ptr(), stream))
                depth = torch.empty(B, H, W, dtype=torch.float32, device=dev)
                intrinsics = torch.empty(B, 3, 3, dtype=torch.float32, device=dev)
                normal_out = torch.empty_like(normal) if normal is not None else None
                mask_out = torch.empty(B, H, W, dtype=torch.uint8, device=dev) if mask is not None else None
                capi.check(L.moge_postprocess(points.data_ptr(), capi.ptr(normal), capi.ptr(mask), capi.ptr(metric_scale),
                                              focal.data_ptr(), shift.data_ptr(), B, H, W, int(bool(force_projection)),
                                              int(bool(apply_mask)), depth.data_ptr(), capi.ptr(normal_out),
                                              capi.ptr(mask_out), intrinsics.data_ptr(), stream))
                ret['points'] = points
                ret['intrinsics'] = intrinsics
                ret['depth'] = depth
                if mask_out is not None:
                    ret['mask'] = mask_out.view(torch.bool)
                if normal_out is not None:
                    ret['normal'] = normal_out
            else:
                mask_binary = None
                if mask is not None:
                    mask_binary = mask > 0.5
                    ret['mask'] = mask_binary
                if normal is not None:
                    if apply_mask and mask_binary is not None:        # v2.py:283-286
                        normal = torch.where(mask_binary[..., None], normal, torch.zeros_like(normal))
                    ret['normal'] = normal
        return ret

    # ------------------------------------------------------------------ public API
    @torch.inference_mode()
    def infer(self,
              image: torch.Tensor,
              num_tokens: int = None,
              resolution_level: int = 9,
              force_projection: bool = True,
              apply_mask: bool = True,
              fov_x: Optional[Union[Number, torch.Tensor]] = None,
              use_fp16: bool = True) -> Dict[str, torch.Tensor]:
        """Same contract as v2.py:194-303.  The engine always multiplies in 16-bit (fp16, or bf16 after
        `.bfloat16()`) with fp32 accumulation, fp32 residual stream and fp32 post-processing; a full-fp32 network pass
        (the reference's `use_fp16=False`, v2.py:241) does not exist here, so asking for it is an error rather than a silent
        precision downgrade."""
        return self._infer(image, num_tokens=num_tokens, resolution_level=resolution_level, force_projection=force_projection,
                           apply_mask=apply_mask, fov_x=fov_x, use_fp16=use_fp16)

    @torch.inference_mode()
    def infer_many(self, images, num_tokens: int = None, resolution_level: int = 9, force_projection: bool = True,
                   apply_mask: bool = True, fov_x: Optional[Number] = None, use_fp16: bool = True) -> List[Dict[str, torch.Tensor]]:
        """`infer()` over a list of images of DIFFERENT sizes (each (3,H,W)): one result dict per image, in order.
        No reference counterpart (the reference processes one shape per call; moge/scripts/infer.py:101 loops over files):
        images are bucketed by shape, the buckets are packed into engine calls of at most `max_chunk_tokens` tokens and every
        call runs the encoder ONCE over the token rows of all its buckets (ragged batching, BASELINE.json configs[2])."""
        return self._infer_many(images, num_tokens=num_tokens, resolution_level=resolution_level,
                                force_projection=force_projection, apply_mask=apply_mask, fov_x=fov_x, use_fp16=use_fp16)
