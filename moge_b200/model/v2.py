"""Drop-in `MoGeModel` for the MoGe-2 inference hot path, backed by libmoge_b200.so (hand-written sm_90a CUDA).

Mirrors the public surface of /root/reference/moge/model/v2.py:
  __init__ kwargs (v2.py:30-57), from_pretrained (v2.py:76-107), .to/.eval/.half, .device/.dtype (v2.py:59-65),
  forward(image, num_tokens) -> {'points','normal','mask','metric_scale'} (v2.py:138-192),
  infer(image, num_tokens, resolution_level, force_projection, apply_mask, fov_x, use_fp16)
      -> {'points','intrinsics','depth','mask','normal'} (v2.py:194-303).
This file is host logic only: tensor allocation and checkpoint I/O use PyTorch, every arithmetic step of the path
runs in the C-ABI library.  There is no CPU / eager fallback.
"""
from __future__ import annotations

import warnings
from numbers import Number
from typing import Any, Dict, List, Optional, Union

import ctypes as C
import torch

from .. import capi
from ..configs import backbone_dims, default_num_tokens, token_grid
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

    # ------------------------------------------------------------------ engine
    def _create_engine(self, handle: C.c_void_p):
        cfg = capi.make_config(self.model_config, self._compute_code())
        capi.check(capi.lib().moge_engine_create(C.byref(cfg), self._device.index, C.byref(handle)))

    def _alloc_outputs(self, B: int, H: int, W: int):
        """fp32 (points, normal, mask_prob, metric_scale) buffers for B images of H x W, absent heads as None."""
        dev = self._device
        points = torch.empty(B, H, W, 3, dtype=torch.float32, device=dev) if hasattr(self, "points_head") else None
        normal = torch.empty(B, H, W, 3, dtype=torch.float32, device=dev) if hasattr(self, "normal_head") else None
        mask = torch.empty(B, H, W, dtype=torch.float32, device=dev) if hasattr(self, "mask_head") else None
        scale = torch.empty(B, dtype=torch.float32, device=dev) if hasattr(self, "scale_head") else None
        return points, normal, mask, scale

    def _forward_raw(self, image: torch.Tensor, h: int, w: int):
        """Runs the engine forward; returns fp32 (points, normal, mask_prob, metric_scale), absent heads as None."""
        self._ensure_engine()
        image = self._engine_input(image)
        B, _, H, W = image.shape
        L = capi.lib()
        with torch.cuda.device(self._device):
            outs = self._alloc_outputs(B, H, W)
            for lo, n in self._chunks(B, h * w + 1):
                nbytes = C.c_size_t()
                capi.check(L.moge_engine_workspace_bytes(self._engine, n, H, W, h, w, C.byref(nbytes)))
                ws, ws_bytes = self._workspace_for(nbytes.value)
                points, normal, mask, scale = (None if t is None else t[lo:lo + n] for t in outs)
                capi.check(L.moge_engine_forward(
                    self._engine, image[lo:lo + n].data_ptr(), capi.torch_dtype_code(image.dtype), n, H, W, h, w, ws, ws_bytes,
                    capi.ptr(points), capi.ptr(normal), capi.ptr(mask), capi.ptr(scale), capi.current_stream()))
        return outs

    def _forward_groups(self, groups):
        """ONE engine call over several shape groups: `groups` = [(image (B,3,H,W), h, w)].  The encoder runs once over the
        packed token rows of all groups (moge_engine_forward_groups).  Returns [(points, normal, mask_prob, metric_scale)]."""
        self._ensure_engine()
        n = len(groups)
        arr = (capi.Group * n)()
        keep, outs = [], []
        with torch.cuda.device(self._device):
            for i, (image, h, w) in enumerate(groups):
                image = self._engine_input(image)
                B, _, H, W = image.shape
                points, normal, mask, scale = self._alloc_outputs(B, H, W)
                g = arr[i]
                g.image, g.image_dtype = image.data_ptr(), capi.torch_dtype_code(image.dtype)
                g.B, g.H, g.W, g.h, g.w = B, H, W, h, w
                g.points, g.normal, g.mask_prob, g.metric_scale = capi.ptr(points), capi.ptr(normal), capi.ptr(mask), capi.ptr(scale)
                keep.append(image)
                outs.append((points, normal, mask, scale))
            nbytes = C.c_size_t()
            capi.check(capi.lib().moge_engine_workspace_bytes_groups(self._engine, arr, n, C.byref(nbytes)))
            ws, ws_bytes = self._workspace_for(nbytes.value)
            capi.check(capi.lib().moge_engine_forward_groups(self._engine, arr, n, ws, ws_bytes, capi.current_stream()))
        return outs

    @torch.inference_mode()
    def infer_many(self, images, num_tokens: int = None, resolution_level: int = 9, force_projection: bool = True,
                   apply_mask: bool = True, fov_x: Optional[Number] = None, use_fp16: bool = True) -> List[Dict[str, torch.Tensor]]:
        """`infer()` over a list of images of DIFFERENT sizes (each (3,H,W)): one result dict per image, in order.
        No reference counterpart (the reference processes one shape per call; moge/scripts/infer.py:101 loops over files):
        images are bucketed by shape, the buckets are packed into engine calls of at most `max_chunk_tokens` tokens and every
        call runs the encoder ONCE over the token rows of all its buckets (ragged batching, BASELINE.json configs[2])."""
        self._check_use_fp16(use_fp16)
        if num_tokens is None:
            num_tokens = default_num_tokens(self.num_tokens_range, resolution_level)

        def geometry(H, W):
            h, w = token_grid(H, W, int(num_tokens))
            return (h, w), h * w + 1

        calls = self._pack_calls(images, geometry)
        results: List[Optional[Dict[str, torch.Tensor]]] = [None] * len(images)
        for call in calls:
            groups = [(torch.stack([images[i].to(self._device) for i in idx]), h, w) for (H, W, (h, w), idx) in call]
            outs = self._forward_groups(groups)
            for (H, W, _, idx), (points, normal, mask, scale) in zip(call, outs):
                ret = self._postprocess(points, normal, mask, scale, W / H, force_projection, apply_mask, fov_x)
                for j, i in enumerate(idx):
                    results[i] = {k: v[j] for k, v in ret.items()}
        return results

    # ------------------------------------------------------------------ public API
    def forward(self, image: torch.Tensor, num_tokens: Union[int, torch.LongTensor]) -> Dict[str, torch.Tensor]:
        if image.dim() != 4 or image.shape[1] != 3:
            raise ValueError(f"image must be (B, 3, H, W), got {tuple(image.shape)}")
        H, W = image.shape[-2:]
        if isinstance(num_tokens, torch.Tensor):
            num_tokens = int(num_tokens.item())
        h, w = token_grid(H, W, int(num_tokens))
        points, normal, mask, scale = self._forward_raw(image, h, w)
        out = {'points': points, 'normal': normal, 'mask': mask, 'metric_scale': scale}
        return {k: v for k, v in out.items() if v is not None}

    __call__ = forward

    def _postprocess(self, points, normal, mask, metric_scale, aspect_ratio, force_projection, apply_mask, fov_x):
        """K18 + K19 of infer() (v2.py:246-298) on the raw forward outputs of one shape group; all on the device."""
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
        self._check_use_fp16(use_fp16)
        omit_batch_dim = image.dim() == 3
        if omit_batch_dim:
            image = image.unsqueeze(0)
        H, W = image.shape[-2:]
        aspect_ratio = W / H
        if num_tokens is None:
            num_tokens = default_num_tokens(self.num_tokens_range, resolution_level)
        h, w = token_grid(H, W, int(num_tokens))
        points, normal, mask, metric_scale = self._forward_raw(image, h, w)
        ret = self._postprocess(points, normal, mask, metric_scale, aspect_ratio, force_projection, apply_mask, fov_x)
        if omit_batch_dim:
            ret = {k: v.squeeze(0) for k, v in ret.items()}
        return ret
