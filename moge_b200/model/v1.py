"""Drop-in MoGe-1 `MoGeModel`, backed by libmoge_b200.so (hand-written sm_90a CUDA).

Mirrors the public surface of /root/reference/moge/model/v1.py:
  __init__ kwargs incl. mask_threshold and the `trained_area_range` conversion (v1.py:149-172), from_pretrained with a strict
  load (v1.py:214-242), .to/.half/.bfloat16, .device/.dtype, forward(image, num_tokens) -> {'points', 'mask'} (v1.py:269-299),
  infer(image, fov_x, resolution_level, num_tokens, apply_mask, force_projection, use_fp16)
      -> {'points', 'intrinsics', 'depth', 'mask'} (v1.py:301-392),
and, with no reference counterpart, infer_many(images, ...) over a list of images of different sizes (one encoder pass per call).
This file holds the MoGe-1 config, its engine hooks (resized image, output buffers, group struct, post-processing) and the public
signatures; the forward path itself (engine calls, chunking, packing, the bodies of forward / infer / infer_many) is EngineModel's
in _engine.py.  Host logic only: tensor allocation and checkpoint I/O use PyTorch, every arithmetic step runs in the C-ABI library.
"""
from __future__ import annotations

import ctypes as C
import warnings
from numbers import Number
from typing import Dict, List, Optional, Tuple, Union

import torch

from .. import capi
from ..configs import backbone_dims, v1_resized_size
from ._engine import EngineModel


class MoGeModel(EngineModel):
    _strict_load = True             # the reference's from_pretrained loads strictly (v1.py:241)
    _fp32_pass_error = (
        "moge_b200: use_fp16=False (full-fp32 network pass) is not provided; the engine computes with 16-bit "
        "tensor-core operands, fp32 accumulation and fp32 post-processing.  Call infer(..., use_fp16=True).")

    def __init__(self,
                 encoder: str = 'dinov2_vitb14',
                 intermediate_layers: Union[int, List[int]] = 4,
                 dim_proj: int = 512,
                 dim_upsample: List[int] = [256, 128, 128],
                 dim_times_res_block_hidden: int = 1,
                 num_res_blocks: int = 1,
                 remap_output: str = 'linear',
                 res_block_norm: str = 'group_norm',
                 num_tokens_range: Tuple[Number, Number] = [1200, 2500],
                 last_res_blocks: int = 0,
                 last_conv_channels: int = 32,
                 last_conv_size: int = 1,
                 mask_threshold: float = 0.5,
                 **deprecated_kwargs):
        if deprecated_kwargs:
            if 'trained_area_range' in deprecated_kwargs:         # v1.py:169-171
                num_tokens_range = [deprecated_kwargs['trained_area_range'][0] // 14 ** 2,
                                    deprecated_kwargs['trained_area_range'][1] // 14 ** 2]
                del deprecated_kwargs['trained_area_range']
            warnings.warn(f"The following deprecated/invalid arguments are ignored: {deprecated_kwargs}")
        if remap_output not in capi.REMAP:
            raise ValueError(f"Invalid remap output type: {remap_output}")
        backbone_dims(encoder)                       # validates the backbone name
        self.encoder = encoder
        self.remap_output = remap_output
        self.intermediate_layers = intermediate_layers
        self.num_tokens_range = num_tokens_range
        self.mask_threshold = mask_threshold
        self.model_config = dict(encoder=encoder, intermediate_layers=intermediate_layers, dim_proj=dim_proj,
                                 dim_upsample=list(dim_upsample), dim_times_res_block_hidden=dim_times_res_block_hidden,
                                 num_res_blocks=num_res_blocks, remap_output=remap_output, res_block_norm=res_block_norm,
                                 num_tokens_range=list(num_tokens_range), last_res_blocks=last_res_blocks,
                                 last_conv_channels=last_conv_channels, last_conv_size=last_conv_size)
        capi.make_v1_config(self.model_config, capi.F16)     # config errors the host can see, before any weight is loaded
        super().__init__()

    def init_weights(self):
        raise NotImplementedError("training-only (v1.py:244-247)")

    def enable_gradient_checkpointing(self):
        raise NotImplementedError("training-only (v1.py:249-251)")

    def _expected_keys(self) -> List[str]:
        from ..synthetic import v1_expected_keys
        return v1_expected_keys(self.model_config)

    # ------------------------------------------------------------------ engine hooks (EngineModel runs the forward path)
    _group_t = capi.V1Group
    _c_workspace_bytes_groups = "moge_v1_workspace_bytes_groups"
    _c_forward_groups = "moge_v1_forward_groups"
    _output_names = ("points", "mask")

    def _create_engine(self, handle: C.c_void_p):
        cfg = capi.make_v1_config(self.model_config, self._compute_code())
        capi.check(capi.lib().moge_engine_create_v1(C.byref(cfg), self._device.index, C.byref(handle)))

    def _geometry(self, H: int, W: int, num_tokens):
        """((rh, rw) resized image, token rows per image) of an H x W image at `num_tokens`, taken as given (v1.py:272-274)."""
        rh, rw = v1_resized_size(H, W, num_tokens)
        return (rh, rw), (rh // 14) * (rw // 14) + 1

    def _alloc_outputs(self, B: int, H: int, W: int):
        """fp32 (points, raw mask) buffers for B images of H x W."""
        return (torch.empty(B, H, W, 3, dtype=torch.float32, device=self._device),
                torch.empty(B, H, W, dtype=torch.float32, device=self._device))

    def _fill_group(self, g: capi.V1Group, geom, outputs):
        g.rh, g.rw = geom
        g.points, g.mask = (t.data_ptr() for t in outputs)

    def _postprocess(self, outputs, aspect_ratio, fov_x, apply_mask, force_projection) -> Dict[str, torch.Tensor]:
        """The fp32 part of infer() (v1.py:352-380) on the raw forward outputs of one shape group; all on the device."""
        points, mask = outputs
        B, H, W = mask.shape
        dev = self._device
        with torch.cuda.device(dev):
            focal_in = self._focal_in(fov_x, aspect_ratio, B)
            focal = torch.empty(B, dtype=torch.float32, device=dev)
            shift = torch.empty(B, dtype=torch.float32, device=dev)
            depth = torch.empty(B, H, W, dtype=torch.float32, device=dev)
            mask_out = torch.empty(B, H, W, dtype=torch.uint8, device=dev)
            intrinsics = torch.empty(B, 3, 3, dtype=torch.float32, device=dev)
            capi.check(capi.lib().moge_v1_postprocess(
                points.data_ptr(), mask.data_ptr(), float(self.mask_threshold), capi.ptr(focal_in), B, H, W,
                int(bool(force_projection)), int(bool(apply_mask)), depth.data_ptr(), mask_out.data_ptr(), intrinsics.data_ptr(),
                focal.data_ptr(), shift.data_ptr(), capi.current_stream()))
        return {'points': points, 'intrinsics': intrinsics, 'depth': depth, 'mask': mask_out.view(torch.bool)}

    # ------------------------------------------------------------------ public API
    @torch.inference_mode()
    def infer(self,
              image: torch.Tensor,
              fov_x: Union[Number, torch.Tensor] = None,
              resolution_level: int = 9,
              num_tokens: int = None,
              apply_mask: bool = True,
              force_projection: bool = True,
              use_fp16: bool = True) -> Dict[str, torch.Tensor]:
        """Same contract as v1.py:301-392 (note the argument order differs from MoGe-2's infer).  The engine multiplies in 16-bit
        with fp32 accumulation and post-processes in fp32; `use_fp16=False` (a full-fp32 network pass) is not provided."""
        return self._infer(image, num_tokens=num_tokens, resolution_level=resolution_level, force_projection=force_projection,
                           apply_mask=apply_mask, fov_x=fov_x, use_fp16=use_fp16)

    @torch.inference_mode()
    def infer_many(self,
                   images,
                   fov_x: Optional[Number] = None,
                   resolution_level: int = 9,
                   num_tokens: int = None,
                   apply_mask: bool = True,
                   force_projection: bool = True,
                   use_fp16: bool = True) -> List[Dict[str, torch.Tensor]]:
        """`infer()` over a list of images of DIFFERENT sizes (each (3,H,W)), with infer()'s argument order: one result dict per
        image, in order.  No reference counterpart (the reference processes one shape per call): images are bucketed by shape,
        the buckets are packed into engine calls of at most `max_chunk_tokens` tokens and every call runs the encoder ONCE over
        the token rows of all its buckets.  `fov_x` is one horizontal field of view for every image, or None."""
        return self._infer_many(images, num_tokens=num_tokens, resolution_level=resolution_level,
                                force_projection=force_projection, apply_mask=apply_mask, fov_x=fov_x, use_fp16=use_fp16)
