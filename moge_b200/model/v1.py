"""Drop-in MoGe-1 `MoGeModel`, backed by libmoge_b200.so (hand-written sm_90a CUDA).

Mirrors the public surface of /root/reference/moge/model/v1.py:
  __init__ kwargs incl. mask_threshold and the `trained_area_range` conversion (v1.py:149-172), from_pretrained with a strict
  load (v1.py:214-242), .to/.half/.bfloat16, .device/.dtype, forward(image, num_tokens) -> {'points', 'mask'} (v1.py:269-299),
  infer(image, fov_x, resolution_level, num_tokens, apply_mask, force_projection, use_fp16)
      -> {'points', 'intrinsics', 'depth', 'mask'} (v1.py:301-392).
Host logic only: tensor allocation and checkpoint I/O use PyTorch, every arithmetic step runs in the C-ABI library.
"""
from __future__ import annotations

import ctypes as C
import warnings
from numbers import Number
from typing import Dict, List, Tuple, Union

import torch

from .. import capi
from ..configs import backbone_dims, default_num_tokens, v1_resized_size
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

    # ------------------------------------------------------------------ engine
    def _create_engine(self, handle: C.c_void_p):
        cfg = capi.make_v1_config(self.model_config, self._compute_code())
        capi.check(capi.lib().moge_engine_create_v1(C.byref(cfg), self._device.index, C.byref(handle)))

    def _forward_raw(self, image: torch.Tensor, rh: int, rw: int):
        """Engine forward in chunks of at most `max_chunk_tokens` tokens; returns fp32 (points (B,H,W,3), raw mask (B,H,W))."""
        self._ensure_engine()
        image = self._engine_input(image)
        B, _, H, W = image.shape
        dev = self._device
        L = capi.lib()
        with torch.cuda.device(dev):
            points = torch.empty(B, H, W, 3, dtype=torch.float32, device=dev)
            mask = torch.empty(B, H, W, dtype=torch.float32, device=dev)
            for lo, n in self._chunks(B, (rh // 14) * (rw // 14) + 1):
                nbytes = C.c_size_t()
                capi.check(L.moge_v1_workspace_bytes(self._engine, n, H, W, rh, rw, C.byref(nbytes)))
                ws, ws_bytes = self._workspace_for(nbytes.value)
                capi.check(L.moge_v1_forward(
                    self._engine, image[lo:lo + n].data_ptr(), capi.torch_dtype_code(image.dtype), n, H, W, rh, rw, ws, ws_bytes,
                    points[lo:lo + n].data_ptr(), mask[lo:lo + n].data_ptr(), capi.current_stream()))
        return points, mask

    # ------------------------------------------------------------------ public API
    def forward(self, image: torch.Tensor, num_tokens: Union[int, torch.LongTensor]) -> Dict[str, torch.Tensor]:
        if image.dim() != 4 or image.shape[1] != 3:
            raise ValueError(f"image must be (B, 3, H, W), got {tuple(image.shape)}")
        H, W = image.shape[-2:]
        if isinstance(num_tokens, torch.Tensor):
            num_tokens = int(num_tokens.item())
        rh, rw = v1_resized_size(H, W, num_tokens)
        points, mask = self._forward_raw(image, rh, rw)
        return {'points': points, 'mask': mask}

    __call__ = forward

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
        self._check_use_fp16(use_fp16)
        omit_batch_dim = image.dim() == 3
        if omit_batch_dim:
            image = image.unsqueeze(0)
        H, W = image.shape[-2:]
        aspect_ratio = W / H
        if num_tokens is None:
            num_tokens = default_num_tokens(self.num_tokens_range, resolution_level)
        rh, rw = v1_resized_size(H, W, int(num_tokens))
        points, mask = self._forward_raw(image, rh, rw)
        B = points.shape[0]
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
        ret = {'points': points, 'intrinsics': intrinsics, 'depth': depth, 'mask': mask_out.view(torch.bool)}
        if omit_batch_dim:
            ret = {k: v.squeeze(0) for k, v in ret.items()}
        return ret
