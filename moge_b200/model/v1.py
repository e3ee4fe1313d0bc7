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
from pathlib import Path
from typing import IO, Any, Dict, List, Optional, Tuple, Union

import torch

from .. import capi
from ..configs import backbone_dims, v1_resized_size
from . import v2 as _v2


class MoGeModel:
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
        self._state: Dict[str, torch.Tensor] = {}
        self._device = torch.device("cpu")
        self._param_dtype = torch.float32
        self._engine = None
        self._workspace: Optional[torch.Tensor] = None
        self.training = False
        self.max_chunk_tokens = 48 * 1370          # images per engine call = max_chunk_tokens // (tokens per image)

    # nn.Module-like plumbing: the same engine-handle / dtype / device bookkeeping as the MoGe-2 class
    device = _v2.MoGeModel.device
    dtype = _v2.MoGeModel.dtype
    eval = _v2.MoGeModel.eval
    train = _v2.MoGeModel.train
    requires_grad_ = _v2.MoGeModel.requires_grad_
    state_dict = _v2.MoGeModel.state_dict
    to = _v2.MoGeModel.to
    cuda = _v2.MoGeModel.cuda
    cpu = _v2.MoGeModel.cpu
    half = _v2.MoGeModel.half
    bfloat16 = _v2.MoGeModel.bfloat16
    float = _v2.MoGeModel.float
    _set_dtype = _v2.MoGeModel._set_dtype
    _drop_engine = _v2.MoGeModel._drop_engine
    __del__ = _v2.MoGeModel.__del__
    _compute_code = _v2.MoGeModel._compute_code
    engine_ops = _v2.MoGeModel.engine_ops
    engine_profile = _v2.MoGeModel.engine_profile

    def init_weights(self):
        raise NotImplementedError("training-only (v1.py:244-247)")

    def enable_gradient_checkpointing(self):
        raise NotImplementedError("training-only (v1.py:249-251)")

    def load_state_dict(self, state_dict: Dict[str, torch.Tensor], strict: bool = True):
        """nn.Module.load_state_dict semantics; from_pretrained loads strictly, as v1.py:241 does."""
        from torch.nn.modules.module import _IncompatibleKeys
        from ..synthetic import v1_expected_keys
        want = v1_expected_keys(self.model_config)
        wanted = set(want)
        missing = [k for k in want if k not in state_dict]
        unexpected = [k for k in state_dict.keys() if k not in wanted]
        if strict and (missing or unexpected):
            raise RuntimeError("Error(s) in loading state_dict for MoGeModel:\n\tMissing key(s): "
                               f"{missing}\n\tUnexpected key(s): {unexpected}")
        self._state = {k: v.detach() for k, v in state_dict.items()}
        self._drop_engine()
        return _IncompatibleKeys(missing, unexpected)

    @classmethod
    def from_pretrained(cls, pretrained_model_name_or_path: Union[str, Path, IO[bytes]],
                        model_kwargs: Optional[Dict[str, Any]] = None, **hf_kwargs) -> 'MoGeModel':
        """Load `{'model_config', 'model'}` checkpoints like v1.py:214-242 (local path, else HF hub), strictly."""
        if Path(pretrained_model_name_or_path).exists():
            checkpoint_path = pretrained_model_name_or_path
        else:
            from huggingface_hub import hf_hub_download
            checkpoint_path = hf_hub_download(repo_id=pretrained_model_name_or_path, repo_type="model",
                                              filename="model.pt", **hf_kwargs)
        checkpoint = torch.load(checkpoint_path, map_location='cpu', weights_only=True)
        model_config = checkpoint['model_config']
        if model_kwargs is not None:
            model_config.update(model_kwargs)
        model = cls(**model_config)
        model.load_state_dict(checkpoint['model'])
        return model

    # ------------------------------------------------------------------ engine
    def _ensure_engine(self):
        if self._engine is not None:
            return
        if self._device.type != "cuda":
            raise capi.MogeError("moge_b200 has no CPU path: move the model to an H100 with .to('cuda') first")
        if not self._state:
            raise capi.MogeError("no weights loaded (use from_pretrained or load_state_dict)")
        L = capi.lib()
        cfg = capi.make_v1_config(self.model_config, self._compute_code())
        handle = C.c_void_p()
        with torch.cuda.device(self._device):
            capi.check(L.moge_engine_create_v1(C.byref(cfg), self._device.index, C.byref(handle)))
            stream = capi.current_stream()
            try:
                for key, t in self._state.items():
                    if not t.is_floating_point():
                        continue
                    d = t.to(self._device).contiguous()
                    if d.dtype not in (torch.float32, torch.float16, torch.bfloat16):
                        d = d.float()
                    shape = (C.c_int64 * max(d.dim(), 1))(*d.shape)
                    capi.check(L.moge_engine_set_weight(handle, key.encode(), d.data_ptr(), shape, d.dim(),
                                                        capi.torch_dtype_code(d.dtype), stream))
                    torch.cuda.current_stream().synchronize()
                capi.check(L.moge_engine_finalize(handle, stream))
            except Exception:
                L.moge_engine_destroy(handle)
                raise
        self._engine = handle

    def _get_workspace(self, B, H, W, rh, rw) -> torch.Tensor:
        n = C.c_size_t()
        capi.check(capi.lib().moge_v1_workspace_bytes(self._engine, B, H, W, rh, rw, C.byref(n)))
        need = n.value + 1024
        if self._workspace is None or self._workspace.numel() < need:
            self._workspace = None
            self._workspace = torch.empty(need, dtype=torch.uint8, device=self._device)
        return self._workspace

    def _forward_raw(self, image: torch.Tensor, rh: int, rw: int):
        """Engine forward in chunks of at most `max_chunk_tokens` tokens; returns fp32 (points (B,H,W,3), raw mask (B,H,W))."""
        self._ensure_engine()
        B, _, H, W = image.shape
        image = image.to(self._device)
        if image.dtype not in (torch.float32, torch.float16, torch.bfloat16):
            image = image.float()
        image = image.contiguous()
        dev = self._device
        chunk = max(1, min(B, self.max_chunk_tokens // ((rh // 14) * (rw // 14) + 1)))
        with torch.cuda.device(dev):
            points = torch.empty(B, H, W, 3, dtype=torch.float32, device=dev)
            mask = torch.empty(B, H, W, dtype=torch.float32, device=dev)
            for lo in range(0, B, chunk):
                n = min(chunk, B - lo)
                ws = self._get_workspace(n, H, W, rh, rw)
                base = ws.data_ptr()
                aligned = (base + 1023) & ~1023
                capi.check(capi.lib().moge_v1_forward(
                    self._engine, image[lo:lo + n].data_ptr(), capi.torch_dtype_code(image.dtype), n, H, W, rh, rw, aligned,
                    ws.numel() - (aligned - base), points[lo:lo + n].data_ptr(), mask[lo:lo + n].data_ptr(), capi.current_stream()))
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
        if not use_fp16:
            raise NotImplementedError(
                "moge_b200: use_fp16=False (full-fp32 network pass) is not provided; the engine computes with 16-bit "
                "tensor-core operands, fp32 accumulation and fp32 post-processing.  Call infer(..., use_fp16=True).")
        if image.dim() == 3:
            omit_batch_dim = True
            image = image.unsqueeze(0)
        else:
            omit_batch_dim = False
        H, W = image.shape[-2:]
        aspect_ratio = W / H
        if num_tokens is None:
            min_tokens, max_tokens = self.num_tokens_range
            num_tokens = int(min_tokens + (resolution_level / 9) * (max_tokens - min_tokens))
        rh, rw = v1_resized_size(H, W, int(num_tokens))
        points, mask = self._forward_raw(image, rh, rw)
        B = points.shape[0]
        dev = self._device
        with torch.cuda.device(dev):
            focal_in = None
            if fov_x is not None:
                fx_t = torch.as_tensor(fov_x, device=dev, dtype=torch.float32)
                focal_in = aspect_ratio / (1 + aspect_ratio ** 2) ** 0.5 / torch.tan(torch.deg2rad(fx_t / 2))
                if focal_in.ndim == 0:
                    focal_in = focal_in[None].expand(B)
                focal_in = focal_in.contiguous()
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
