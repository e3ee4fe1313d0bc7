"""Host plumbing shared by the drop-in MoGe-2 and MoGe-1 models (v2.py, v1.py): the nn.Module-like surface, checkpoint
loading, the engine handle with its weight upload, the activation workspace and the batch chunking.
Host logic only: every arithmetic step runs in the C-ABI library.
"""
from __future__ import annotations

import ctypes as C
from pathlib import Path
from typing import IO, Any, Dict, List, Optional, Tuple, Union

import torch

from .. import capi


class EngineModel:
    """Base of both drop-in `MoGeModel` classes.  A subclass supplies `_expected_keys()` (the checkpoint keys of its config),
    `_create_engine(handle)` (its config struct and create call, which sets the C handle), `_strict_load` (how
    `from_pretrained` loads) and `_fp32_pass_error` (why `use_fp16=False` is refused)."""

    def __init__(self):
        self._state: Dict[str, torch.Tensor] = {}
        self._device = torch.device("cpu")
        self._param_dtype = torch.float32
        self._engine = None                 # C handle
        self._workspace: Optional[torch.Tensor] = None
        self.training = False
        self.max_chunk_tokens = 48 * 1370          # images per engine call = max_chunk_tokens // (tokens per image)

    # ------------------------------------------------------------------ nn.Module-like plumbing
    @property
    def device(self) -> torch.device:
        return self._device

    @property
    def dtype(self) -> torch.dtype:
        return self._param_dtype

    def eval(self):
        self.training = False
        return self

    def train(self, mode: bool = True):
        if mode:
            raise NotImplementedError("moge_b200 is an inference engine")
        return self

    def requires_grad_(self, flag: bool = False):
        return self

    def state_dict(self) -> Dict[str, torch.Tensor]:
        return dict(self._state)

    def load_state_dict(self, state_dict: Dict[str, torch.Tensor], strict: bool = True):
        """nn.Module.load_state_dict semantics: returns the (missing_keys, unexpected_keys) report; strict=True raises
        RuntimeError when either list is non-empty."""
        from torch.nn.modules.module import _IncompatibleKeys
        want = self._expected_keys()
        wanted = set(want)
        missing = [k for k in want if k not in state_dict]
        unexpected = [k for k in state_dict.keys() if k not in wanted]
        if strict and (missing or unexpected):
            raise RuntimeError("Error(s) in loading state_dict for MoGeModel:\n\tMissing key(s): "
                               f"{missing}\n\tUnexpected key(s): {unexpected}")
        self._state = {k: v.detach() for k, v in state_dict.items()}
        self._drop_engine()
        return _IncompatibleKeys(missing, unexpected)

    def to(self, *args, **kwargs):
        device = kwargs.get("device")
        dtype = kwargs.get("dtype")
        for a in args:
            if isinstance(a, torch.dtype):
                dtype = a
            elif a is not None:
                device = a
        if dtype is not None:
            self._set_dtype(dtype)
        if device is not None:
            device = torch.device(device)
            if device.type == "cuda" and device.index is None:
                device = torch.device("cuda", torch.cuda.current_device())
            if device != self._device:
                self._device = device
                self._drop_engine()
        return self

    def cuda(self, device=None):
        return self.to(torch.device("cuda", device if device is not None else torch.cuda.current_device()))

    def cpu(self):
        return self.to("cpu")

    def half(self):
        return self._set_dtype(torch.float16)

    def bfloat16(self):
        return self._set_dtype(torch.bfloat16)

    def float(self):
        return self._set_dtype(torch.float32)

    def _set_dtype(self, dtype: torch.dtype):
        if dtype not in (torch.float32, torch.float16, torch.bfloat16):
            raise TypeError(f"unsupported dtype {dtype}")
        if dtype != self._param_dtype:
            self._param_dtype = dtype
            self._drop_engine()
        return self

    def _drop_engine(self):
        if self._engine is not None:
            capi.lib().moge_engine_destroy(self._engine)
        self._engine = None
        self._workspace = None

    def __del__(self):
        try:
            self._drop_engine()
        except Exception:
            pass

    # ------------------------------------------------------------------ checkpoint
    @classmethod
    def from_pretrained(cls, pretrained_model_name_or_path: Union[str, Path, IO[bytes]],
                        model_kwargs: Optional[Dict[str, Any]] = None, **hf_kwargs):
        """Load a `{'model_config', 'model'}` checkpoint like the reference classes do (local path, else HF hub)."""
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
        model.load_state_dict(checkpoint['model'], strict=cls._strict_load)
        return model

    # ------------------------------------------------------------------ engine
    def _compute_code(self) -> int:
        return capi.BF16 if self._param_dtype == torch.bfloat16 else capi.F16

    def _ensure_engine(self):
        if self._engine is not None:
            return
        if self._device.type != "cuda":
            raise capi.MogeError("moge_b200 has no CPU path: move the model to an H100 with .to('cuda') first")
        if not self._state:
            raise capi.MogeError("no weights loaded (use from_pretrained or load_state_dict)")
        L = capi.lib()
        handle = C.c_void_p()
        with torch.cuda.device(self._device):
            self._create_engine(handle)
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

    def _workspace_for(self, nbytes: int) -> Tuple[int, int]:
        """(1024-byte aligned pointer, usable bytes) of a workspace that holds the `nbytes` the engine asked for.  The buffer only
        grows: the engine keys its cached plans on the workspace pointer and size, so calls whose request fits reuse their plans."""
        need = nbytes + 1024
        if self._workspace is None or self._workspace.numel() < need:
            self._workspace = None
            self._workspace = torch.empty(need, dtype=torch.uint8, device=self._device)
        base = self._workspace.data_ptr()
        aligned = (base + 1023) & ~1023
        return aligned, self._workspace.numel() - (aligned - base)

    def _chunks(self, B: int, tokens_per_image: int) -> List[Tuple[int, int]]:
        """(first image, images) of each engine call over B images.  Images are independent: large batches run as chunks of at
        most `max_chunk_tokens` tokens so that the activation workspace stays bounded (ViT-L, 1370 tokens/image: 32 images
        ~ 21 GB)."""
        chunk = max(1, min(B, self.max_chunk_tokens // tokens_per_image))
        return [(lo, min(chunk, B - lo)) for lo in range(0, B, chunk)]

    def _engine_input(self, image: torch.Tensor) -> torch.Tensor:
        """`image` as the engine reads it: on the model's device, fp32 / fp16 / bf16, contiguous."""
        image = image.to(self._device)
        if image.dtype not in (torch.float32, torch.float16, torch.bfloat16):
            image = image.float()
        return image.contiguous()

    def _focal_in(self, fov_x: Optional[Union[float, torch.Tensor]], aspect_ratio: float, B: int) -> Optional[torch.Tensor]:
        """The (B,) fp32 focal (in units of the half-diagonal) that a horizontal field of view `fov_x` in degrees fixes, per image;
        None without `fov_x`."""
        if fov_x is None:
            return None
        fx_t = torch.as_tensor(fov_x, device=self._device, dtype=torch.float32)
        focal_in = aspect_ratio / (1 + aspect_ratio ** 2) ** 0.5 / torch.tan(torch.deg2rad(fx_t / 2))
        if focal_in.ndim == 0:
            focal_in = focal_in[None].expand(B)
        return focal_in.contiguous()

    def _check_use_fp16(self, use_fp16: bool):
        if not use_fp16:
            raise NotImplementedError(self._fp32_pass_error)

    # ------------------------------------------------------------------ introspection
    def engine_ops(self):
        """[(kernel name, algorithmic flops, algorithmic HBM bytes)] of the launch list of the most recent forward."""
        L = capi.lib()
        n = C.c_int()
        capi.check(L.moge_engine_num_ops(self._engine, C.byref(n)))
        out = []
        buf = C.create_string_buffer(96)
        fl, by = C.c_double(), C.c_double()
        for i in range(n.value):
            capi.check(L.moge_engine_op_info(self._engine, i, buf, 96, C.byref(fl), C.byref(by)))
            out.append((buf.value.decode(), fl.value, by.value))
        return out

    def engine_profile(self):
        """Replays the most recent forward with a CUDA-event pair around every launch; returns ms per launch."""
        L = capi.lib()
        n = C.c_int()
        capi.check(L.moge_engine_num_ops(self._engine, C.byref(n)))
        ms = (C.c_float * n.value)()
        with torch.cuda.device(self._device):
            capi.check(L.moge_engine_profile(self._engine, ms, n.value, capi.current_stream()))
        return list(ms)
