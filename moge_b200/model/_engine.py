"""Host code shared by the drop-in MoGe-2 and MoGe-1 models (v2.py, v1.py): the nn.Module-like surface, checkpoint loading,
the engine handle with its weight upload, the activation workspace, and the whole forward path: the engine call over an array
of shape groups, the chunked single-shape forward, the mixed-shape packing, and the bodies of `forward`, `infer` and
`infer_many`.  The model files keep their configs, the small per-model hooks and the public signatures.
Host logic only: every arithmetic step runs in the C-ABI library.
"""
from __future__ import annotations

import ctypes as C
from pathlib import Path
from typing import IO, Any, Callable, Dict, List, Optional, Tuple, Union

import torch

from .. import capi
from ..configs import default_num_tokens


class EngineModel:
    """Base of both drop-in `MoGeModel` classes.  A subclass supplies
      `_expected_keys()` (the checkpoint keys of its config), `_create_engine(handle)` (its config struct and create call, which
      sets the C handle), `_strict_load` (how `from_pretrained` loads) and `_fp32_pass_error` (why `use_fp16=False` is refused);
      `_group_t`, `_c_workspace_bytes_groups`, `_c_forward_groups` (its C group struct and the names of its two group entry points);
      `_geometry(H, W, num_tokens)` -> (geom, token rows per image), geom being what one group struct carries besides B, H, W;
      `_alloc_outputs(B, H, W)` (its fp32 output buffers, absent heads None), `_fill_group(g, geom, outputs)`, `_output_names`
      (the keys `forward` returns them under) and `_postprocess(outputs, aspect_ratio, fov_x, apply_mask, force_projection)`."""

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
            raise RuntimeError(f"Error(s) in loading state_dict for {type(self).__name__}:\n\tMissing key(s): "
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

    def _pack_calls(self, images, geometry: Callable[[int, int], Tuple[Tuple[int, int], int]],
                    max_units: Optional[int] = None) -> List[List[tuple]]:
        """The engine calls of `infer_many` over `images` (each (3, H, W)), as lists of units (H, W, geom, indices).  Images are
        bucketed by shape and dtype; `geometry(H, W)` gives a bucket's (geom, token rows per image), geom being what the model's
        engine call takes per group.  Each bucket is chunked like a batch (`_chunks`), and the chunks are packed largest first into
        calls of at most `max_chunk_tokens` tokens (a unit larger than that is a call of its own) and, given `max_units`, at most
        that many units (shape groups).  Raises ValueError, before anything touches a device, on an element that is not
        (3, H, W)."""
        buckets: Dict[tuple, List[int]] = {}
        for i, im in enumerate(images):
            if im.dim() != 3 or im.shape[0] != 3:
                raise ValueError(f"images[{i}] must be (3, H, W), got {tuple(im.shape)}")
            buckets.setdefault((int(im.shape[1]), int(im.shape[2]), im.dtype), []).append(i)
        units = []
        for (H, W, _), idx in buckets.items():
            geom, tokens = geometry(H, W)
            for lo, n in self._chunks(len(idx), tokens):
                units.append((n * tokens, (H, W, geom, idx[lo:lo + n])))
        units.sort(key=lambda u: -u[0])
        calls, cur, cur_tok = [], [], 0
        for tok, unit in units:
            if cur and (cur_tok + tok > self.max_chunk_tokens or len(cur) == max_units):
                calls.append(cur)
                cur, cur_tok = [], 0
            cur.append(unit)
            cur_tok += tok
        if cur:
            calls.append(cur)
        return calls

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

    # ------------------------------------------------------------------ forward path
    def _engine_call(self, groups) -> None:
        """ONE engine call over shape groups [(engine-input image (B,3,H,W), geom, outputs)], `outputs` being caller-allocated
        buffers or views of them (`_alloc_outputs`).  The encoder runs once over the packed token rows of all groups, and each
        group's decoder writes its outputs."""
        self._ensure_engine()
        arr = (self._group_t * len(groups))()
        for g, (image, geom, outputs) in zip(arr, groups):
            g.image, g.image_dtype = image.data_ptr(), capi.torch_dtype_code(image.dtype)
            g.B, g.H, g.W = image.shape[0], image.shape[2], image.shape[3]
            self._fill_group(g, geom, outputs)
        L = capi.lib()
        with torch.cuda.device(self._device):
            nbytes = C.c_size_t()
            capi.check(getattr(L, self._c_workspace_bytes_groups)(self._engine, arr, len(groups), C.byref(nbytes)))
            ws, ws_bytes = self._workspace_for(nbytes.value)
            capi.check(getattr(L, self._c_forward_groups)(self._engine, arr, len(groups), ws, ws_bytes, capi.current_stream()))

    def _forward_groups(self, groups):
        """ONE engine call over shape groups [(image (B,3,H,W), *geom)], into newly allocated outputs; returns them per group."""
        bound = []
        for image, *geom in groups:
            image = self._engine_input(image)
            bound.append((image, geom, self._alloc_outputs(image.shape[0], image.shape[2], image.shape[3])))
        self._engine_call(bound)
        return [outputs for _, _, outputs in bound]

    def _forward_chunks(self, image: torch.Tensor, geom, tokens_per_image: int):
        """The forward of a (B,3,H,W) batch of one shape: the full-batch outputs, written by one engine call per chunk of
        `_chunks`, each over one group of the chunk's images and output views."""
        image = self._engine_input(image)
        B, _, H, W = image.shape
        outputs = self._alloc_outputs(B, H, W)
        for lo, n in self._chunks(B, tokens_per_image):
            views = tuple(None if t is None else t[lo:lo + n] for t in outputs)
            self._engine_call([(image[lo:lo + n], geom, views)])
        return outputs

    def forward(self, image: torch.Tensor, num_tokens: Union[int, torch.LongTensor]) -> Dict[str, torch.Tensor]:
        if image.dim() != 4 or image.shape[1] != 3:
            raise ValueError(f"image must be (B, 3, H, W), got {tuple(image.shape)}")
        H, W = image.shape[-2:]
        if isinstance(num_tokens, torch.Tensor):
            num_tokens = int(num_tokens.item())
        outputs = self._forward_chunks(image, *self._geometry(H, W, num_tokens))
        return {k: v for k, v in zip(self._output_names, outputs) if v is not None}

    __call__ = forward

    def _infer(self, image, *, num_tokens, resolution_level, force_projection, apply_mask, fov_x, use_fp16):
        """The body of both models' `infer`."""
        self._check_use_fp16(use_fp16)
        omit_batch_dim = image.dim() == 3
        if omit_batch_dim:
            image = image.unsqueeze(0)
        H, W = image.shape[-2:]
        if num_tokens is None:
            num_tokens = default_num_tokens(self.num_tokens_range, resolution_level)
        outputs = self._forward_chunks(image, *self._geometry(H, W, int(num_tokens)))
        ret = self._postprocess(outputs, W / H, fov_x, apply_mask, force_projection)
        if omit_batch_dim:
            ret = {k: v.squeeze(0) for k, v in ret.items()}
        return ret

    def _infer_many(self, images, *, num_tokens, resolution_level, force_projection, apply_mask, fov_x,
                    use_fp16) -> List[Dict[str, torch.Tensor]]:
        """The body of both models' `infer_many`: the images bucketed and packed into engine calls (`_pack_calls`, then
        `_forward_groups`), each call's groups post-processed, and the per-image results returned in input order."""
        self._check_use_fp16(use_fp16)
        if num_tokens is None:
            num_tokens = default_num_tokens(self.num_tokens_range, resolution_level)
        calls = self._pack_calls(images, lambda H, W: self._geometry(H, W, int(num_tokens)))
        results: List[Optional[Dict[str, torch.Tensor]]] = [None] * len(images)
        for call in calls:
            outs = self._forward_groups([(torch.stack([images[i].to(self._device) for i in idx]), *geom)
                                         for (H, W, geom, idx) in call])
            for (H, W, _, idx), outputs in zip(call, outs):
                ret = self._postprocess(outputs, W / H, fov_x, apply_mask, force_projection)
                for j, i in enumerate(idx):
                    results[i] = {k: v[j] for k, v in ret.items()}
        return results

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
