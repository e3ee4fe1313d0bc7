"""Drop-in DINOv2 backbone, backed by libmoge_b200.so: the MoGe engines' encoder kernels (folded-LayerNorm wgmma linears,
the warp-specialised attention, the bicubic pos-embed table) on their own, with sm_90a kernels for the two ends (dinov2.cu).

Mirrors the public surface of the reference's moge/model/dinov2 package:
  DinoVisionTransformer (models/vision_transformer.py:44-340): get_intermediate_layers, forward_features, forward, and the
      nn.Module-like plumbing of the MoGe models (.to / .half / .bfloat16, state_dict, load_state_dict); and, for lists of
      (3, H, W) images of mixed shapes, get_intermediate_layers_many, forward_features_many and forward_many, one encoder pass
      per engine call over the token rows of every shape (the reference's forward_features_list needs xformers and stays
      refused);
  vit_small / vit_base / vit_large (vision_transformer.py:351-390);
  dinov2_vits14 / dinov2_vitb14 / dinov2_vitl14 (hub/backbones.py:64-82), pretrained=False only: there is no download, load a
      state dict instead.
Registers (the *_reg constructors), ViT-g / SwiGLU, iBOT masks and training mode are not provided and raise with the reason.
The input is what the reference's forward takes: an image that is already normalised, H and W multiples of 14.  Host logic only:
every arithmetic step runs in the C-ABI library; there is no CPU / eager fallback.
"""
from __future__ import annotations

import ctypes as C
from typing import Dict, List, Optional, Sequence, Tuple, Union

import torch

from . import capi
from .model._engine import EngineModel

_BLOCK_KEYS = ("norm1.weight", "norm1.bias", "attn.qkv.weight", "attn.qkv.bias", "attn.proj.weight", "attn.proj.bias",
               "ls1.gamma", "norm2.weight", "norm2.bias", "mlp.fc1.weight", "mlp.fc1.bias", "mlp.fc2.weight", "mlp.fc2.bias",
               "ls2.gamma")


def _unsupported(what: str):
    return NotImplementedError(f"moge_b200 DINOv2: {what}")


class DinoVisionTransformer(EngineModel):
    """The reference's DinoVisionTransformer (vision_transformer.py:44) for the configurations the engine covers: patch 14, no
    registers, the GELU MLP, LayerScale, a 518-pixel (37 x 37) position grid, bicubic pos-embed interpolation with offset 0.1."""
    _strict_load = True
    _fp32_pass_error = "moge_b200 DINOv2: the engine computes with 16-bit tensor-core operands and fp32 accumulation"

    def __init__(self, img_size=224, patch_size=16, in_chans=3, embed_dim=768, depth=12, num_heads=12, mlp_ratio=4.0,
                 qkv_bias=True, ffn_bias=True, proj_bias=True, drop_path_rate=0.0, drop_path_uniform=False, init_values=None,
                 embed_layer=None, act_layer=None, block_fn=None, ffn_layer="mlp", block_chunks=1, num_register_tokens=0,
                 interpolate_antialias=False, interpolate_offset=0.1):
        super().__init__()
        if ffn_layer not in capi.DINO_FFN:
            raise NotImplementedError(f"ffn_layer {ffn_layer!r}")          # vision_transformer.py:135
        if capi.DINO_FFN[ffn_layer] != capi.DINO_FFN["mlp"]:
            raise _unsupported(f"ffn_layer={ffn_layer!r} (SwiGLU / identity FFNs, as in ViT-g) is not provided: the encoder kernels "
                               "run the GELU MLP only")
        if num_register_tokens:
            raise _unsupported(f"{num_register_tokens} register tokens are not provided: the engine's rows are the class token and "
                               "the patch tokens only")
        if patch_size != 14:
            raise _unsupported(f"patch_size={patch_size} is not provided (14 only)")
        if img_size != 518:
            raise _unsupported(f"img_size={img_size} is not provided: the position embedding must be the 37 x 37 grid of 518")
        if in_chans != 3 or mlp_ratio != 4 or not (qkv_bias and ffn_bias and proj_bias):
            raise _unsupported("only 3 input channels, mlp_ratio 4 and biased linears are provided")
        if init_values is None or init_values == 0:
            raise _unsupported("a backbone without LayerScale (init_values None or 0) is not provided")
        if block_chunks != 0:
            raise _unsupported(f"block_chunks={block_chunks} is not provided (0, the hub constructors' setting)")
        if interpolate_antialias or interpolate_offset != 0.1:
            raise _unsupported("pos-embed interpolation with antialias or an offset other than 0.1 is not provided")
        if embed_dim % 128 or embed_dim > 1024 or num_heads * 64 != embed_dim:
            raise _unsupported(f"embed_dim={embed_dim}, num_heads={num_heads}: the encoder takes head_dim 64 and embed_dim a "
                               "multiple of 128 up to 1024 (ViT-S/B/L)")
        self.num_features = self.embed_dim = embed_dim
        self.num_tokens = 1
        self.n_blocks = depth
        self.num_heads = num_heads
        self.patch_size = patch_size
        self.num_register_tokens = 0
        self.interpolate_antialias = interpolate_antialias
        self.interpolate_offset = interpolate_offset
        self.chunked_blocks = False
        self.ffn_layer = ffn_layer

    # ------------------------------------------------------------------ what the reference module has and this one refuses
    @property
    def onnx_compatible_mode(self):
        return False

    @onnx_compatible_mode.setter
    def onnx_compatible_mode(self, value: bool):
        if value:
            raise _unsupported("onnx_compatible_mode is not provided")

    def init_weights(self):
        raise _unsupported("init_weights is not provided: load a state dict")

    # ------------------------------------------------------------------ EngineModel hooks
    def _expected_keys(self) -> List[str]:
        keys = ["cls_token", "pos_embed", "mask_token", "patch_embed.proj.weight", "patch_embed.proj.bias"]
        for i in range(self.n_blocks):
            keys += [f"blocks.{i}.{k}" for k in _BLOCK_KEYS]
        return keys + ["norm.weight", "norm.bias"]

    def _create_engine(self, handle):
        c = capi.DinoConfig()
        c.embed_dim, c.depth, c.num_heads = self.embed_dim, self.n_blocks, self.num_heads
        c.patch_size, c.num_register_tokens = self.patch_size, self.num_register_tokens
        c.interpolate_offset, c.interpolate_antialias = self.interpolate_offset, int(self.interpolate_antialias)
        c.ffn_layer, c.compute_dtype = capi.DINO_FFN[self.ffn_layer], self._compute_code()
        capi.check(capi.lib().moge_dino_create(C.byref(c), self._device.index, C.byref(handle)))

    # ------------------------------------------------------------------ host checks (before any device work)
    def _layers(self, n: Union[int, Sequence[int]]) -> List[int]:
        """The block indices `n` selects, in block order, as the reference's loop collects them (vision_transformer.py:283-293): an
        int n is the last n blocks, a sequence names them.  Raises AssertionError with the reference's message when some are not
        found (an index out of range, a repeated one, n > depth)."""
        take = range(self.n_blocks - n, self.n_blocks) if isinstance(n, int) else list(n)
        found = [i for i in range(self.n_blocks) if i in take]
        if len(found) != len(take):
            raise AssertionError(f"only {len(found)} / {len(take)} blocks found")
        return found

    def _check_hw(self, H: int, W: int):
        # dinov2/layers/patch_embed.py:72-73 (its messages)
        if H % self.patch_size:
            raise AssertionError(f"Input image height {H} is not a multiple of patch height {self.patch_size}")
        if W % self.patch_size:
            raise AssertionError(f"Input image width {W} is not a multiple of patch width: {self.patch_size}")

    def _check_input(self, x) -> Tuple[int, int, int]:
        if isinstance(x, list):
            raise _unsupported("a list of images (forward_features_list) is not provided: call forward_features_many or "
                               "get_intermediate_layers_many")
        if not isinstance(x, torch.Tensor) or x.dim() != 4 or x.shape[1] != 3:
            raise ValueError(f"x must be a (B, 3, H, W) tensor, got {tuple(x.shape) if isinstance(x, torch.Tensor) else type(x)}")
        if x.dtype not in (torch.float32, torch.float16, torch.bfloat16):
            raise TypeError(f"x must be float32, float16 or bfloat16, got {x.dtype}")
        B, _, H, W = x.shape
        self._check_hw(H, W)
        if B == 0:
            raise ValueError("x has no images")
        return B, H, W

    def _check_images(self, images):
        """The `_many` calls' argument checks, before any device work: a list of (3, H, W) fp32 / fp16 / bf16 tensors, H and W
        multiples of 14."""
        if not isinstance(images, list):
            raise TypeError(f"images must be a list of (3, H, W) tensors, got {type(images).__name__}")
        for i, im in enumerate(images):
            if not isinstance(im, torch.Tensor) or im.dim() != 3 or im.shape[0] != 3:
                raise ValueError(f"images[{i}] must be (3, H, W), got {tuple(im.shape) if isinstance(im, torch.Tensor) else type(im)}")
            if im.dtype not in (torch.float32, torch.float16, torch.bfloat16):
                raise TypeError(f"images[{i}] must be float32, float16 or bfloat16, got {im.dtype}")
            self._check_hw(im.shape[1], im.shape[2])

    # ------------------------------------------------------------------ forward path
    def _alloc(self, b: int, h: int, w: int, L: int, flags: int, tokens: bool, cls: bool, prenorm: bool):
        """The fp32 outputs of b images on an h x w token grid, each None unless asked for: tokens (L,b,T,D) or (L,b,D,h,w), cls
        (L,b,D), prenorm (b,T+1,D)."""
        T, D = h * w, self.embed_dim
        f = dict(dtype=torch.float32, device=self._device)
        tshape = (L, b, D, h, w) if flags & capi.DINO_CHANNEL_MAJOR else (L, b, T, D)
        return (torch.empty(tshape, **f) if tokens and L else None, torch.empty((L, b, D), **f) if cls and L else None,
                torch.empty((b, T + 1, D), **f) if prenorm else None)

    def _dino_call(self, groups, layers: List[int], flags: int):
        """ONE engine call over shape groups [(engine input (b,3,H,W), outputs of `_alloc`)]: the encoder runs once over the token
        rows of every group, and each group's outputs are written to its buffers."""
        self._ensure_engine()
        arr = (capi.DinoGroup * len(groups))()
        for g, (x, outs) in zip(arr, groups):
            g.x, g.x_dtype = x.data_ptr(), capi.torch_dtype_code(x.dtype)
            g.B, g.H, g.W = x.shape[0], x.shape[2], x.shape[3]
            g.out_tokens, g.out_cls, g.out_prenorm = (None if t is None else t.data_ptr() for t in outs)
        L = len(layers)
        lay = (C.c_int * max(L, 1))(*layers)
        lib = capi.lib()
        with torch.cuda.device(self._device):
            nbytes = C.c_size_t()
            capi.check(lib.moge_dino_workspace_bytes_groups(self._engine, arr, len(groups), lay, L, flags, C.byref(nbytes)))
            ws, ws_bytes = self._workspace_for(nbytes.value)
            capi.check(lib.moge_dino_forward_groups(self._engine, arr, len(groups), lay, L, flags, ws, ws_bytes,
                                                    capi.current_stream()))

    def _run(self, x: torch.Tensor, layers: List[int], flags: int, tokens: bool, cls: bool, prenorm: bool):
        """One backbone pass over x (B,3,H,W): the batch's outputs (`_alloc`), L = len(layers).  Large batches run as chunks
        (`_chunks`), one engine call each; a chunk's outputs are copied into the batch's."""
        B, H, W = x.shape[0], x.shape[2], x.shape[3]
        h, w = H // self.patch_size, W // self.patch_size
        want = (len(layers), flags, tokens, cls, prenorm)
        x = self._engine_input(x)
        out = self._alloc(B, h, w, *want)
        chunks = self._chunks(B, h * w + 1)
        for lo, n in chunks:
            part = out if len(chunks) == 1 else self._alloc(n, h, w, *want)
            self._dino_call([(x[lo:lo + n], part)], layers, flags)
            if part is not out:
                for full, p, dim in zip(out, part, (1, 1, 0)):
                    if full is not None:
                        full.narrow(dim, lo, n).copy_(p)
        return out

    def _run_many(self, images: List[torch.Tensor], layers: List[int], flags: int, tokens: bool, cls: bool, prenorm: bool):
        """One backbone pass over checked (3, H, W) images of any shapes: per image, in input order, its outputs (`_alloc`) with the
        batch dimension dropped, as views of its group's buffers.  The images are bucketed by shape and dtype and packed into engine
        calls of at most `max_chunk_tokens` tokens and MOGE_DINO_MAX_GROUPS shape groups (`_pack_calls`)."""
        p = self.patch_size
        calls = self._pack_calls(images, lambda H, W: ((H // p, W // p), (H // p) * (W // p) + 1), max_units=capi.DINO_MAX_GROUPS)
        want = (len(layers), flags, tokens, cls, prenorm)
        results: List[Optional[tuple]] = [None] * len(images)
        for call in calls:
            groups = [(self._engine_input(torch.stack([images[i].to(self._device) for i in idx])), self._alloc(len(idx), h, w, *want))
                      for (_, _, (h, w), idx) in call]
            self._dino_call(groups, layers, flags)
            for (_, _, _, idx), (_, (t, c, pre)) in zip(call, groups):
                for j, i in enumerate(idx):
                    results[i] = (None if t is None else t[:, j], None if c is None else c[:, j], None if pre is None else pre[j])
        return results

    def get_intermediate_layers(self, x: torch.Tensor, n: Union[int, Sequence] = 1, reshape: bool = False,
                                return_class_token: bool = False, norm=True) -> Tuple[Union[torch.Tensor, Tuple[torch.Tensor]]]:
        """vision_transformer.py:309-333: the patch tokens after the selected blocks, through the final norm (norm=True), as
        (B, T, D) or, reshape=True, (B, D, H/14, W/14); with return_class_token, (tokens, class token (B, D)) pairs."""
        self._check_input(x)
        layers = self._layers(n)
        if not layers:
            return ()
        flags = (capi.DINO_NORM if norm else 0) | (capi.DINO_CHANNEL_MAJOR if reshape else 0)
        tokens, cls, _ = self._run(x, layers, flags, True, return_class_token, False)
        outputs = list(tokens.unbind(0))
        if return_class_token:
            return tuple(zip(outputs, cls.unbind(0)))
        return tuple(outputs)

    def forward_features(self, x, masks=None) -> Dict[str, Optional[torch.Tensor]]:
        """vision_transformer.py:265-281: the normed class and patch tokens after the last block and the pre-norm stream."""
        if masks is not None:
            raise _unsupported("masks (iBOT mask tokens) are not provided")
        B = self._check_input(x)[0]
        tokens, cls, prenorm = self._run(x, [self.n_blocks - 1], capi.DINO_NORM, True, True, True)
        return {
            "x_norm_clstoken": cls[0],
            "x_norm_regtokens": tokens.new_empty((B, 0, self.embed_dim)),
            "x_norm_patchtokens": tokens[0],
            "x_prenorm": prenorm,
            "masks": masks,
        }

    def forward(self, *args, is_training=False, **kwargs):
        """vision_transformer.py:335-340: the normed class token through the Identity head."""
        if is_training:
            raise _unsupported("is_training=True is not provided (inference engine)")
        x = args[0] if args else kwargs.pop("x")
        if kwargs.get("masks") is not None:
            raise _unsupported("masks (iBOT mask tokens) are not provided")
        self._check_input(x)
        return self._run(x, [self.n_blocks - 1], capi.DINO_NORM, False, True, False)[1][0]

    __call__ = forward

    # ------------------------------------------------------------------ mixed-shape lists
    def get_intermediate_layers_many(self, images: List[torch.Tensor], n: Union[int, Sequence] = 1, reshape: bool = False,
                                     return_class_token: bool = False, norm=True) -> List[tuple]:
        """`get_intermediate_layers` over a list of (3, H, W) images of any shapes (H and W multiples of 14) and dtypes: entry i is
        bitwise `get_intermediate_layers(images[i][None], ...)` with the batch dimension dropped.  Each engine call runs the
        encoder once over the token rows of every shape it carries (`_run_many`)."""
        self._check_images(images)
        layers = self._layers(n)
        if not layers:
            return [() for _ in images]
        flags = (capi.DINO_NORM if norm else 0) | (capi.DINO_CHANNEL_MAJOR if reshape else 0)
        out = []
        for tokens, cls, _ in self._run_many(images, layers, flags, True, return_class_token, False):
            outputs = list(tokens.unbind(0))
            out.append(tuple(zip(outputs, cls.unbind(0))) if return_class_token else tuple(outputs))
        return out

    def forward_features_many(self, images: List[torch.Tensor]) -> List[Dict[str, Optional[torch.Tensor]]]:
        """`forward_features` over a list of (3, H, W) images of any shapes: one dict per image, in input order, with the batch
        dimension dropped and `masks` None."""
        self._check_images(images)
        return [{
            "x_norm_clstoken": cls[0],
            "x_norm_regtokens": tokens.new_empty((0, self.embed_dim)),
            "x_norm_patchtokens": tokens[0],
            "x_prenorm": prenorm,
            "masks": None,
        } for tokens, cls, prenorm in self._run_many(images, [self.n_blocks - 1], capi.DINO_NORM, True, True, True)]

    def forward_many(self, images: List[torch.Tensor]) -> List[torch.Tensor]:
        """`forward` over a list of (3, H, W) images of any shapes: the normed class token (D,) of each image, in input order."""
        self._check_images(images)
        return [cls[0] for _, cls, _ in self._run_many(images, [self.n_blocks - 1], capi.DINO_NORM, False, True, False)]


# ---------------------------------------------------------------------------------------------- constructors
def _vit(embed_dim, depth, num_heads, patch_size=16, num_register_tokens=0, **kwargs):
    return DinoVisionTransformer(patch_size=patch_size, embed_dim=embed_dim, depth=depth, num_heads=num_heads, mlp_ratio=4,
                                 num_register_tokens=num_register_tokens, **kwargs)


def vit_small(patch_size=16, num_register_tokens=0, **kwargs):
    return _vit(384, 12, 6, patch_size, num_register_tokens, **kwargs)


def vit_base(patch_size=16, num_register_tokens=0, **kwargs):
    return _vit(768, 12, 12, patch_size, num_register_tokens, **kwargs)


def vit_large(patch_size=16, num_register_tokens=0, **kwargs):
    return _vit(1024, 24, 16, patch_size, num_register_tokens, **kwargs)


def vit_giant2(patch_size=16, num_register_tokens=0, **kwargs):
    raise _unsupported("ViT-g (embed_dim 1536, SwiGLU FFN) is not provided: the encoder kernels take embed_dim <= 1024 and the "
                       "GELU MLP only")


_ARCHS = {"vit_small": vit_small, "vit_base": vit_base, "vit_large": vit_large}


def _make_dinov2_model(*, arch_name="vit_large", img_size=518, patch_size=14, init_values=1.0, ffn_layer="mlp", block_chunks=0,
                       num_register_tokens=0, interpolate_antialias=False, interpolate_offset=0.1, pretrained=True,
                       weights="LVD142M", **kwargs):
    """hub/backbones.py:18-61 without the download: pretrained=True raises."""
    if pretrained:
        raise _unsupported("pretrained=True is not provided (no download): build with pretrained=False and load a state dict with "
                           "load_state_dict")
    if weights not in ("LVD142M",) and getattr(weights, "value", None) != "LVD142M":
        raise AssertionError(f"Unsupported weights: {weights}")
    return _ARCHS[arch_name](img_size=img_size, patch_size=patch_size, init_values=init_values, ffn_layer=ffn_layer,
                             block_chunks=block_chunks, num_register_tokens=num_register_tokens,
                             interpolate_antialias=interpolate_antialias, interpolate_offset=interpolate_offset, **kwargs)


def dinov2_vits14(*, pretrained: bool = True, weights="LVD142M", **kwargs):
    """DINOv2 ViT-S/14 (hub/backbones.py:64-68); pretrained=False only."""
    return _make_dinov2_model(arch_name="vit_small", pretrained=pretrained, weights=weights, **kwargs)


def dinov2_vitb14(*, pretrained: bool = True, weights="LVD142M", **kwargs):
    """DINOv2 ViT-B/14 (hub/backbones.py:71-75); pretrained=False only."""
    return _make_dinov2_model(arch_name="vit_base", pretrained=pretrained, weights=weights, **kwargs)


def dinov2_vitl14(*, pretrained: bool = True, weights="LVD142M", **kwargs):
    """DINOv2 ViT-L/14 (hub/backbones.py:78-82); pretrained=False only."""
    return _make_dinov2_model(arch_name="vit_large", pretrained=pretrained, weights=weights, **kwargs)


def _no_registers(name):
    def f(*, pretrained: bool = True, weights="LVD142M", **kwargs):
        raise _unsupported(f"{name}: register tokens are not provided (they would add rows between the class token and the "
                           "patches, and no MoGe checkpoint uses them)")
    f.__name__ = name
    return f


def dinov2_vitg14(*, pretrained: bool = True, weights="LVD142M", **kwargs):
    """DINOv2 ViT-g/14 (hub/backbones.py:85-95): not provided."""
    vit_giant2()


dinov2_vits14_reg = _no_registers("dinov2_vits14_reg")
dinov2_vitb14_reg = _no_registers("dinov2_vitb14_reg")
dinov2_vitl14_reg = _no_registers("dinov2_vitl14_reg")
dinov2_vitg14_reg = _no_registers("dinov2_vitg14_reg")
