"""The reference's `moge/utils/vis.py` colourisers in numpy, with matplotlib's "Spectral" colour map restated.  TEST
INFRASTRUCTURE ONLY, and the host comparator of tools/bench_cli.py.

matplotlib is not a dependency, so the colour map is restated from its published semantics:
- `LinearSegmentedColormap.from_list` puts the 11 ColorBrewer "Spectral" colours (8-bit values over 255) at np.linspace(0, 1, 11),
  and `_create_lookup_table(256, data, gamma=1.0)` interpolates them in float64 into a (256, 3) table, clipped to [0, 1];
- `Colormap.__call__(X)` on a float array: xa = X * 256 in X's dtype, xa == 256 becomes 255, then xa < 0 takes the "under"
  colour (the first entry), xa >= 256 the "over" colour (the last entry) and NaN the "bad" colour (0, 0, 0, 0); everything else
  takes entry int(xa), truncated.
The colourisers below are the reference's lines with `spectral(...)` in place of `matplotlib.colormaps['Spectral'](...)`;
the quantiles are np.nanquantile itself.  tests/test_vis_host.py checks this restatement against matplotlib where it is
installed.
"""
import numpy as np

SPECTRAL_COLORS = ((158, 1, 66), (213, 62, 79), (244, 109, 67), (253, 174, 97), (254, 224, 139), (255, 255, 191),
                   (230, 245, 152), (171, 221, 164), (102, 194, 165), (50, 136, 189), (94, 79, 162))
N = 256


def create_lookup_table(n: int, data: np.ndarray, gamma: float = 1.0) -> np.ndarray:
    """matplotlib.colors._create_lookup_table for an (K, 3) segment array [x, y0, y1]."""
    adata = np.array(data)
    x, y0, y1 = adata[:, 0], adata[:, 1], adata[:, 2]
    x = x * (n - 1)
    xind = (n - 1) * np.linspace(0, 1, n) ** gamma
    ind = np.searchsorted(x, xind)[1:-1]
    distance = (xind[1:-1] - x[ind - 1]) / (x[ind] - x[ind - 1])
    lut = np.concatenate([[y1[0]], distance * (y0[ind] - y1[ind - 1]) + y1[ind - 1], [y0[-1]]])
    return np.clip(lut, 0.0, 1.0)


def spectral_lut() -> np.ndarray:
    """The (256 + 3, 4) float64 table of matplotlib's Spectral map: 256 colours, then under, over and bad."""
    rgb = np.array(SPECTRAL_COLORS, dtype=np.float64) / 255
    vals = np.linspace(0, 1, len(rgb))
    lut = np.ones((N + 3, 4), dtype=np.float64)
    for c in range(3):
        lut[:N, c] = create_lookup_table(N, np.column_stack([vals, rgb[:, c], rgb[:, c]]))
    lut[N] = lut[0]
    lut[N + 1] = lut[N - 1]
    lut[N + 2] = 0.0
    return lut


_LUT = spectral_lut()


def colormap_index(X: np.ndarray) -> np.ndarray:
    """The table row Colormap.__call__ takes for each value: 0..255, 256 (under), 257 (over) or 258 (bad)."""
    xa = np.array(X, copy=True)
    xa *= N
    xa[xa == N] = N - 1
    mask_under = xa < 0
    mask_over = xa >= N
    mask_bad = np.isnan(xa)
    with np.errstate(invalid="ignore"):
        xa = xa.astype(int)
    xa[mask_under] = N
    xa[mask_over] = N + 1
    xa[mask_bad] = N + 2
    return xa


def spectral(X: np.ndarray) -> np.ndarray:
    """matplotlib.colormaps['Spectral'](X): float64 RGBA."""
    return _LUT.take(colormap_index(X), axis=0, mode="clip")


def lut_u8() -> np.ndarray:
    """The (256, 3) uint8 table the colourisers end up with: trunc(clip(lut, 0, 1) * 255)."""
    return (_LUT[:N, :3].clip(0, 1) * 255).astype(np.uint8)


def _cmap(cmap: str):
    if cmap != "Spectral":
        raise ValueError(f"only the 'Spectral' colour map is restated, not {cmap!r}")
    return spectral


def colorize_depth(depth: np.ndarray, mask: np.ndarray = None, normalize: bool = True, cmap: str = 'Spectral') -> np.ndarray:
    if mask is None:
        depth = np.where(depth > 0, depth, np.nan)
    else:
        depth = np.where((depth > 0) & mask, depth, np.nan)
    disp = 1 / depth
    if normalize:
        min_disp, max_disp = np.nanquantile(disp, 0.001), np.nanquantile(disp, 0.99)
        disp = (disp - min_disp) / (max_disp - min_disp)
    colored = np.nan_to_num(_cmap(cmap)(1.0 - disp)[..., :3], 0)
    colored = np.ascontiguousarray((colored.clip(0, 1) * 255).astype(np.uint8))
    return colored


def colorize_depth_affine(depth: np.ndarray, mask: np.ndarray = None, cmap: str = 'Spectral') -> np.ndarray:
    if mask is not None:
        depth = np.where(mask, depth, np.nan)

    min_depth, max_depth = np.nanquantile(depth, 0.001), np.nanquantile(depth, 0.999)
    depth = (depth - min_depth) / (max_depth - min_depth)
    colored = np.nan_to_num(_cmap(cmap)(depth)[..., :3], 0)
    colored = np.ascontiguousarray((colored.clip(0, 1) * 255).astype(np.uint8))
    return colored


def colorize_disparity(disparity: np.ndarray, mask: np.ndarray = None, normalize: bool = True, cmap: str = 'Spectral') -> np.ndarray:
    if mask is not None:
        disparity = np.where(mask, disparity, np.nan)

    if normalize:
        min_disp, max_disp = np.nanquantile(disparity, 0.001), np.nanquantile(disparity, 0.999)
        disparity = (disparity - min_disp) / (max_disp - min_disp)
    colored = np.nan_to_num(_cmap(cmap)(1.0 - disparity)[..., :3], 0)
    colored = np.ascontiguousarray((colored.clip(0, 1) * 255).astype(np.uint8))
    return colored


def colorize_normal(normal: np.ndarray, mask: np.ndarray = None) -> np.ndarray:
    if mask is not None:
        normal = np.where(mask[..., None], normal, 0)
    normal = normal * [0.5, -0.5, -0.5] + 0.5
    normal = (normal.clip(0, 1) * 255).astype(np.uint8)
    return normal


def nanquantile_from_sorted(valid_sorted: np.ndarray, q: float) -> np.float32:
    """np.nanquantile(values, q) of fp32 values from their sorted valid (non-NaN) values, written out as the kernels compute it:
    v = fp32(n - 1) * fp32(q); previous = floor(v), next = previous + 1, both n - 1 when v >= n - 1; gamma = fp32(v - previous)
    with previous an integer (-1 above the bounds); then numpy's _lerp in fp32."""
    n = len(valid_sorted)
    if n == 0:
        return np.float32(np.nan)
    f32 = np.float32
    last = f32(n - 1)
    v = last * f32(q)
    if v >= last:
        i = j = n - 1
        gamma = f32(np.float64(v) + 1.0)
    else:
        p = np.floor(v)
        i, j = int(p), int(p + f32(1))
        gamma = f32(np.float64(v) - np.float64(i))
    a, b = valid_sorted[i], valid_sorted[j]
    with np.errstate(invalid="ignore", over="ignore"):
        diff = f32(b - a)
        return f32(b - diff * (f32(1) - gamma)) if gamma >= 0.5 else f32(a + diff * gamma)
