"""Drop-in alias of the reference's `moge.utils` package: `moge.utils.alignment` resolves to the GPU solvers (moge_b200.alignment),
`moge.utils.geometry_torch` to the geometry utilities (moge_b200.geometry)."""
