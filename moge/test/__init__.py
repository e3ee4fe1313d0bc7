"""Drop-in alias of the reference's `moge.test` package: `moge.test.metrics` resolves to the GPU metrics (moge_b200.metrics)."""
