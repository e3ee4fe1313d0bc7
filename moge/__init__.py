"""Drop-in alias: `from moge.model.v2 import MoGeModel` resolves to the H100-native engine (moge_b200)."""
