from moge_b200.model.v1 import MoGeModel  # noqa: F401
