from moge_b200.geometry import *  # noqa: F401,F403
from moge_b200.geometry import __all__  # noqa: F401
