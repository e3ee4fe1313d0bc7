from moge_b200.metrics import *  # noqa: F401,F403
from moge_b200.metrics import __all__  # noqa: F401
