from moge_b200.alignment import *  # noqa: F401,F403
from moge_b200.alignment import __all__  # noqa: F401
