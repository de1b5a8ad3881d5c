"""Drop-in for the reference's src/GraphGAN/config.py: same names, same defaults.

Kept as a thin alias so that ``import config`` from the working directory src/GraphGAN (the
reference's import style, graph_gan.py:8) resolves to the one configuration module the CUDA
implementation reads."""
import os
import sys

_ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
if _ROOT not in sys.path:
    sys.path.insert(0, _ROOT)

from graphgan_b200 import config as _cfg  # noqa: E402

sys.modules[__name__] = _cfg
