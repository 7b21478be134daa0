"""Drop-in module: put this repository's root on sys.path (instead of the reference's `code/`) and
`from models_rd import *` in code/Raindrop.py:19 resolves to the H100-native implementation."""
from raindrop_b200.models_rd import *  # noqa: F401,F403
from raindrop_b200.models_rd import __all__  # noqa: F401
