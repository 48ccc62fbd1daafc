"""b200z -- H100-native block-parallel codec engine for 7-Zip's ZSTD (4F71101) and LZMA2 (21) coders.

The directory name (`7-zip-zstd_b200`) is not a Python identifier; load it with
`__graft_entry__.load_package()` (importlib), which registers it as module `b200z`.
"""
from .binding import Codec, B200zError, lib_path, load_library  # noqa: F401
from . import corpus  # noqa: F401
