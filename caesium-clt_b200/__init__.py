"""b200-caesium: H100-native drop-in for caesiumclt's per-image compress path.

The product is the C-ABI shared library libb200caesium.so (include/b200_caesium.h, sources in csrc/);
this package only binds it (`_lib`) and mirrors the reference's host interface (`compressor`).
"""
from . import _lib  # noqa: F401
