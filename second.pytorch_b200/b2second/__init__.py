"""b2second -- host side of the H100-native SECOND inference hot path.

Everything here sits above the C-ABI library ``libb2second.so`` (see include/b2second.h) and mirrors
the operator interface second.pytorch exposes for this path.  ``refcompat`` is container-only glue
for importing the unmodified reference in tests.
"""
__version__ = "0.1.0"
