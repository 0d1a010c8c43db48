"""hap_b200 -- H100-native (sm_90a) Hap frame codec.

The product is the C-ABI shared library `libhap_b200.so` (sources in hap_b200/csrc, API in include/).
This package only loads it and mirrors its entry points for Python callers (tests, bench):

    from hap_b200 import load
    lib = load()                 # HapB200: the hap.h calls + the device-resident batch extensions
    r, frame = lib.encode([dxt_bytes], [HapTextureFormat_YCoCg_DXT5], [HapCompressorSnappy], [8])

There is no Python or CPU implementation behind these calls: if the CUDA library is missing or cannot
be loaded, `load()` raises.
"""
from .abi import *  # noqa: F401,F403
from .lib import HapB200, library_path, load  # noqa: F401
