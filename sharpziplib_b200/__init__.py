"""sharpziplib_b200 -- host-side mirror of the SharpZipLib codec surface over libb200z.so (sm_90a kernels).

Only the hot path is here: Deflater / Inflater / DeflaterOutputStream / InflaterInputStream / Crc32 / Adler32 / BZip2Crc
and the batch plans the benchmark drives.  Names and argument meaning follow the reference (see each class's docstring for the
file:line it mirrors).  All compression work happens on the GPU inside libb200z.so; nothing here falls back to a CPU codec.
"""
from ._lib import (SharpZipBaseException, StreamDecodingException, B200zUnsupported, B200zCudaError,  # noqa: F401
                   InvalidOperationException, init, lib, SO_PATH, EXPORTS, STAGE_SEARCH, STAGE_ENCODE, STAGE_ALL)
from .checksum import Crc32, Adler32, BZip2Crc  # noqa: F401
from .codec import Deflater, Inflater, DeflateStrategy  # noqa: F401
from .streams import DeflaterOutputStream, InflaterInputStream, GZipOutputStream, GZipInputStream  # noqa: F401
from .batch import DeflatePlan, InflatePlan, Pipeline, DeflaterSet, InflaterSet, deflate_batch, inflate_batch, zip_entries, unzip_entries  # noqa: F401
from .lzw import LzwException, LzwInputStream, LzwPlan, lzw_batch  # noqa: F401
from . import encryption  # noqa: F401
