"""alfalfa_b200 -- H100-native VP8 pixel pipeline behind excamera/alfalfa's state-passing codec API.

Python here is plumbing over the C ABI of include/vp8gpu.h (ctypes): the product is
alfalfa_b200/libvp8gpu.so = hand-written sm_90a CUDA kernels + a C++ host library.
"""
from .capi import CudaError, Invalid, LogicError, Unsupported, Vp8Error  # noqa: F401
from .decoder import (Context, Decoder, DecoderState, Encoder, FilePlayer, ParsedFrame, RasterHandle,  # noqa: F401
                      decode_ivf, reencode_chunks, write_ivf)
