"""ctypes wrapper of oracle/_ref/libtcnn_ref.so (oracle/tcnn_ref): the reference's tiny-cuda-nn decoder network compiled for sm_90a.
TEST / BASELINE INFRASTRUCTURE ONLY.  The library exists only where the reference's sources were present at build time."""
from __future__ import annotations

import ctypes as C
import os

SO = os.path.join(os.path.dirname(os.path.abspath(__file__)), "_ref", "libtcnn_ref.so")


def available() -> bool:
    return os.path.exists(SO)


class TcnnDecoder:
    """tcnn NetworkWithInputEncoding(Composite[Identity(F), SH(degree)], FullyFusedMLP(128, n_hidden_layers)) on cuda:0, driven like
    the tcnn torch binding (fp16 params, loss scale 128).  Inputs are torch CUDA fp32 tensors; input rows are [features, (dir*s+1)/2]."""

    def __init__(self, n_features: int, sh_degree: int, n_hidden_layers: int, output_activation: str = "Sigmoid"):
        lib = C.CDLL(SO)
        vp, i64 = C.c_void_p, C.c_int64
        lib.tcnnref_create.argtypes = [C.c_int, C.c_int, C.c_int, C.c_char_p, C.POINTER(vp)]
        lib.tcnnref_destroy.argtypes = [vp]
        lib.tcnnref_n_params.restype = i64
        lib.tcnnref_n_params.argtypes = [vp]
        lib.tcnnref_padded_input_width.argtypes = [vp]
        lib.tcnnref_set_params.argtypes = [vp, vp, vp]
        lib.tcnnref_forward.argtypes = [vp, vp, i64, vp, vp, C.c_int]
        lib.tcnnref_backward.argtypes = [vp, vp, i64, vp, vp, vp]
        self._lib, self._h = lib, vp()
        if lib.tcnnref_create(n_features, sh_degree, n_hidden_layers, output_activation.encode(), C.byref(self._h)) != 0:
            raise RuntimeError("tcnnref_create failed")
        self.n_features = n_features

    @property
    def n_params(self) -> int:
        return int(self._lib.tcnnref_n_params(self._h))

    @property
    def padded_input_width(self) -> int:
        return int(self._lib.tcnnref_padded_input_width(self._h))

    @staticmethod
    def _stream():
        import torch

        return torch.cuda.current_stream().cuda_stream

    def set_params(self, params):
        assert self._lib.tcnnref_set_params(self._h, self._stream(), params.data_ptr()) == 0

    def forward(self, inputs, out, training: bool = True):
        assert self._lib.tcnnref_forward(self._h, self._stream(), inputs.shape[0], inputs.data_ptr(), out.data_ptr(), int(training)) == 0

    def backward(self, n: int, d_out, d_inputs, d_params):
        assert self._lib.tcnnref_backward(self._h, self._stream(), n, d_out.data_ptr(), d_inputs.data_ptr(), d_params.data_ptr()) == 0

    def close(self):
        if self._h:
            self._lib.tcnnref_destroy(self._h)
            self._h = C.c_void_p()
