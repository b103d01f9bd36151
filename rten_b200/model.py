"""Host-side mirror of `rten::Model` (src/model.rs) over rten_b200_model_*: load an ONNX file, run it by input / output
names.  The graph executor itself is native (csrc/model.cu); this module only marshals descriptors."""
from __future__ import annotations

import ctypes as C
import json
from typing import Dict, List, Optional, Sequence, Union

import numpy as np

from . import _lib
from .ops import Context, DeviceTensor, OpError, _Args, _RT2NP
from ._lib import RtenTensor


def onnx_summary(data: bytes) -> dict:
    """The reader alone (no GPU): decoded structure of an ONNX file as a dict."""
    lib = _lib.load()
    need = C.c_size_t(0)
    st = lib.rten_b200_onnx_summary(data, len(data), None, 0, C.byref(need))
    if st != 0:
        raise OpError(st, "ONNX decode failed")
    buf = C.create_string_buffer(need.value)
    st = lib.rten_b200_onnx_summary(data, len(data), buf, need.value, None)
    if st != 0:
        raise OpError(st, "ONNX decode failed")
    return json.loads(buf.value.decode())


class Model:
    """`Model::load` / `Model::run` (src/model.rs:300-760): inputs and outputs are addressed by name."""

    def __init__(self, ctx: Context, data: Union[bytes, str]):
        if isinstance(data, str):
            data = open(data, "rb").read()
        self.ctx = ctx
        self._bytes = data
        h = C.c_void_p()
        ctx.check(ctx.lib.rten_b200_model_load(ctx.handle, data, len(data), C.byref(h)))
        self.handle = h
        lib = ctx.lib
        self.input_names = [lib.rten_b200_model_input_name(h, i).decode() for i in range(lib.rten_b200_model_num_inputs(h))]
        self.output_names = [lib.rten_b200_model_output_name(h, i).decode() for i in range(lib.rten_b200_model_num_outputs(h))]
        self.node_ops = [lib.rten_b200_model_node_op(h, i).decode() for i in range(lib.rten_b200_model_num_nodes(h))]

    @property
    def summary(self) -> dict:
        return json.loads(self.ctx.lib.rten_b200_model_summary(self.handle).decode())

    def run(self, inputs: Dict[str, object], outputs: Optional[Sequence[str]] = None) -> List[object]:
        """Inputs are numpy arrays, DeviceTensors or KvCacheHandles (generate.py).  A handle is passed as a writable view
        of its first seq_len positions with its capacity (rten_b200_model_run_ex): an attention node may write its present
        cache into it, and such an output comes back as a KvCacheHandle over the same buffer with the new length."""
        from .generate import KvCacheHandle
        outputs = list(outputs) if outputs is not None else self.output_names
        A = _Args(self.ctx)
        names = list(inputs)
        in_names = (C.c_char_p * len(names))(*[n.encode() for n in names])
        in_t = (RtenTensor * max(len(names), 1))()
        opts = (_lib.RtenModelInputOpts * max(len(names), 1))()
        handles = {}
        for i, n in enumerate(names):
            v = inputs[n]
            if isinstance(v, KvCacheHandle):
                if v.transposed:
                    raise OpError(5, f"{n}: a transposed cache handle cannot be a model input")
                t = v.tensor
                v = t.view(t.shape[:2] + (v.seq_len,) + t.shape[3:], t.strides)
                opts[i].writable, opts[i].grow_axis, opts[i].capacity = 1, 2, inputs[n].capacity
                handles[i] = inputs[n]
            ref = A.t(v)
            C.memmove(C.byref(in_t, i * C.sizeof(RtenTensor)), ref, C.sizeof(RtenTensor))
        out_names = (C.c_char_p * len(outputs))(*[n.encode() for n in outputs])
        out_t = (RtenTensor * len(outputs))()
        if handles:
            alias = (C.c_int32 * len(outputs))()
            self.ctx.check(self.ctx.lib.rten_b200_model_run_ex(self.handle, len(names), in_names, in_t, C.cast(opts, C.c_void_p),
                                                               len(outputs), out_names, out_t, alias))
        else:
            alias = [-1] * len(outputs)
            self.ctx.check(self.ctx.lib.rten_b200_model_run(self.handle, len(names), in_names, in_t, len(outputs), out_names, out_t))
        res = []
        for d, a in zip(out_t, alias):
            if a >= 0:
                h = handles[a]
                res.append(KvCacheHandle(h.tensor, int(d.shape[2]), h.capacity))
                continue
            shape = tuple(d.shape[i] for i in range(d.ndim))
            strides = tuple(d.strides[i] for i in range(d.ndim))
            res.append(DeviceTensor(self.ctx, d.data, shape, strides, _RT2NP[d.dtype], owner=True))
        return res

    def close(self):
        if getattr(self, "handle", None) and self.ctx.handle:
            self.ctx.lib.rten_b200_model_free(self.handle)
            self.handle = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass
