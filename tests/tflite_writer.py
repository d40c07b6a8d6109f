"""Minimal .tflite (schema v3, "TFL3") flatbuffer writer, and a graph builder on top of it (test helper).

Writes the schema subset that tools/tflite_graph.py and backscrub_b200/csrc/tflite_model.cpp read (field numbering
of tensorflow/lite/schema/schema.fbs: Model, SubGraph, Tensor, Buffer, OperatorCode, Operator and the option tables
of the fourteen supported operators), so tests can build graphs of any shape the planner admits, not only the five
bundled models.

Layout: the root offset, then every object after the object that refers to it (flatbuffer offsets point forward);
each table is preceded by its own vtable.  Constant data is 16-byte aligned, as TFLite's converter writes it.
"""
from __future__ import annotations

import struct

import numpy as np

CODE = {"ADD": 0, "AVERAGE_POOL_2D": 1, "CONCATENATION": 2, "CONV_2D": 3, "DEPTHWISE_CONV_2D": 4, "DEQUANTIZE": 6,
        "FULLY_CONNECTED": 9, "LOGISTIC": 14, "MUL": 18, "RELU": 19, "RELU6": 21, "RESIZE_BILINEAR": 23, "CUSTOM": 32,
        "HARD_SWISH": 117}
ACT = {"NONE": 0, "RELU": 1, "RELU_N1_TO_1": 2, "RELU6": 3}
TTYPE = {"f32": 0, "f16": 1, "i32": 2}
PAD = {"SAME": 0, "VALID": 1}
# BuiltinOptions union member ids (schema.fbs: union BuiltinOptions)
OPT_TYPE = {"CONV_2D": 1, "DEPTHWISE_CONV_2D": 2, "AVERAGE_POOL_2D": 5, "FULLY_CONNECTED": 8, "CONCATENATION": 10,
            "ADD": 11, "RESIZE_BILINEAR": 15, "MUL": 21}
TCONV = "Convolution2DTransposeBias"


# ------------------------------------------------------------------------------------------------ flatbuffer objects
class _Table:
    def __init__(self, fields):
        self.fields = fields          # list of (slot, fmt, value): fmt a struct code, or "ref" for an object


class _Vec:
    def __init__(self, fmt, items, align=4):
        self.fmt, self.items, self.align = fmt, items, align     # fmt a struct code, "ref" or "bytes"


def _str(s: str) -> _Vec:
    return _Vec("str", s.encode())


def _serialize(root: _Table, ident: bytes = b"TFL3") -> bytes:
    buf = bytearray(8)
    buf[4:8] = ident
    patches = [(0, root)]                          # (position of a uoffset, object it must point at)
    queue = [root]
    placed = {}

    def pad_to(a):
        while len(buf) % a:
            buf.append(0)

    while queue:
        obj = queue.pop(0)
        if id(obj) in placed:
            continue
        if isinstance(obj, _Table):
            fields = sorted(obj.fields, key=lambda f: f[0])
            nslots = 1 + max((f[0] for f in fields), default=-1)
            # table body: soffset, then the fields, each aligned to its size relative to the table start (8-aligned)
            body = bytearray(4)
            offs = {}
            for slot, fmt, val in sorted(fields, key=lambda f: -(4 if f[1] == "ref" else struct.calcsize("<" + f[1]))):
                size = 4 if fmt == "ref" else struct.calcsize("<" + fmt)
                while len(body) % size:
                    body.append(0)
                offs[slot] = len(body)
                body += bytes(4) if fmt == "ref" else struct.pack("<" + fmt, val)
            vt = struct.pack("<HH", 4 + 2 * nslots, len(body)) + b"".join(
                struct.pack("<H", offs.get(s, 0)) for s in range(nslots))
            pad_to(2)
            vt_pos = len(buf)
            buf += vt
            # the table start must be 8-aligned (8-byte scalars are never written here, so 4 would do)
            while (len(buf)) % 8:
                buf.append(0)
            pos = len(buf)
            struct.pack_into("<i", body, 0, pos - vt_pos)
            buf += body
            for slot, fmt, val in fields:
                if fmt == "ref":
                    patches.append((pos + offs[slot], val))
                    queue.append(val)
        else:
            if obj.fmt == "str":
                pad_to(4)
                pos = len(buf)
                buf += struct.pack("<I", len(obj.items)) + obj.items + b"\0"
            elif obj.fmt == "bytes":
                while (len(buf) + 4) % obj.align:
                    buf.append(0)
                pos = len(buf)
                buf += struct.pack("<I", len(obj.items)) + bytes(obj.items)
            elif obj.fmt == "ref":
                pad_to(4)
                pos = len(buf)
                buf += struct.pack("<I", len(obj.items)) + bytes(4 * len(obj.items))
                for k, it in enumerate(obj.items):
                    patches.append((pos + 4 + 4 * k, it))
                    queue.append(it)
            else:
                pad_to(4)
                pos = len(buf)
                buf += struct.pack("<I", len(obj.items)) + struct.pack("<%d%s" % (len(obj.items), obj.fmt), *obj.items)
        placed[id(obj)] = pos
    for at, obj in patches:
        target = placed[id(obj)]
        assert target > at
        struct.pack_into("<I", buf, at, target - at)
    return bytes(buf)


# ------------------------------------------------------------------------------------------------ model description
def _options(kind: str, o: dict):
    """(builtin_options_type, option table) of an operator, or (0, None)"""
    a = lambda k: ACT[o.get(k, "NONE")]
    if kind == "CONV_2D":
        f = [(0, "b", o["padding"]), (1, "i", o["stride_w"]), (2, "i", o["stride_h"]), (3, "b", a("act")),
             (4, "i", o.get("dil_w", 1)), (5, "i", o.get("dil_h", 1))]
    elif kind == "DEPTHWISE_CONV_2D":
        f = [(0, "b", o["padding"]), (1, "i", o["stride_w"]), (2, "i", o["stride_h"]), (3, "i", o.get("mult", 1)),
             (4, "b", a("act")), (5, "i", o.get("dil_w", 1)), (6, "i", o.get("dil_h", 1))]
    elif kind == "AVERAGE_POOL_2D":
        f = [(0, "b", o["padding"]), (1, "i", o["stride_w"]), (2, "i", o["stride_h"]), (3, "i", o["fw"]),
             (4, "i", o["fh"]), (5, "b", a("act"))]
    elif kind == "RESIZE_BILINEAR":
        f = [(2, "B", int(o.get("align_corners", False))), (3, "B", int(o.get("half_pixel", False)))]
    elif kind == "FULLY_CONNECTED":
        f = [(0, "b", a("act")), (2, "B", int(o.get("keep_num_dims", False)))]
    elif kind in ("ADD", "MUL"):
        f = [(0, "b", a("act"))]
    elif kind == "CONCATENATION":
        f = [(0, "i", o["axis"]), (1, "b", a("act"))]
    else:
        return 0, None
    return OPT_TYPE[kind], _Table(f)


def serialize(tensors, ops, inputs, outputs, version=3) -> bytes:
    """tensors: dicts {shape, dtype ('f32' | 'f16' | 'i32'), name, data (None or array)};
    ops: dicts {kind, inputs, outputs, opts, custom (name, for CUSTOM), custom_options (bytes)}."""
    buffers = [_Table([])]                                        # buffer 0: the empty buffer of every activation
    ttabs = []
    for t in tensors:
        bidx = 0
        if t.get("data") is not None:
            dt = {"f32": "<f4", "f16": "<f2", "i32": "<i4"}[t["dtype"]]
            raw = np.ascontiguousarray(t["data"], dt).tobytes()
            buffers.append(_Table([(0, "ref", _Vec("bytes", raw, align=16))]))
            bidx = len(buffers) - 1
        ttabs.append(_Table([(0, "ref", _Vec("i", [int(v) for v in t["shape"]])), (1, "b", TTYPE[t["dtype"]]),
                             (2, "I", bidx), (3, "ref", _str(t.get("name", "")))]))
    codes, code_tabs, otabs = {}, [], []
    for op in ops:
        key = (op["kind"], op.get("custom", ""))
        if key not in codes:
            c = CODE[op["kind"]]
            f = [(0, "b", min(c, 127)), (2, "i", 1), (3, "i", c)]
            if op["kind"] == "CUSTOM":
                f.append((1, "ref", _str(op["custom"])))
            codes[key] = len(code_tabs)
            code_tabs.append(_Table(f))
        f = [(0, "I", codes[key]), (1, "ref", _Vec("i", list(op["inputs"]))), (2, "ref", _Vec("i", list(op["outputs"])))]
        ot, otab = _options(op["kind"], op.get("opts", {}))
        if otab is not None:
            f += [(3, "B", ot), (4, "ref", otab)]
        if op.get("custom_options") is not None:
            f.append((5, "ref", _Vec("bytes", op["custom_options"])))
        otabs.append(_Table(f))
    sg = _Table([(0, "ref", _Vec("ref", ttabs)), (1, "ref", _Vec("i", list(inputs))), (2, "ref", _Vec("i", list(outputs))),
                 (3, "ref", _Vec("ref", otabs)), (4, "ref", _str("main"))])
    model = _Table([(0, "I", version), (1, "ref", _Vec("ref", code_tabs)), (2, "ref", _Vec("ref", [sg])),
                    (3, "ref", _str("generated")), (4, "ref", _Vec("ref", buffers))])
    return _serialize(model)


def tconv_options(padding_same=True, stride_w=2, stride_h=2) -> bytes:
    """custom_options of Convolution2DTransposeBias: TfLiteTransposeConvParams {padding (C enum, 1 = SAME), stride_w, stride_h}"""
    return struct.pack("<iii", 1 if padding_same else 2, stride_w, stride_h)


def from_graph(g) -> bytes:
    """Re-serialise a graph parsed by tools/tflite_graph.load."""
    tensors = [dict(shape=t.shape, dtype=t.dtype, name=t.name, data=t.data) for t in g.tensors]
    ops = []
    for op in g.ops:
        d = dict(kind=op.kind, inputs=op.inputs, outputs=op.outputs, opts=dict(op.opts))
        if op.kind == "CUSTOM":
            d["custom"] = op.opts["custom"]
            if op.opts["custom"] == TCONV:
                d["custom_options"] = tconv_options(op.opts["padding_c_enum"] == 1, op.opts["stride_w"], op.opts["stride_h"])
        assert d["opts"].get("act", "NONE") in ACT, op
        ops.append(d)
    return serialize(tensors, ops, g.inputs, g.outputs)


# ------------------------------------------------------------------------------------------------ graph builder
def conv_out(n, k, stride, dil, padding):
    """TF SAME / VALID output size (tensorflow/lite/kernels/padding.h)"""
    eff = (k - 1) * dil + 1
    return (n + stride - 1) // stride if padding == "SAME" else (n + stride - eff) // stride


class Builder:
    """Graph builder: every method takes and returns tensor indices, computes the output shape and draws seeded
    weights.  `dyadic=True` draws weights and biases as small integers times 2^-3 (with `wmax` the largest integer), so
    graphs of linear ops have exactly representable results; otherwise weights are uniform in +-1/sqrt(fan-in)."""

    def __init__(self, h, w, c=3, seed=0, dyadic=False, wmax=2, fp16=False):
        self.rng = np.random.default_rng(seed)
        self.dyadic, self.wmax, self.fp16 = dyadic, wmax, fp16
        self.tensors, self.ops = [], []
        self.x = self.act_tensor(h, w, c, "input")
        self.output = None

    # -- tensors
    def act_tensor(self, h, w, c, name=None):
        self.tensors.append(dict(shape=[1, h, w, c], dtype="f32", name=name or f"t{len(self.tensors)}", data=None))
        return len(self.tensors) - 1

    def shape(self, t):
        s = self.tensors[t]["shape"]
        return s[1:] if len(s) == 4 else [1, 1, s[-1]]

    def const(self, data, dtype="f32", name=None, shape=None):
        data = np.asarray(data)
        self.tensors.append(dict(shape=list(data.shape if shape is None else shape), dtype=dtype,
                                 name=name or f"c{len(self.tensors)}", data=data.reshape(-1)))
        return len(self.tensors) - 1

    def weight(self, shape, fan_in):
        if self.dyadic:
            v = self.rng.integers(-self.wmax, self.wmax + 1, shape).astype(np.float32) / 8
        else:
            v = self.rng.uniform(-1, 1, shape).astype(np.float32) / np.float32(np.sqrt(fan_in))
        if not self.fp16:
            return self.const(v)
        # fp16 storage behind DEQUANTIZE, as the MLKit model stores its weights
        h = self.const(v.astype(np.float16), dtype="f16")
        t = len(self.tensors)
        self.tensors.append(dict(shape=list(shape), dtype="f32", name=f"dq{t}", data=None))
        self.ops.append(dict(kind="DEQUANTIZE", inputs=[h], outputs=[t]))
        return t

    def _op(self, kind, inputs, out, opts=None, **kw):
        self.ops.append(dict(kind=kind, inputs=list(inputs), outputs=[out], opts=opts or {}, **kw))
        return out

    # -- operators
    def conv(self, x, oc, k=1, stride=1, dil=1, pad="SAME", act="NONE", bias=True):
        h, w, c = self.shape(x)
        kh, kw = (k, k) if isinstance(k, int) else k
        sh, sw = (stride, stride) if isinstance(stride, int) else stride
        oh, ow = conv_out(h, kh, sh, dil, pad), conv_out(w, kw, sw, dil, pad)
        wt = self.weight((oc, kh, kw, c), kh * kw * c)
        ins = [x, wt] + ([self.weight((oc,), kh * kw * c)] if bias else [-1])
        return self._op("CONV_2D", ins, self.act_tensor(oh, ow, oc),
                        dict(padding=PAD[pad], stride_w=sw, stride_h=sh, act=act, dil_w=dil, dil_h=dil))

    def pw(self, x, oc, act="NONE", bias=True):
        return self.conv(x, oc, 1, act=act, bias=bias)

    def dw(self, x, k=3, stride=1, dil=1, pad="SAME", act="NONE", mult=1):
        h, w, c = self.shape(x)
        oh, ow = conv_out(h, k, stride, dil, pad), conv_out(w, k, stride, dil, pad)
        ins = [x, self.weight((1, k, k, c * mult), k * k), self.weight((c * mult,), k * k)]
        return self._op("DEPTHWISE_CONV_2D", ins, self.act_tensor(oh, ow, c * mult),
                        dict(padding=PAD[pad], stride_w=stride, stride_h=stride, mult=mult, act=act, dil_w=dil, dil_h=dil))

    def pool(self, x, act="NONE", fh=None, fw=None, stride=1):
        """AVERAGE_POOL_2D, global unless a filter size is given (VALID padding)"""
        h, w, c = self.shape(x)
        fh, fw = fh or h, fw or w
        oh, ow = conv_out(h, fh, stride, 1, "VALID"), conv_out(w, fw, stride, 1, "VALID")
        return self._op("AVERAGE_POOL_2D", [x], self.act_tensor(oh, ow, c),
                        dict(padding=PAD["VALID"], stride_w=stride, stride_h=stride, fw=fw, fh=fh, act=act))

    def fc(self, x, n, act="NONE"):
        h, w, c = self.shape(x)
        ins = [x, self.weight((n, c), c), self.weight((n,), c)]
        return self._op("FULLY_CONNECTED", ins, self.act_tensor(h, w, n), dict(act=act, keep_num_dims=True))

    def se(self, x, mid, fc="conv", n=None, gate="LOGISTIC"):
        """squeeze-excite scale vector: global pool -> FC(mid, RELU) -> FC(n or C) -> gate, as 1x1 convs or FCs"""
        c = self.shape(x)[2]
        p = self.pool(x)
        if fc == "conv":
            s = self.pw(p, mid, act="RELU")
            s = self.pw(s, n or c)
        else:
            s = self.fc(p, mid, act="RELU")
            s = self.fc(s, n or c)
        return self.unary(gate, s) if gate else s

    def pool_se(self, x, mid, fc="conv", gate="LOGISTIC"):
        """x * SE(x): the channel-broadcast MUL of a squeeze-excite block"""
        return self.mul(x, self.se(x, mid, fc=fc, gate=gate))

    def resize(self, x, oh, ow, mode="half_pixel"):
        h, w, c = self.shape(x)
        size = self.const(np.array([oh, ow], np.int32), dtype="i32")
        return self._op("RESIZE_BILINEAR", [x, size], self.act_tensor(oh, ow, c),
                        dict(align_corners=mode == "align_corners", half_pixel=mode == "half_pixel"))

    def tconv(self, x, oc, out_hw=None, same=True, stride=2):
        h, w, c = self.shape(x)
        oh, ow = out_hw or (2 * h, 2 * w)
        ins = [x, self.weight((oc, 2, 2, c), c), self.weight((oc,), c)]
        return self._op("CUSTOM", ins, self.act_tensor(oh, ow, oc), custom=TCONV,
                        custom_options=tconv_options(same, stride, stride))

    def custom(self, name, x, options=b""):
        h, w, c = self.shape(x)
        return self._op("CUSTOM", [x], self.act_tensor(h, w, c), custom=name, custom_options=options)

    def add(self, a, b, act="NONE"):
        sa, sb = self.shape(a), self.shape(b)
        out = self.act_tensor(*max(sa, sb, key=lambda s: s[0] * s[1] * s[2]))
        return self._op("ADD", [a, b], out, dict(act=act))

    def mul(self, a, b, act="NONE"):
        sa, sb = self.shape(a), self.shape(b)
        out = self.act_tensor(*max(sa, sb, key=lambda s: s[0] * s[1] * s[2]))
        return self._op("MUL", [a, b], out, dict(act=act))

    def unary(self, kind, x):
        return self._op(kind, [x], self.act_tensor(*self.shape(x)))

    def concat(self, xs, axis=3):
        shapes = [self.shape(x) for x in xs]
        h, w, _ = shapes[0]
        if axis in (3, -1):
            out = self.act_tensor(h, w, sum(s[2] for s in shapes))
        else:                          # (only to build refusals: concatenation along the height)
            out = self.act_tensor(sum(s[0] for s in shapes), w, shapes[0][2])
        return self._op("CONCATENATION", xs, out, dict(axis=axis, act="NONE"))

    # -- output
    def bytes(self, out=None):
        out = self.ops[-1]["outputs"][0] if out is None else out
        return serialize(self.tensors, self.ops, [self.x], [out])

    def write(self, path, out=None):
        with open(path, "wb") as f:
            f.write(self.bytes(out))
        return path
