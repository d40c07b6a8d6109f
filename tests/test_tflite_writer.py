"""tests/tflite_writer.py: what it writes reads back identically through both readers (tools/tflite_graph.py and the
C oracle's loader), and the five bundled models re-serialised from their parsed graphs give the oracle's output bits."""
import os

import numpy as np
import pytest

from oracle import pyoracle as po
from tests import tflite_writer as tw
from tests.conftest import MODELS, model_path
from tools import tflite_graph as tg


def every_op_graph(fp16):
    b = tw.Builder(8, 10, seed=4, fp16=fp16)
    x = b.conv(b.x, 8, 3, 2, pad="VALID", act="RELU6")
    x = b.dw(x, 3, 1, dil=2, act="RELU")
    y = b.fc(b.pool(x), 6, act="RELU")
    x = b.mul(b.pw(x, 8), b.unary("LOGISTIC", b.pw(y, 8)))
    x = b.concat([b.unary("HARD_SWISH", x), b.unary("RELU6", b.pw(x, 4))])
    x = b.add(b.resize(x, 5, 7, "align_corners"), b.resize(b.pw(x, 12), 5, 7, "half_pixel"))
    x = b.tconv(b.mul(x, x), 4)
    b.pw(b.resize(x, 6, 9), 1)
    return b


@pytest.mark.parametrize("fp16", [False, True])
def test_generated_graph_reads_back(tmp_path, fp16):
    b = every_op_graph(fp16)
    path = b.write(str(tmp_path / "g.tflite"))
    g = tg.load(path)
    assert [t["shape"] for t in b.tensors] == [t.shape for t in g.tensors]
    assert [t["dtype"] for t in b.tensors] == [t.dtype for t in g.tensors]
    for t, u in zip(b.tensors, g.tensors):
        assert (t["data"] is None) == (u.data is None)
        if t["data"] is not None:
            assert t["data"].tobytes() == u.data.tobytes()
    assert [(o["kind"], o["inputs"], o["outputs"]) for o in b.ops] == [(o.kind, o.inputs, o.outputs) for o in g.ops]
    for o, u in zip(b.ops, g.ops):
        for k, v in o.get("opts", {}).items():
            if k == "padding":
                assert u.opts[k] == v
            elif k == "keep_num_dims" or k in u.opts:
                assert u.opts[k] == v, (o["kind"], k)
        if o["kind"] == "CUSTOM":
            assert (u.opts["stride_w"], u.opts["stride_h"], u.opts["padding_c_enum"]) == (2, 2, 1)
    assert {"DEQUANTIZE" in [o.kind for o in g.ops]} == {fp16}
    # the C oracle's loader: same shapes, constants (f16 widened through DEQUANTIZE), op structure
    m = po.Model(path)
    assert m.n_tensors == len(b.tensors) and m.n_ops == len(b.ops)
    assert m.input == b.x and m.output == b.ops[-1]["outputs"][0]
    for i, t in enumerate(b.tensors):
        assert m.shape(i) == t["shape"]
        if t["data"] is not None and t["dtype"] != "i32":
            assert np.array_equal(m.tensor(i).reshape(-1), t["data"].astype(np.float32))
    for i, o in enumerate(b.ops):
        _, ins, out = m.op(i)
        assert ins == o["inputs"][:4] and out == o["outputs"][0]
    x = np.random.default_rng(0).uniform(0, 1, (8, 10, 3)).astype(np.float32)
    from tests import torch_graph
    assert np.abs(m.invoke(x)[0] - torch_graph.run(path, x)).max() < 1e-5
    m.close()


@pytest.mark.parametrize("key", sorted(MODELS))
def test_bundled_models_reserialised(tmp_path, key):
    g = tg.load(model_path(key))
    path = str(tmp_path / os.path.basename(model_path(key)))
    with open(path, "wb") as f:
        f.write(tw.from_graph(g))
    h = tg.load(path)
    assert len(h.tensors) == len(g.tensors) and len(h.ops) == len(g.ops)
    for t, u in zip(g.tensors, h.tensors):
        assert (t.shape, t.dtype, t.name) == (u.shape, u.dtype, u.name)
        assert (t.data is None) == (u.data is None) and (t.data is None or t.data.tobytes() == u.data.tobytes())
    for o, u in zip(g.ops, h.ops):
        assert (o.kind, o.inputs, o.outputs, o.opts) == (u.kind, u.inputs, u.outputs, u.opts)
    a, b = po.Model(model_path(key)), po.Model(path)
    rng = np.random.default_rng(2)
    for _ in range(2):
        x = rng.uniform(-1 if key == "deeplab" else 0, 1, a.shape(a.input)).astype(np.float32)
        assert np.array_equal(a.invoke(x).view(np.uint32), b.invoke(x).view(np.uint32)), key
    a.close(); b.close()
