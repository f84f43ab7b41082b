"""serializer.py -- checkpoint / resume in ModelSerializer's container (reference J:606-618, SURVEY.md 8f #1).

DL4J's `ModelSerializer.writeModel(net, file, saveUpdater)` writes a zip with `configuration.json`, `coefficients.bin` = `Nd4j.write(net.params())`
and `updaterState.bin` = `Nd4j.write(updater state view)`.  This module writes the same container with the same two array payloads:

  coefficients.bin   the flattened parameter row vector [1, numParams] in DL4J's flatten order (what b2g_net_get_params returns), in ND4J's
                     stream format: for the shape-info buffer and then the data buffer  writeUTF(allocationMode) | writeLong(length) |
                     writeUTF(dataType) | big-endian elements  (BaseDataBuffer.write of nd4j 1.0.0-beta3, allocation mode LONG_SHAPE; restated
                     from memory -- no JVM here to pin it: PARITY UNPINNED like the rest of the DL4J semantics, see DESIGN.md 1)
  updaterState.bin   the updater state, same format.  Layout = this library's [state0 | state1] (RmsProp cache / Adam m, then Adam v), each in
                     parameter order, and a third slot [state0 | state1 | state2] (AMSGrad's v-hat) when some layer uses AMSGrad; the slot
                     each updater kind uses is stated at b2g_updater in include/b200gan.h -- NOT DL4J's per-UpdaterBlock interleaving; a DL4J
                     reader must regroup it
  configuration.json this library's layer specification (the arguments of b2g_net_create), NOT DL4J's Jackson schema: a Java user rebuilds the
                     graph with the same builder calls (the driver's own code, J:118-310) and loads the arrays.  An updater's learning-rate
                     schedule is part of its spec (a MapSchedule as a list of [key, value] pairs)
  b200gan.json       precision, input shape, iteration counter, dropout pass counter, epoch count

`read_model` reads the container back (and accepts legacy int-length headers), so the library can resume training -- the reference can only save.
"""
from __future__ import annotations

import io
import json
import struct
import zipfile
from typing import Dict, Optional, Sequence

import numpy as np


def _write_utf(out, s: str):
    b = s.encode("utf-8"); out.write(struct.pack(">H", len(b))); out.write(b)          # DataOutputStream.writeUTF (ASCII subset)


def _read_utf(inp) -> str:
    (n,) = struct.unpack(">H", inp.read(2)); return inp.read(n).decode("utf-8")


def _write_buffer(out, arr: np.ndarray, dtype_name: str):
    _write_utf(out, "LONG_SHAPE"); out.write(struct.pack(">q", arr.size)); _write_utf(out, dtype_name)
    be = {"LONG": ">i8", "FLOAT": ">f4", "DOUBLE": ">f8", "INT": ">i4"}[dtype_name]
    out.write(np.ascontiguousarray(arr).astype(be).tobytes())


def _read_buffer(inp) -> np.ndarray:
    mode = _read_utf(inp)
    n = struct.unpack(">i", inp.read(4))[0] if mode in ("DIRECT", "HEAP", "JAVACPP") else struct.unpack(">q", inp.read(8))[0]
    t = _read_utf(inp)
    be = {"LONG": ">i8", "FLOAT": ">f4", "DOUBLE": ">f8", "INT": ">i4"}[t]
    return np.frombuffer(inp.read(n * np.dtype(be).itemsize), be).astype(be[1:])


def write_nd4j_row_vector(out, v: np.ndarray):
    """Nd4j.write(INDArray [1,n] 'c' float): shape-info buffer {rank, shape..., stride..., offset, elementWiseStride, order} then the data."""
    v = np.asarray(v, np.float32).ravel(); n = v.size
    shape_info = np.array([2, 1, n, n, 1, 0, 1, ord("c")], np.int64)
    _write_buffer(out, shape_info, "LONG"); _write_buffer(out, v, "FLOAT")


def read_nd4j_array(inp) -> np.ndarray:
    info = _read_buffer(inp).astype(np.int64); rank = int(info[0]); shape = tuple(int(x) for x in info[1:1 + rank]); order = chr(int(info[-1]))
    data = _read_buffer(inp)
    return np.asarray(data).reshape(shape, order="F" if order == "f" else "C")


def write_model(path, specs: Sequence[Dict], input_shape, params: np.ndarray, updater_state: Optional[np.ndarray] = None, meta: Optional[Dict] = None):
    with zipfile.ZipFile(path, "w", zipfile.ZIP_DEFLATED) as z:
        z.writestr("configuration.json", json.dumps({"format": "b200gan layer specs (arguments of b2g_net_create), not DL4J's Jackson schema",
                                                      "input_shape": list(input_shape), "layers": list(specs)}, indent=1))
        b = io.BytesIO(); write_nd4j_row_vector(b, params); z.writestr("coefficients.bin", b.getvalue())
        if updater_state is not None:
            b = io.BytesIO(); write_nd4j_row_vector(b, updater_state); z.writestr("updaterState.bin", b.getvalue())
        z.writestr("b200gan.json", json.dumps(dict(meta or {}, num_params=int(np.asarray(params).size))))


def read_model(path) -> Dict:
    with zipfile.ZipFile(path) as z:
        names = set(z.namelist())
        cfg = json.loads(z.read("configuration.json"))
        out = {"specs": cfg["layers"], "input_shape": tuple(cfg["input_shape"]), "params": read_nd4j_array(io.BytesIO(z.read("coefficients.bin"))).ravel(),
               "updater_state": read_nd4j_array(io.BytesIO(z.read("updaterState.bin"))).ravel() if "updaterState.bin" in names else None,
               "meta": json.loads(z.read("b200gan.json")) if "b200gan.json" in names else {}}
    if out["meta"].get("num_params", out["params"].size) != out["params"].size:
        raise ValueError("coefficients.bin does not hold num_params values")
    return out


def save_net(net, path, specs: Sequence[Dict], input_shape, save_updater: bool = True, meta: Optional[Dict] = None):
    """ModelSerializer.writeModel(net, file, saveUpdater) for a gan_deeplearning4j_b200.Net (anything with params() / updater_state())."""
    write_model(path, specs, input_shape, net.params(), net.updater_state() if save_updater else None, meta)


def restore_into(net, path, load_updater: bool = True) -> Dict:
    """ModelSerializer.restoreComputationGraph for an already constructed net of the same architecture: parameters (and updater state) are set."""
    m = read_model(path)
    if m["params"].size != net.num_params():
        raise ValueError(f"checkpoint holds {m['params'].size} parameters, the net has {net.num_params()}")
    net.set_params(m["params"])
    if load_updater and m["updater_state"] is not None:
        net.set_updater_state(m["updater_state"])
        # Adam's bias correction depends on the iteration count: warm moments with t = 1 would diverge from an uninterrupted run
        if "iteration" in m["meta"] and hasattr(net, "set_iteration"):
            net.set_iteration(int(m["meta"]["iteration"]))
    # the DropoutLayer pass counter: a resumed run draws the masks an uninterrupted one would have drawn
    if "dropout_pass" in m["meta"] and hasattr(net, "set_dropout_pass"):
        net.set_dropout_pass(int(m["meta"]["dropout_pass"]))
    # the epoch count EPOCH learning-rate schedules read
    if "epoch" in m["meta"] and hasattr(net, "set_epoch"):
        net.set_epoch(int(m["meta"]["epoch"]))
    # the loss layer's per-output weights (new LossMCXENT(weights), ...) are part of its configuration
    if m["specs"] and m["specs"][-1].get("type") in ("output", "loss", "cnn_loss") and hasattr(net, "set_loss_weights"):
        net.set_loss_weights(m["specs"][-1].get("loss_weights"))
    return m
