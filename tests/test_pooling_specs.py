"""CPU checks of the pooling layers' interfaces: the spec builders' b2g_layer_desc codes, the codes in include/b200gan.h, the Python maps and the
Java facade agree; the builders refuse what the engine would; a checkpoint round-trips the new specs."""
import os
import re

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
JAVA = os.path.join(ROOT, "java", "src", "main", "java", "org", "deeplearning4j", "nn", "conf", "layers")


def _header():
    return re.sub(r"/\*.*?\*/", "", open(os.path.join(ROOT, "include", "b200gan.h")).read(), flags=re.S)


def test_header_codes_match_the_python_maps():
    from gan_deeplearning4j_b200 import engine
    h = _header()
    assert int(re.search(r"B2G_LAYER_SUBSAMPLING\s*=\s*(\d+)", h).group(1)) == engine.LAYER_TYPES["subsampling"] == 12
    assert int(re.search(r"B2G_LAYER_GLOBAL_POOLING\s*=\s*(\d+)", h).group(1)) == engine.LAYER_TYPES["global_pooling"] == 13
    for name, code in engine.POOLINGS.items():
        assert int(re.search(rf"B2G_POOL_{name.upper()}\s*=\s*(\d+)", h).group(1)) == code
    assert int(re.search(r"B2G_TEST_POOL2D\s*=\s*(\d+)", h).group(1)) == engine.POOL_TEST_OPS["pool2d"] == 0
    assert int(re.search(r"B2G_TEST_GLOBAL_POOL\s*=\s*(\d+)", h).group(1)) == engine.POOL_TEST_OPS["global_pool"] == 1
    assert re.search(r"#define B2G_VERSION 101\b", open(os.path.join(ROOT, "include", "b200gan.h")).read())


def test_test_pool_struct_matches_the_c_header(tmp_path):
    import ctypes as C
    import subprocess
    from gan_deeplearning4j_b200 import _lib
    T = _lib.TestPoolOpts
    prog = tmp_path / "layout.c"
    prog.write_text('#include <stdio.h>\n#include <stddef.h>\n#include "b200gan.h"\nint main(){' +
                    "".join(f'printf("%zu\\n", offsetof(b2g_test_pool_opts,{f}));' for f, _ in T._fields_) +
                    'printf("%zu\\n", sizeof(b2g_test_pool_opts));return 0;}')
    exe = tmp_path / "layout"
    subprocess.run(["gcc", "-I", os.path.join(ROOT, "include"), str(prog), "-o", str(exe)], check=True)
    got = [int(v) for v in subprocess.run([str(exe)], capture_output=True, text=True).stdout.split()]
    assert got == [getattr(T, f).offset for f, _ in T._fields_] + [C.sizeof(T)]


def test_java_facade_codes():
    from gan_deeplearning4j_b200 import engine
    kinds = re.search(r"enum PoolingType \{([^}]*)\}", open(os.path.join(JAVA, "PoolingType.java")).read()).group(1)
    assert [k.strip().lower() for k in kinds.split(",")] == sorted(engine.POOLINGS, key=engine.POOLINGS.get)
    sub = open(os.path.join(JAVA, "SubsamplingLayer.java")).read()
    assert "l.type = t == PoolingType.MAX ? 5 : 12" in sub and "t.ordinal()" in sub and "pnorm(int p)" in sub
    glb = open(os.path.join(JAVA, "GlobalPoolingLayer.java")).read()
    assert "l.type = 13" in glb and "l.alpha = 2" in glb and "collapseDimensions(boolean" in glb and "public Builder()" in glb
    assert "DESC_BYTES = 4 + 64 + 4 * 2 + 4 * 6 + 4 + 4 + 4 + 4 + 4 * 4 + 4 + 4 * 2 + 4 * 3 + 4 * 2;" in open(os.path.join(JAVA, "Layer.java")).read()


@pytest.mark.parametrize("pooling,code", [("avg", 1), ("sum", 2), ("pnorm", 3)])
def test_subsampling_desc(pooling, code):
    from gan_deeplearning4j_b200 import engine, models as m
    d = engine.layer_desc(m.subsampling(pooling, (3, 2), (2, 1), (1, 0), pnorm=3 if pooling == "pnorm" else None, name="s"))
    assert (d.type, d.act, d.k_h, d.k_w, d.s_h, d.s_w, d.p_h, d.p_w) == (12, code, 3, 2, 2, 1, 1, 0)
    if pooling == "pnorm":
        assert d.act_alpha == 3.0


@pytest.mark.parametrize("pooling,code", [("max", 0), ("avg", 1), ("sum", 2), ("pnorm", 3)])
def test_global_pooling_desc(pooling, code):
    from gan_deeplearning4j_b200 import engine, models as m
    d = engine.layer_desc(m.global_pooling(pooling, 4, name="g"))
    assert (d.type, d.act) == (13, code)
    assert d.act_alpha == (4.0 if pooling == "pnorm" else 2.0)
    d = engine.layer_desc({"type": "global_pooling", "name": "g"})               # GlobalPoolingLayer.Builder(): MAX, p = 2
    assert (d.act, d.act_alpha) == (0, 2.0)


def test_builders_refuse_what_the_engine_refuses():
    from gan_deeplearning4j_b200 import models as m
    with pytest.raises(ValueError):
        m.subsampling("max", (2, 2))                    # SubsamplingLayer(MAX) is the maxpool spec
    with pytest.raises(ValueError):
        m.subsampling("pnorm", (2, 2))                  # PNORM needs p
    with pytest.raises(ValueError):
        m.global_pooling("median")
    from gan_deeplearning4j_b200 import engine
    d = engine.layer_desc({"type": "subsampling", "name": "s", "pooling": "pnorm", "kernel": (2, 2), "stride": (2, 2)})
    assert d.act_alpha == 0.0                           # no p given: the engine's B2G_ERR_ARG


def test_dcgan_discriminator_global_pooling_head():
    from gan_deeplearning4j_b200 import models as m
    base = m.dcgan_discriminator(32, 16, 3)
    assert base == m.dcgan_discriminator(32, 16, 3, global_pooling=None)      # today's head by default
    for kind in ("sum", "avg"):
        d = m.dcgan_discriminator(32, 16, 3, loss="mse", global_pooling=kind)
        assert d[:-2] == base[:-2]
        assert d[-2] == {"type": "global_pooling", "name": "dis_global_pool", "pooling": kind}
        assert d[-1]["type"] == "output" and d[-1]["n_out"] == 1 and d[-1]["loss"] == "mse"
    assert m.forward_macs(m.dcgan_discriminator(32, 16, 3, global_pooling="sum"), (3, 32, 32)) == \
        m.forward_macs(base, (3, 32, 32)) - 4 * 4 * 64 + 64


def test_checkpoint_round_trip(tmp_path):
    from gan_deeplearning4j_b200 import engine, models as m, serializer
    specs = m.dcgan_discriminator(16, 8, 3, global_pooling="pnorm")[:-2] + [
        dict(m.subsampling("pnorm", (3, 3), (2, 2), (1, 1), pnorm=3), name="s"), dict(m.global_pooling("pnorm", 5), name="g"),
        {"type": "output", "name": "o", "n_out": 1}]
    params = np.arange(10, dtype=np.float32)
    serializer.write_model(tmp_path / "c.zip", specs, (3, 16, 16), params, None, {"iteration": 3})
    back = serializer.read_model(tmp_path / "c.zip")
    assert len(back["specs"]) == len(specs)
    fields = [f for f, _ in engine.LayerDesc._fields_]
    for a, b in zip(specs, back["specs"]):
        da, db = engine.layer_desc(a), engine.layer_desc(b)
        assert [getattr(da, f) for f in fields] == [getattr(db, f) for f in fields], a
    assert np.array_equal(back["params"], params)
