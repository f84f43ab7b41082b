"""CPU-side checks of the drop-in boundary: the C-ABI library loads, exports every symbol include/b200gan.h
declares, and its struct layouts agree with the ctypes mirror (the same layouts the Java facade writes into
direct ByteBuffers).  No compute calls: there is no GPU here and no CPU fallback to call."""
import ctypes as C
import os
import re
import subprocess
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.fixture(scope="module")
def lib():
    import gan_deeplearning4j_b200 as b
    if not os.path.exists(b.LIB_PATH):
        sys.path.insert(0, ROOT)
        import __graft_entry__
        __graft_entry__.build()
    return b.load()


def header_functions():
    src = open(os.path.join(ROOT, "include", "b200gan.h")).read()
    src = re.sub(r"/\*.*?\*/", "", src, flags=re.S)
    return sorted(set(re.findall(r"\b(b2g_[a-z0-9_]+)\s*\(", src)))


def test_every_declared_symbol_is_exported_and_bound(lib):
    import gan_deeplearning4j_b200 as b
    names = header_functions()
    assert len(names) >= 35
    for n in names:
        assert hasattr(lib, n), f"libb200gan.so does not export {n}"
    assert sorted(b.PROTOTYPES) == names, set(names) ^ set(b.PROTOTYPES)
    assert lib.b2g_version() == 101


def test_jni_symbols_exported_without_jni_h(lib):
    out = subprocess.run(["nm", "-D", "--defined-only", os.path.join(ROOT, "gan_deeplearning4j_b200", "lib", "libb200gan.so")], capture_output=True, text=True).stdout
    for n in ("ctxCreate", "netCreate", "netFit", "netOutput", "netSetParam", "netGetParam", "ganCreate", "ganStep", "ctxCommInit",
              "netSetUpdaterState", "netGetIteration", "netSetIteration", "netSetSyncBn", "netAverageParameters", "netEnableP2pAllreduce"):
        assert f"Java_org_deeplearning4j_b200_Native_{n}" in out


def test_struct_layouts_match_the_c_header(tmp_path):
    from gan_deeplearning4j_b200 import _lib
    prog = tmp_path / "layout.c"
    prog.write_text('#include <stdio.h>\n#include <stddef.h>\n#include "b200gan.h"\nint main(){'
                    'printf("%zu %zu %zu %zu %zu %zu %zu %zu %zu\\n", sizeof(b2g_layer_desc), offsetof(b2g_layer_desc,n_in), offsetof(b2g_layer_desc,updater),'
                    ' offsetof(b2g_layer_desc,pre_c), sizeof(b2g_net_config), offsetof(b2g_net_config,seed), sizeof(b2g_gan_config), sizeof(b2g_conv_geom), offsetof(b2g_net_config,bn_groups));'
                    'printf("%zu %zu %zu %zu %zu %zu %zu\\n", sizeof(b2g_test_conv_opts), offsetof(b2g_test_conv_opts,stats), offsetof(b2g_test_conv_opts,kernel),'
                    ' offsetof(b2g_test_conv_opts,bn), offsetof(b2g_test_conv_opts,max_ctas), offsetof(b2g_test_conv_opts,poison), offsetof(b2g_test_conv_opts,w_mn));'
                    'printf("%zu %zu %zu %zu\\n", offsetof(b2g_test_conv_opts,per_tap), offsetof(b2g_test_conv_opts,slab), offsetof(b2g_test_conv_opts,defer), offsetof(b2g_test_conv_opts,db));'
                    'printf("%zu %zu\\n", offsetof(b2g_test_conv_opts,param_offset), offsetof(b2g_test_conv_opts,splits));'
                    'printf("%zu %zu %zu\\n", sizeof(b2g_ew_reduce_job), offsetof(b2g_ew_reduce_job,splits), offsetof(b2g_ew_reduce_job,wide));'
                    + "".join(f'printf("%zu\\n", offsetof(b2g_test_ew_opts,{f}));' for f, _ in _lib.TestEwOpts._fields_) +
                    'printf("%zu\\n", sizeof(b2g_test_ew_opts));'
                    + "".join(f'printf("%zu\\n", offsetof(b2g_test_bn_opts,{f}));' for f, _ in _lib.TestBnOpts._fields_) +
                    'printf("%zu\\n", sizeof(b2g_test_bn_opts));return 0;}')
    exe = tmp_path / "layout"
    subprocess.run(["gcc", "-I", os.path.join(ROOT, "include"), str(prog), "-o", str(exe)], check=True)
    got = [int(v) for v in subprocess.run([str(exe)], capture_output=True, text=True).stdout.split()]
    L, N, T, E, J = _lib.LayerDesc, _lib.NetConfig, _lib.TestConvOpts, _lib.TestEwOpts, _lib.EwReduceJob
    assert got == [C.sizeof(L), L.n_in.offset, L.updater.offset, L.pre_c.offset, C.sizeof(N), N.seed.offset, C.sizeof(_lib.GanConfig), C.sizeof(_lib.ConvGeom), N.bn_groups.offset,
                   C.sizeof(T), T.stats.offset, T.kernel.offset, T.bn.offset, T.max_ctas.offset, T.poison.offset, T.w_mn.offset,
                   T.per_tap.offset, T.slab.offset, T.defer.offset, T.db.offset, T.param_offset.offset, T.splits.offset,
                   C.sizeof(J), J.splits.offset, J.wide.offset] + \
        [getattr(E, f).offset for f, _ in E._fields_] + [C.sizeof(E)] + \
        [getattr(_lib.TestBnOpts, f).offset for f, _ in _lib.TestBnOpts._fields_] + [C.sizeof(_lib.TestBnOpts)]
    assert (T.stats.offset, T.kernel.offset, T.bn.offset, T.slab.offset) == (56, 64, 128, 148)       # the fields older callers fill keep their offsets
    assert (T.defer.offset, T.db.offset) == (152, 160)
    assert (T.param_offset.offset, T.splits.offset, C.sizeof(T)) == (168, 172, 176)                 # appended after db


def test_no_device_fails_loudly_not_silently(lib):
    import torch
    if torch.cuda.is_available():
        pytest.skip("a GPU is present")
    import gan_deeplearning4j_b200 as b
    with pytest.raises(b.B200GanError) as e:
        b.Context(0)
    assert e.value.code == -7 and "no CPU fallback" in str(e.value)


def test_product_never_imports_the_oracle():
    pkg = os.path.join(ROOT, "gan_deeplearning4j_b200")
    for dirpath, _, files in os.walk(pkg):
        for f in files:
            if f.endswith((".py", ".cu", ".cuh", ".h", ".cpp")):
                txt = open(os.path.join(dirpath, f)).read()
                assert not re.search(r"^\s*(from|import)\s+oracle", txt, flags=re.M), f
