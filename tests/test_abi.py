"""The C-ABI library loads and exports every symbol include/zeekstd_b200.h declares (no compute calls: no GPU here)."""
import os
import re

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def declared_symbols():
    h = open(os.path.join(ROOT, "include", "zeekstd_b200.h")).read()
    h = re.sub(r"/\*.*?\*/", "", h, flags=re.S)
    names = set(re.findall(r"\b(zk_[a-z0-9_]+)\s*\(", h))
    names -= {"zk_write_fn", "zk_flush_fn"}
    return sorted(names)


def test_header_and_binding_agree():
    from zeekstd_b200 import _native
    assert declared_symbols() == _native.EXPORTED_SYMBOLS


def test_product_library_exports_every_symbol():
    from zeekstd_b200 import _native
    from zeekstd_b200.build import build_product
    so = build_product()                      # nvcc cross-compiles for sm_90a without a GPU
    lib = _native.load(so)
    for name in declared_symbols():
        assert hasattr(lib, name), name
    assert b"sm_90a" in lib.zk_version()


def test_product_library_contains_sm90a_sass():
    import subprocess
    from zeekstd_b200 import _native
    out = subprocess.run(["cuobjdump", "-lelf", _native.PRODUCT_SO], capture_output=True, text=True).stdout
    assert "sm_90a" in out


def test_no_device_is_an_error_not_a_fallback():
    import ctypes
    import torch
    from zeekstd_b200 import _native
    if torch.cuda.is_available():
        pytest.skip("a GPU is present")
    lib = _native.load(_native.PRODUCT_SO)
    h = ctypes.c_void_p()
    rc = lib.zk_ctx_create(0, 0, ctypes.byref(h))
    assert rc == -1005 and not h.value        # ZK_ERR_NO_DEVICE


def test_product_never_links_the_oracle():
    import subprocess
    from zeekstd_b200 import _native
    out = subprocess.run(["nm", "-D", _native.PRODUCT_SO], capture_output=True, text=True).stdout
    assert "zko_" not in out and "zkr_" not in out and "ZSTD_" not in out
    for d, _, files in os.walk(os.path.join(ROOT, "zeekstd_b200")):
        for f in files:
            if f.endswith((".cu", ".cuh", ".cpp", ".h", ".py")):
                txt = open(os.path.join(d, f)).read()
                assert "zko_" not in txt and "zkr_" not in txt and "dlopen" not in txt and "libzstd.so" not in txt, f


def test_header_is_plain_c_and_cxx(tmp_path):
    """include/zeekstd_b200.h is what a foreign-language binding consumes: it must compile on its own as C99 and as C++11, and a C program
    that touches every declared function must LINK against the product library (no compute: nothing is called)"""
    import re
    import subprocess
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    hdr = os.path.join(root, "include", "zeekstd_b200.h")
    src = open(hdr).read()
    names = sorted(set(re.findall(r"\b(zk_[a-z0-9_]+)\s*\(", re.sub(r"/\*.*?\*/", "", src, flags=re.S))))
    names = [n for n in names if not n.endswith("_fn")]
    c = tmp_path / "use.c"
    c.write_text('#include "zeekstd_b200.h"\n#include <stdio.h>\nint main(void) {\n  const void* f[] = {' + ", ".join(f"(const void*)&{n}" for n in names)
                 + "};\n  printf(\"%u\\n\", (unsigned)(sizeof f / sizeof f[0]));\n  return 0;\n}\n")
    inc = ["-I", os.path.join(root, "include")]
    subprocess.run(["gcc", "-std=c99", "-Wall", "-Werror", "-fsyntax-only"] + inc + [str(c)], check=True, capture_output=True)
    subprocess.run(["g++", "-std=c++11", "-Wall", "-Werror", "-fsyntax-only", "-x", "c++"] + inc + [str(c)], check=True, capture_output=True)
    from zeekstd_b200 import _native
    if os.path.exists(_native.PRODUCT_SO):
        exe = tmp_path / "use"
        r = subprocess.run(["gcc", "-std=c99"] + inc + [str(c), "-o", str(exe), _native.PRODUCT_SO, "-Wl,--unresolved-symbols=ignore-in-shared-libs"], capture_output=True)
        assert r.returncode == 0, r.stderr.decode()
        assert len(names) > 60


def _build_c_example(tmp_path, so_path):
    import subprocess
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    exe = tmp_path / "roundtrip"
    r = subprocess.run(["gcc", "-std=c99", "-Wall", "-Wextra", "-Werror", "-I", os.path.join(root, "include"), os.path.join(root, "examples", "roundtrip.c"),
                        so_path, "-o", str(exe), "-Wl,-rpath," + os.path.dirname(so_path), "-Wl,--unresolved-symbols=ignore-in-shared-libs"], capture_output=True)
    assert r.returncode == 0, r.stderr.decode()
    return exe


def test_c_example_runs_on_the_emulation_build(tmp_path):
    """examples/roundtrip.c (Encoder with a sink callback -> archive -> Decoder over Seekable callbacks -> ranged + full reads), compiled as C99
    against the public header, run against the CPU emulation build of the sources"""
    import subprocess
    from zeekstd_b200.build import build_emul
    exe = _build_c_example(tmp_path, build_emul())
    r = subprocess.run([str(exe)], capture_output=True, timeout=300)
    assert r.returncode == 0 and r.stdout.startswith(b"ok: 100000 bytes"), (r.stdout, r.stderr)


def test_rust_sys_binding_is_in_sync():
    """bindings/rust/zeekstd_b200_sys.rs (generated by tools/gen_rust_sys.py; there is no rustc in this image to compile it) is up to date and
    declares exactly the functions of the public header -- the same list the Python binding and the product library are held to"""
    import importlib.util
    import re
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    spec = importlib.util.spec_from_file_location("gen_rust_sys", os.path.join(root, "tools", "gen_rust_sys.py"))
    gen = importlib.util.module_from_spec(spec); spec.loader.exec_module(gen)
    text, names = gen.generate()
    assert open(gen.OUT).read() == text, "run python tools/gen_rust_sys.py"
    hdr = re.sub(r"/\*.*?\*/", "", open(gen.HDR).read(), flags=re.S)
    declared = set(re.findall(r"\b(zk_[a-z0-9_]+)\s*\(", hdr)) - {"zk_write_fn", "zk_flush_fn"}
    assert set(names) == declared and len(names) == len(set(names)), sorted(declared ^ set(names))
    assert text.count("pub fn zk_") == len(names) and "*mut *mut zk_decoder" in text and "Option<unsafe extern \"C\" fn" in text
