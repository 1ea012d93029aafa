"""CPU tests: the C-ABI library builds for sm_90a, loads, exports every symbol include/s4g.h
declares, and fails LOUDLY (no CPU fallback) when there is no CUDA device."""
import ctypes
import os
import subprocess

import pytest

from super4pcs_b200 import s4g


def test_library_exports_every_declared_symbol(s4g_lib):
    declared = s4g.declared_symbols()
    assert len(declared) >= 20
    assert set(s4g.exported_symbols()) == set(declared)
    assert s4g_lib.s4g_abi_version() == 1


def test_library_is_sm90a_cuda_code(s4g_lib):
    out = subprocess.run(["cuobjdump", "--list-elf", s4g.lib_path()], capture_output=True, text=True)
    if out.returncode != 0:
        pytest.skip("cuobjdump unavailable")
    assert "sm_90a" in out.stdout


def test_result_struct_layout_matches_header():
    # s4g_tcs_result: u64, u32, i32, u32, u32, float[16], float, float[3], float[3]
    # 8 + 4*4 + 64 + 4 + 12 + 12 + 16 = 132, padded to the 8-byte alignment of the u64 key
    assert ctypes.sizeof(s4g.TcsResult) == 136
    assert s4g.TcsResult.best_T.offset == 24


def test_no_cpu_fallback(s4g_lib):
    import torch
    if torch.cuda.is_available():
        pytest.skip("GPU present")
    with pytest.raises(s4g.S4GError):
        s4g.Context(0)


def test_product_does_not_touch_oracle():
    """nothing under super4pcs_b200/, include/ or the C++ layer may reference oracle/"""
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    bad = []
    for top in ("super4pcs_b200", "include", "cpp"):
        for dp, _, fns in os.walk(os.path.join(root, top)):
            for fn in fns:
                if fn.endswith((".py", ".cu", ".cuh", ".h", ".hpp", ".cc", ".cpp")):
                    txt = open(os.path.join(dp, fn), errors="ignore").read()
                    if "oracle" in txt.replace("oracle/ ", "").lower() and ("import oracle" in txt or "from oracle" in txt
                                                                            or "liboracle" in txt or "oracle/" in txt):
                        bad.append(os.path.join(dp, fn))
    assert not bad, bad


def test_header_is_plain_c(tmp_path):
    """the drop-in boundary is a C ABI: include/s4g.h must compile as C99 (no C++, no CUDA or torch types), and a C
    program that only includes it must link against libs4g.so"""
    import subprocess
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    hdr = os.path.join(root, "include", "s4g.h")
    subprocess.check_call(["gcc", "-std=c99", "-Wall", "-Wextra", "-pedantic", "-Werror", "-fsyntax-only", "-x", "c", hdr])
    src = tmp_path / "probe.c"
    src.write_text('#include <stdio.h>\n#include "s4g.h"\nint main(void) {\n  s4g_ctx* c = 0;\n  int rc = s4g_create(0, &c);\n'
                   '  printf("abi %d rc %d\\n", s4g_abi_version(), rc);\n  if (rc == S4G_OK) s4g_destroy(c);\n  return 0;\n}\n')
    exe = tmp_path / "probe"
    libdir = os.path.join(root, "super4pcs_b200", "lib")
    subprocess.check_call(["gcc", "-std=c99", "-I", os.path.join(root, "include"), str(src), "-o", str(exe), "-L", libdir, "-ls4g",
                           "-Wl,-rpath," + libdir])
    out = subprocess.run([str(exe)], capture_output=True, text=True, timeout=120)
    assert out.returncode == 0 and out.stdout.startswith("abi 1 rc ")


def test_comm_entry_points_without_a_device(s4g_lib):
    """row e inside the library: NCCL is resolved on first use (dlopen), never at load time; without a context the
    calls refuse cleanly.  (The reduction itself needs GPUs: tests/test_comm_gpu.py.)"""
    import ctypes as C
    import subprocess
    from super4pcs_b200 import s4g
    needed = subprocess.run(["objdump", "-p", s4g.lib_path()], capture_output=True, text=True).stdout
    assert "libnccl" not in needed                      # no NEEDED entry: a caller that never shards never loads NCCL
    L = s4g.load_library()
    assert L.s4g_comm_info(None, None) == 2 and L.s4g_comm_destroy(None) == 2 and L.s4g_comm_init_all(None, 0) == 2
    buf = (C.c_ubyte * s4g.COMM_ID_BYTES)()
    rc = L.s4g_comm_unique_id(buf)
    assert rc in (0, 5)                                 # S4G_OK with an NCCL on the box, S4G_ERR_COMM without -- never a crash
    if rc == 0:
        assert any(buf)
