"""CPU: the C-ABI shared library loads and exports every symbol include/b2l.h declares; without a GPU the
product fails loudly (no CPU fallback).  No compute calls here."""
import ctypes
import os
import re

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def declared_symbols():
    text = open(os.path.join(ROOT, "include", "b2l.h")).read()
    text = re.sub(r"/\*.*?\*/", "", text, flags=re.S)
    return sorted(set(re.findall(r"\b(b2l_[a-z0-9_]+)\s*\(", text)))


def test_header_declares_the_hot_path():
    syms = declared_symbols()
    for name in ["b2l_stft", "b2l_istft", "b2l_melspectrogram", "b2l_mfcc", "b2l_plan_create", "b2l_ctx_create",
                 "b2l_comm_scatter", "b2l_comm_gather"]:
        assert name in syms


def test_library_exports_every_declared_symbol():
    from librosa_b200 import _native as nat

    lib = nat.lib()
    missing = [s for s in declared_symbols() if not hasattr(lib, s)]
    assert not missing, f"libb2l.so is missing {missing}"
    # and the ctypes layer binds exactly the declared set
    assert sorted(nat.EXPORTED_SYMBOLS) == declared_symbols()
    assert lib.b2l_version() == 100


def test_plan_desc_layout_matches_header():
    from librosa_b200 import _native as nat

    # int32 x4, ptr, int32 (+pad), ptr, float, int32, ptr, float x3  -> 72 bytes on LP64
    assert ctypes.sizeof(nat.PlanDesc) == 72
    assert nat.PlanDesc.h_window.offset == 16 and nat.PlanDesc.h_mel_basis.offset == 32
    assert nat.PlanDesc.h_dct_basis.offset == 48 and nat.PlanDesc.top_db.offset == 64


def _header_enumerators():
    text = re.sub(r"/\*.*?\*/", "", open(os.path.join(ROOT, "include", "b2l.h")).read(), flags=re.S)
    return [n for body in re.findall(r"\benum\b[^{;]*\{(.*?)\}", text, flags=re.S)
            for n in re.findall(r"\b(B2L_[A-Z0-9_]+)\b", body)]


def _mirror(nat, name):
    """The _native constant that mirrors the header's enumerator ``name``."""
    short = name[len("B2L_"):]
    for prefix, table in (("PAD_", nat.PAD_MODES), ("DTW_", nat.DTW_METRICS)):
        if short.startswith(prefix):
            return table[short[len(prefix):].lower()]
    return getattr(nat, name) if hasattr(nat, name) else getattr(nat, short)


def test_ctypes_mirror_matches_header(tmp_path):
    """Every ctypes.Structure of _native has the size and field offsets of the struct its docstring names (field
    names as in C), and every enumerator of include/b2l.h has the value of its _native constant: a C99 probe
    compiled against the header prints what C sees."""
    import shutil
    import subprocess

    from librosa_b200 import _native as nat

    if shutil.which("gcc") is None:
        pytest.skip("gcc not available")
    structs = {}
    for cls in vars(nat).values():
        if isinstance(cls, type) and issubclass(cls, ctypes.Structure) and cls is not ctypes.Structure:
            tag = re.match(r"struct (b2l_\w+) ", cls.__doc__ or "")
            assert tag, f"{cls.__name__}: the docstring must name its C struct"
            structs[tag.group(1)] = cls
    assert len(structs) >= 19
    enums = _header_enumerators()
    assert "B2L_STATUS_NEGATIVE_EVENT" in enums
    lines = ['#include <stddef.h>', '#include <stdio.h>', '#include "b2l.h"', "int main(void) {"]
    want = {}
    for tag, cls in structs.items():
        lines.append(f'  printf("{tag} %zu\\n", sizeof(struct {tag}));')
        want[tag] = ctypes.sizeof(cls)
        for field, *_ in cls._fields_:
            lines.append(f'  printf("{tag}.{field} %zu\\n", offsetof(struct {tag}, {field}));')
            want[f"{tag}.{field}"] = getattr(cls, field).offset
    for name in enums:
        lines.append(f'  printf("{name} %d\\n", (int){name});')
        want[name] = int(_mirror(nat, name))
    lines += ["  return 0;", "}"]
    src = tmp_path / "probe.c"
    src.write_text("\n".join(lines) + "\n")
    exe = tmp_path / "probe"
    subprocess.run(["gcc", "-std=c99", "-Wall", "-Werror", "-I", os.path.join(ROOT, "include"), str(src), "-o",
                    str(exe)], check=True, capture_output=True)
    got = dict(line.split() for line in subprocess.run([str(exe)], check=True, capture_output=True,
                                                       text=True).stdout.splitlines())
    assert {k: int(v) for k, v in got.items()} == want


def _have_gpu():
    from librosa_b200 import _native as nat

    n = ctypes.c_int()
    return nat.lib().b2l_device_count(ctypes.byref(n)) == 0 and n.value > 0


@pytest.mark.skipif(_have_gpu(), reason="only meaningful on a box without a GPU")
def test_no_cpu_fallback():
    import librosa_b200 as lb

    y = np.zeros(4096, dtype=np.float32)
    for fn in (lambda: lb.stft(y), lambda: lb.feature.melspectrogram(y=y), lambda: lb.feature.mfcc(y=y),
               lambda: lb.istft(np.zeros((1025, 4), dtype=np.complex64))):
        with pytest.raises(lb.NativeLibraryError):
            fn()


def test_product_does_not_import_the_oracle():
    """Only tests/, __graft_entry__.smoke() and bench.py's CPU legs may touch oracle/."""
    pkg = os.path.join(ROOT, "librosa_b200")
    pat = re.compile(r"^\s*(from|import)\s+oracle\b|oracle\.ref_np|#include\s+\"[^\"]*oracle", re.M)
    for dirpath, _, files in os.walk(pkg):
        for f in files:
            if f.endswith((".py", ".cu", ".cuh", ".h")):
                src = open(os.path.join(dirpath, f)).read()
                assert not pat.search(src), f"{os.path.join(dirpath, f)} references the oracle"


def _build_c_demo(tmp_path):
    import shutil
    import subprocess

    if shutil.which("gcc") is None:
        pytest.skip("gcc not available")
    exe = tmp_path / "c_abi_demo"
    cmd = ["gcc", "-std=c99", "-Wall", "-Werror", "-I", os.path.join(ROOT, "include"),
           os.path.join(ROOT, "examples", "c_abi_demo.c"), "-L", os.path.join(ROOT, "librosa_b200", "csrc"), "-lb2l", "-lm",
           "-o", str(exe)]
    subprocess.run(cmd, check=True, capture_output=True)
    return exe


def test_header_is_plain_c_and_links_from_a_c_program(tmp_path):
    """include/b2l.h compiles as C99 (no C++ / torch types in the signatures) and every symbol the demo uses
    resolves against libb2l.so; running it needs a GPU (tests/test_gpu_parity.py)."""
    exe = _build_c_demo(tmp_path)
    assert exe.exists()


@pytest.mark.gpu
def test_c_program_runs_on_the_gpu(tmp_path):
    import subprocess

    exe = _build_c_demo(tmp_path)
    env = dict(os.environ, LD_LIBRARY_PATH=os.path.join(ROOT, "librosa_b200", "csrc") + ":" + os.environ.get("LD_LIBRARY_PATH", ""))
    out = subprocess.run([str(exe)], env=env, capture_output=True, text=True, timeout=120)
    assert out.returncode == 0, out.stdout + out.stderr
    assert "C ABI demo: OK" in out.stdout
