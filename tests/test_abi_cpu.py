"""CPU-side checks of the drop-in boundary: the CUDA library loads without a GPU, exports every
entry point include/swarmdb_b200.h declares, struct layouts match the header, and construction
fails loudly (no CPU fallback) when no device is present."""
import ctypes as C
import re
from pathlib import Path

import pytest

ROOT = Path(__file__).resolve().parents[1]


def _declared():
    text = (ROOT / "include" / "swarmdb_b200.h").read_text()
    text = re.sub(r"/\*.*?\*/", "", text, flags=re.S)
    return sorted(set(re.findall(r"\b(sdb_[a-z_0-9]+)\s*\(", text)))


def test_library_exports_every_declared_symbol():
    from swarmdb_b200 import _native
    lib = _native.load_library()
    names = _declared()
    assert len(names) >= 24
    missing = [n for n in names if not hasattr(lib, n)]
    assert not missing, missing
    assert sorted(_native.EXPORTS) == names           # the binding lists exactly the declared ABI
    assert lib.sdb_abi_version() == 1


def test_struct_layouts_match_header():
    from swarmdb_b200 import _native
    assert C.sizeof(_native.SdbConfig) == 96            # sizeof(sdb_config), checked against gcc
    assert _native.HDR_DTYPE.itemsize == 32
    assert [n for n in _native.HDR_DTYPE.names] == ["seq", "timestamp", "sender", "receiver", "group", "len", "prio", "type"]
    assert C.sizeof(_native.SdbStats) == 80


def test_no_cpu_fallback_without_device():
    import torch
    if torch.cuda.is_available():
        pytest.skip("a GPU is present")
    from swarmdb_b200 import _native
    with pytest.raises(_native.SdbError) as e:
        _native.Shard(16)
    assert "no CPU fallback" in str(e.value)
    import swarmdb_b200
    with pytest.raises(_native.SdbError):
        swarmdb_b200.SwarmsDB(save_dir="/tmp/sdb_nogpu", auto_save=False)


def test_product_never_imports_the_oracle():
    for p in (ROOT / "swarmdb_b200").rglob("*.py"):
        src = p.read_text()
        assert "oracle" not in re.sub(r"#.*", "", src).replace("oracle/", ""), p
    for p in (ROOT / "swarmdb_b200" / "csrc").glob("*.cu*"):
        code = re.sub(r"//.*", "", p.read_text())            # comments may cite the oracle, code may not use it
        assert "oracle" not in code and "cpu_ref" not in code, p
    mk = (ROOT / "swarmdb_b200" / "csrc" / "Makefile").read_text()
    assert "oracle" not in mk


def test_wire_codec_roundtrip_is_host_only():
    """The content/extras codec of core.py (replaces the JSON envelope M:466 / M:575-576)."""
    from swarmdb_b200 import core
    body, flags = core._encode_content({"a": [1, 2]})
    assert flags == core.TYPEF_JSON and body == b'{"a": [1, 2]}'
    body, flags = core._encode_content("héllo")
    assert flags == 0 and body.decode() == "héllo"
    m = core.Message(sender_id="a", content="x")
    d = m.to_dict()
    assert d["type"] == "chat" and d["priority"] == 1 and d["status"] == "pending"
    assert core.Message.from_dict(d).sender_id == "a"


def _build_c_demo(tmp_path):
    import shutil
    import subprocess
    from pathlib import Path
    if shutil.which("gcc") is None:
        pytest.skip("gcc not available")
    root = Path(__file__).resolve().parents[1]
    exe = tmp_path / "c_abi_demo"
    subprocess.check_call(["gcc", "-std=c99", "-Wall", "-Wextra", "-Werror", "-pedantic", f"-I{root / 'include'}",
                           str(root / "examples" / "c_abi_demo.c"), f"-L{root / 'swarmdb_b200' / 'csrc'}", "-lswarmdb_b200",
                           f"-Wl,-rpath,{root / 'swarmdb_b200' / 'csrc'}", "-o", str(exe)])
    return exe


def test_header_is_plain_c_and_a_c_caller_fails_loudly_without_a_device(tmp_path):
    """include/swarmdb_b200.h compiles as strict C99 and links against the library; without a CUDA device the
    caller gets SDB_ECUDA and a message - never a silent CPU path."""
    import subprocess
    import torch
    exe = _build_c_demo(tmp_path)
    if torch.cuda.is_available():
        pytest.skip("a device is present: covered by tests/test_gpu_api.py::test_plain_c_caller")
    p = subprocess.run([str(exe)], capture_output=True, text=True)
    assert p.returncode == 3 and "sizeof(sdb_config)=96" in p.stdout and "no CPU fallback" in p.stdout, p.stdout


def test_every_environment_switch_of_the_library_is_documented():
    """INTEGRATION.md section 5 lists the A/B switches the library reads with getenv; a new one must be written down."""
    import re
    from pathlib import Path
    root = Path(__file__).resolve().parents[1]
    names = set()
    for f in (root / "swarmdb_b200" / "csrc").glob("*.cu"):
        names |= set(re.findall(r'getenv\("([A-Z0-9_]+)"\)', f.read_text()))
    doc = (root / "INTEGRATION.md").read_text()
    missing = sorted(n for n in names if f"`{n}`" not in doc)
    assert names and not missing, missing
    from swarmdb_b200._native import shared_payload_enabled
    import os
    old = os.environ.get("SDB_SHARED_PAYLOAD")
    try:
        os.environ["SDB_SHARED_PAYLOAD"] = "0"; assert not shared_payload_enabled()
        os.environ["SDB_SHARED_PAYLOAD"] = "1"; assert shared_payload_enabled()
        os.environ.pop("SDB_SHARED_PAYLOAD"); assert shared_payload_enabled()          # the library's default
    finally:
        if old is not None:
            os.environ["SDB_SHARED_PAYLOAD"] = old


def _extern_c(text):
    """(name, has_body) of every function declared with C linkage in C++ source text: after an extern "C" specifier, or
    at the top level of an extern "C" { } block."""
    text = re.sub(r"/\*.*?\*/", "", re.sub(r"//[^\n]*", "", text), flags=re.S)
    text = re.sub(r"^\s*#[^\n]*", "", text, flags=re.M)

    def close(i, o, c):                                      # index of the bracket closing the one at i
        depth = 0
        for k in range(i, len(text)):
            depth += (text[k] == o) - (text[k] == c)
            if depth == 0:
                return k

    def decl(i):                                             # the declaration whose parameter list opens at i
        head = re.split(r"[;{}]", text[:i])[-1]
        k = close(i, "(", ")") + 1
        return re.findall(r"\w+", head)[-1], text[k:].lstrip()[:1] == "{", k, re.search(r"\bstatic\b", head)

    out = []
    for m in re.finditer(r'extern\s+"C"\s*', text):
        i = m.end()
        if text[i] != "{":
            out.append(decl(text.index("(", i))[:2])
            continue
        k, end = i + 1, close(i, "{", "}")
        while k < end:
            if text[k] == "{":
                k = close(k, "{", "}") + 1
            elif text[k] == "(":
                name, body, k, internal = decl(k)
                if not internal:                             # static functions have no linkage to check
                    out.append((name, body))
            else:
                k += 1
    return out


def test_launchers_are_declared_once_where_their_definitions_see_them():
    """The two-level scan layout is defined once, and every extern "C" function one source defines for another is declared
    in sdb_common.cuh, which every source includes: C linkage has no name mangling, so a prototype the defining file
    never sees would let a changed signature link and pass wrong arguments."""
    csrc = ROOT / "swarmdb_b200" / "csrc"
    files = sorted(csrc.glob("*.cu")) + sorted(csrc.glob("*.cuh"))
    assert sum(p.read_text().count("#define SDB_SCAN_TILE") for p in files) == 1
    common = (csrc / "sdb_common.cuh").read_text()
    block = re.search(r'extern "C" \{(.*?)\n\}', common, flags=re.S).group(1)
    declared = set(re.findall(r"(\w+)\s*\(", re.sub(r"//[^\n]*", "", block)))
    public = set(_declared())
    defined = set()
    for p in sorted(csrc.glob("*.cu")):
        fns = _extern_c(p.read_text())
        assert all(body for _, body in fns), (p.name, [n for n, body in fns if not body])
        defined |= {n for n, _ in fns}
    assert len(defined) > 60
    assert sorted(defined - public - declared) == []
