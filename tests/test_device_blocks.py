"""The device-side building blocks of the lean kernels, read from ramba_b200/csrc: the strided load of a direct view,
the common operand kinds (spill register, scalar, accumulator), the read of a staged stream tile and the stencil group's
plane loader are each written once, in rb200_lean.cuh or next to their kernels, and every kernel calls that one copy."""
import os
import re

HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(HERE, "..", "ramba_b200", "csrc")


def _strip(src):
    """Comments removed (line structure kept)."""
    src = re.sub(r"/\*.*?\*/", lambda m: "\n" * m.group(0).count("\n"), src, flags=re.S)
    return re.sub(r"//[^\n]*", "", src)


def _read(name):
    with open(os.path.join(CSRC, name)) as f:
        return _strip(f.read())


def _hits(pattern):
    """[file, ...] with one entry per match of pattern across the library's sources."""
    out = []
    for name in sorted(os.listdir(CSRC)):
        if name.endswith((".cu", ".cuh", ".h", ".inc")):
            out += [name] * len(re.findall(pattern, _read(name)))
    return out


def _body(src, name):
    """The text of the function or kernel `name`, from its name to its closing brace."""
    m = re.search(r"\b%s\s*\(" % name, src)
    assert m, name
    i = src.index("{", m.end())
    depth = 0
    for j in range(i, len(src)):
        depth += {"{": 1, "}": -1}.get(src[j], 0)
        if depth == 0:
            return src[m.start():j + 1]
    raise AssertionError(name)


def test_direct_view_load_is_written_once():
    """The valid-masked strided load of an LDirect view: ldirect_load only."""
    assert _hits(r"\?\s*\(F\)ldg<(?:float|double)>\(p\)") == ["rb200_lean.cuh"] * 2


def test_context_stores_use_the_shared_direct_store():
    for name in ("rb200_stream.cu", "rb200_tile.cu"):
        assert "ldirect_store<F, LV>" in _body(_read(name), "store_view"), name
    assert not re.search(r"\bstg<", _read("rb200_tile.cu"))
    assert not re.search(r"\bterm_store\b", _read("rb200_tile.cu"))


def test_common_operand_kinds_are_written_once():
    """Spill-register addressing and scalar bits -> class: LeanRegs and scal_as only."""
    assert _hits(r"reg_s\s*\+\s*\(unsigned\)\w+\s*\*\s*\(LV \* kThreads \* 8\)") == ["rb200_lean.cuh"] * 2
    assert _hits(r"__longlong_as_double\(\(long long\)\w+\)\s*:\s*\(F\)__uint_as_float") == ["rb200_lean.cuh"]
    for name in ("rb200_stream.cu", "rb200_tile.cu"):
        assert re.search(r"struct \w+Ctx : LeanRegs", _read(name)), name


def test_staged_stream_tile_read_is_written_once():
    assert _hits(r"lean_lds<float>\([^;]*k \* kThreads \* 4\)") == ["rb200_stream.cu"]


def test_stencil_plane_loader_is_written_once():
    tile = _read("rb200_tile.cu")
    assert len(re.findall(r"\btma_load_3d\(", tile)) == 2  # its definition and its one call, in tile_request
    assert len(re.findall(r"\bcp_async[48]\(", tile)) == 2  # the cooperative fill, one call per element size
    assert "tma_load_3d(" in _body(tile, "tile_request") and "cp_async4(" in _body(tile, "tile_request")
    kernel = _body(tile, "stencil_tile_kernel")
    assert not re.search(r"\bcp_async[48]\(|\btma_load_3d\(", kernel)
    assert "tile_request<TE>(" in kernel
