"""The host-side planning rules of the CUDA library, read from ramba_b200/csrc: each rule that several kernel families
share (which operand slots hold values, the row-broadcast hoist, the row split of axis reductions, the global-reduction
scratch header, the stencil group test) is stated in one place; no two host functions share a name; and the C-ABI file
holds no interpreter planning."""
import collections
import os
import re

HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(HERE, "..", "ramba_b200", "csrc")

# a definition at the start of a line: qualifiers / return type, name, parameters, body
_DEF = re.compile(r"^(?!\s)((?:template\s*<[^>]*>\s*)?[\w:<>,*&\s]*?)\b(\w+)\s*\(([^;{}]*?)\)\s*(?:const\s*)?\{", re.M)
_NOT_NAMES = {"if", "for", "while", "switch", "return"}


def _strip(src):
    """Comments and string literals removed (line structure kept)."""
    src = re.sub(r"/\*.*?\*/", lambda m: "\n" * m.group(0).count("\n"), src, flags=re.S)
    src = re.sub(r"//[^\n]*", "", src)
    return re.sub(r'"(?:\\.|[^"\\])*"', '""', src)


def _sources():
    for name in sorted(os.listdir(CSRC)):
        if name.endswith((".cu", ".cuh", ".h")):
            with open(os.path.join(CSRC, name)) as f:
                yield name, _strip(f.read())


def _host_defs(src):
    """(offset, name) of every host function defined at file level."""
    out = []
    for m in _DEF.finditer(src):
        quals, name = m.group(1), m.group(2)
        if name in _NOT_NAMES or "__global__" in quals or ("__device__" in quals and "__host__" not in quals):
            continue
        out.append((m.start(), name))
    return out


def _enclosing(pattern):
    """{(file, function)} of the host functions whose bodies match pattern."""
    where = set()
    for name, src in _sources():
        defs = _host_defs(src)
        for m in re.finditer(pattern, src):
            fn = [n for off, n in defs if off < m.start()]
            where.add((name, fn[-1] if fn else None))
    return where


def test_value_slots_are_stated_once():
    """RED's b is its reduction slot and SINCOS's c its store target; every planner asks value_slot."""
    assert _enclosing(r"(?:RB200_OP_RED|LO_RED)\s*&&\s*q\s*==\s*1|\b(?:I\.op|lop)\s*!=\s*(?:RB200_OP_RED|LO_RED)\b") == {("rb200_plan.h", "value_slot")}
    assert _enclosing(r"RB200_OP_SINCOS\s*&&\s*q\s*==\s*2|\bI\.op\s*!=\s*RB200_OP_SINCOS\b") == {("rb200_plan.h", "value_slot")}


def test_row_split_is_stated_once():
    assert _enclosing(r"/\s*(?:\w+\.)?n_chunks\b") == {("rb200_plan.h", "row_split")}


def test_row_broadcast_hoist_is_stated_once():
    """Only the shared hoist turns a view operand into a register operand."""
    assert _enclosing(r"_kind\s*=\s*(?:RB200_K_REG|L_REG)\b") == {("rb200_plan.h", "hoist_row_broadcast")}


def test_global_reduction_scratch_is_stated_once():
    assert _enclosing(r"red_scratch\s*\+|\b256\s*\+\s*8\s*\*") == {("rb200_plan.h", "bind_red_scratch")}
    for const in ("kRedScratchPartials", "kRedScratchHeader"):
        defs = [name for name, src in _sources() for _ in re.finditer(r"\b%s\s*=" % const, src)]
        assert defs == ["rb200_plan.h"], (const, defs)
    assert not [name for name, src in _sources() if "max_red_blocks" in src]


def test_stencil_group_test_is_stated_once():
    """The +-3 / +-8 / +-8 shift window of a stencil group member."""
    hits = [name for name, src in _sources() for _ in re.finditer(r"-3\b[^\n]*\b3\b[^\n]*-8\b[^\n]*\b8\b[^\n]*-8\b[^\n]*\b8\b", src)]
    assert hits == ["rb200_tile.cu"], hits


def test_no_two_host_functions_share_a_name():
    where = collections.defaultdict(list)
    for name, src in _sources():
        for _, fn in _host_defs(src):
            where[fn].append(name)
    assert "plan_stream" in where and "plan_stencil_tile" in where  # (the scan sees the planners)
    dups = {fn: files for fn, files in where.items() if len(files) > 1}
    assert not dups, dups


def test_the_c_abi_file_holds_no_interpreter_planning():
    with open(os.path.join(CSRC, "rb200_api.cu")) as f:
        api = {fn for _, fn in _host_defs(_strip(f.read()))}
    assert not api & {"plan_axis_as_1d", "assign_handlers", "static_kind"}, api
    assert {"validate", "make_plan", "launch"} <= api
