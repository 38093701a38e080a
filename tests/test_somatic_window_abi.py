"""CPU: the somatic window pass's structs in include/strelka_b200.h against their ctypes / numpy mirrors -- sizes and every field's offset, as a C
compiler lays them out."""
import ctypes as C
import os
import shutil
import subprocess

import pytest

from strelka_b200 import _abi as A

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))

# (C type, mirror, [field names])
STRUCTS = [
    ("sx_somatic_window_batch", A.SxSomaticWindowBatch, [n for n, _ in A.SxSomaticWindowBatch._fields_]),
    ("sx_somatic_window_out", A.SxSomaticWindowOut, [n for n, _ in A.SxSomaticWindowOut._fields_]),
    ("sx_somatic_site_call", A.SOMATIC_SITE_CALL_DT, list(A.SOMATIC_SITE_CALL_DT.names)),
    ("sx_somatic_indel_call", A.SOMATIC_INDEL_CALL_DT, list(A.SOMATIC_INDEL_CALL_DT.names)),
]


def _mirror_layout(m, fields):
    if isinstance(m, type):
        return C.sizeof(m), [getattr(m, f).offset for f in fields]
    return m.itemsize, [m.fields[f][1] for f in fields]


@pytest.fixture(scope="module")
def c_layout(tmp_path_factory):
    cc = shutil.which("cc") or shutil.which("gcc")
    if cc is None:
        pytest.skip("no C compiler")
    d = tmp_path_factory.mktemp("swin_abi")
    lines = ['#include <stddef.h>', '#include <stdio.h>', '#include "strelka_b200.h"', "int main(void) {"]
    for name, _, fields in STRUCTS:
        lines.append(f'printf("%zu", sizeof({name}));')
        for f in fields:
            lines.append(f'printf(" %zu", offsetof({name}, {f}));')
        lines.append('printf("\\n");')
    lines += [f'printf("%d %d\\n", SX_SWIN_TOTALS, SX_SWIN_N_STAGES);', "return 0; }"]
    src = d / "layout.c"
    src.write_text("\n".join(lines))
    exe = d / "layout"
    subprocess.check_call([cc, "-std=c99", "-I", os.path.join(ROOT, "include"), str(src), "-o", str(exe)])
    return subprocess.check_output([str(exe)], text=True).split("\n")


def test_struct_layouts(c_layout):
    for (name, mirror, fields), line in zip(STRUCTS, c_layout):
        got = [int(x) for x in line.split()]
        size, offsets = _mirror_layout(mirror, fields)
        assert got == [size] + offsets, name


def test_constants(c_layout):
    assert [int(x) for x in c_layout[len(STRUCTS)].split()] == [A.SX_SWIN_TOTALS, A.SX_SWIN_N_STAGES]
    assert len(A.SX_SWIN_STAGE_NAMES) == A.SX_SWIN_N_STAGES


def test_record_sizes():
    """the record layouts the host filter and sx_gatherv_records move as bytes"""
    assert A.SOMATIC_SITE_CALL_DT.itemsize == 16 + A.SSNV_RESULT_DT.itemsize == 304
    assert A.SOMATIC_INDEL_CALL_DT.itemsize == 8 + A.SINDEL_RESULT_DT.itemsize == 408
