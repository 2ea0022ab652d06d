"""The Python side of the C ABI against include/pcb200.h: every integer `#define PCB_*` has its constant in `_lib`, and the ctypes
mirrors of `struct pcb_unit` / `struct pcb_tile_desc` have the C compiler's size and field offsets.  A mismatch would pass the library
wrong flags or make it read the wrong pointer, with no error."""
import ctypes
import os
import re
import shutil
import subprocess

from pointcontrast_b200 import _lib, build

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
HEADER = os.path.join(ROOT, "include", "pcb200.h")


def test_lib_has_every_integer_define_of_the_header():
    hdr = re.sub(r"/\*.*?\*/", "", open(HEADER).read(), flags=re.S)
    defines = dict(re.findall(r"^\s*#define\s+PCB_(\w+)\s+(-?\d+)\s*$", hdr, flags=re.M))
    assert len(defines) >= 18
    for name, value in defines.items():
        assert getattr(_lib, name, None) == int(value), f"_lib.{name} != PCB_{name} ({value})"


def test_struct_layouts_match_the_c_compiler(tmp_path):
    structs = {"pcb_unit": _lib.PcbUnit, "pcb_tile_desc": _lib.PcbTileDesc}
    lines = ['#include <stdio.h>', '#include "pcb200.h"', "int main(void) {"]
    for cname, cls in structs.items():
        lines.append(f'  printf("{cname} sizeof %zu %zu\\n", sizeof(struct {cname}), (size_t)0);')
        for field, _ in cls._fields_:
            lines.append(f'  printf("{cname} {field} %zu %zu\\n", offsetof(struct {cname}, {field}), '
                         f"sizeof(((struct {cname}*)0)->{field}));")
    lines += ["  return 0;", "}"]
    src = tmp_path / "abi.c"
    src.write_text("\n".join(lines) + "\n")
    exe = tmp_path / "abi"
    cc = shutil.which("cc") or shutil.which(build.NVCC)
    assert cc, f"no C compiler: neither cc nor {build.NVCC} (which the library build needs) was found"
    subprocess.run([cc, "-I", os.path.dirname(HEADER), str(src), "-o", str(exe)], check=True, capture_output=True, text=True)
    out = subprocess.run([str(exe)], check=True, capture_output=True, text=True).stdout
    c_layout = {}
    for line in out.splitlines():
        cname, field, off, size = line.split()
        c_layout.setdefault(cname, []).append((field, int(off), int(size)))
    for cname, cls in structs.items():
        py = [("sizeof", ctypes.sizeof(cls), 0)] + [(f, getattr(cls, f).offset, getattr(cls, f).size) for f, _ in cls._fields_]
        assert py == c_layout[cname], cname
