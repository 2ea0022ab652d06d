"""VoteNet loss, host side (csrc/det_loss.cu, DESIGN.md 8f-12): the ctypes mirrors of `pcb_det_loss_args` / `pcb_strided` have the C
compiler's layout, and pcb_det_loss_forward / _backward reject bad arguments with PCB_ERR_ARG before touching the device."""
import ctypes
import os
import shutil
import subprocess

from pointcontrast_b200 import _lib, build

HEADER = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "include", "pcb200.h")
FAKE = 256                                   # never dereferenced: every call below fails its checks before any CUDA call


def test_struct_layouts_match_the_c_compiler(tmp_path):
    structs = {"pcb_det_loss_args": _lib.PcbDetLossArgs, "pcb_strided": _lib.PcbStrided}
    lines = ['#include <stdio.h>', '#include <stddef.h>', '#include "pcb200.h"', "int main(void) {"]
    for cname, cls in structs.items():
        lines.append(f'  printf("{cname} sizeof %zu 0\\n", sizeof(struct {cname}));')
        for field, _ in cls._fields_:
            lines.append(f'  printf("{cname} {field} %zu %zu\\n", offsetof(struct {cname}, {field}), sizeof(((struct {cname}*)0)->{field}));')
    lines += ["  return 0;", "}"]
    src = tmp_path / "abi.c"
    src.write_text("\n".join(lines) + "\n")
    exe = tmp_path / "abi"
    cc = shutil.which("cc") or shutil.which(build.NVCC)
    assert cc
    subprocess.run([cc, "-I", os.path.dirname(HEADER), str(src), "-o", str(exe)], check=True, capture_output=True, text=True)
    got = {}
    for line in subprocess.run([str(exe)], check=True, capture_output=True, text=True).stdout.splitlines():
        cname, field, off, size = line.split()
        got.setdefault(cname, []).append((field, int(off), int(size)))
    for cname, cls in structs.items():
        py = [("sizeof", ctypes.sizeof(cls), 0)] + [(f, getattr(cls, f).offset, getattr(cls, f).size) for f, _ in cls._fields_]
        assert py == got[cname], cname


def valid_args(B=2, S=16, V=1, N=100, K=8, K2=4, NH=1, NS=3, C=5):
    a = _lib.PcbDetLossArgs(B, S, V, N, K, K2, NH, NS, C, 0, 1.0)
    ms = (ctypes.c_float * (3 * NS))(*([1.0] * 3 * NS))
    a.mean_size = ctypes.addressof(ms)
    for f, t in _lib.PcbDetLossArgs._fields_:
        if t is ctypes.c_void_p and f != "mean_size":
            setattr(a, f, FAKE)
        elif t is _lib.PcbStrided:
            setattr(a, f, _lib.PcbStrided(FAKE, 1, 1, 1, 1))
    a.center_label_ld = 3
    return a, ms


def fwd(a, ws=None, sb=None):
    B, S, K, K2 = a.B, a.S, a.K, a.K2
    ws = _lib.lib.pcb_det_loss_ws_bytes(B, S, K, K2) if ws is None else ws
    sb = _lib.lib.pcb_det_loss_state_bytes(B, S, K, K2) if sb is None else sb
    return _lib.lib.pcb_det_loss_forward(ctypes.byref(a), FAKE, FAKE, FAKE, FAKE, FAKE, sb, FAKE, ws, None)


def bwd(a, sb=None):
    sb = _lib.lib.pcb_det_loss_state_bytes(a.B, a.S, a.K, a.K2) if sb is None else sb
    return _lib.lib.pcb_det_loss_backward(ctypes.byref(a), FAKE, FAKE, FAKE, FAKE, FAKE, sb, *([None] * 9), None)


def test_bad_arguments_return_status_2():
    assert _lib.lib.pcb_det_loss_ws_bytes(8, 1024, 256, 64) > 0 and _lib.lib.pcb_det_loss_ws_bytes(0, 1024, 256, 64) == 0
    assert _lib.lib.pcb_det_loss_state_bytes(8, 1024, 256, 64) >= 4 * (8 * (1024 + 256 + 64))
    assert _lib.lib.pcb_det_loss_forward(None, FAKE, FAKE, FAKE, FAKE, FAKE, 1 << 20, FAKE, 1 << 20, None) == _lib.ERR_ARG
    for field, value in (("B", 0), ("B", 65536), ("S", 0), ("V", 0), ("N", 0), ("K", 0), ("K2", 0), ("NH", 0), ("NS", 0), ("NS", 65),
                         ("C", 0), ("center_label_ld", 2), ("seed_inds", None), ("vote_label", None), ("box_label_mask", None),
                         ("mean_size", None), ("N", 1 << 28)):
        a, ms = valid_args()
        setattr(a, field, value)
        assert fwd(a) == _lib.ERR_ARG, field
        assert bwd(a) == _lib.ERR_ARG, field
    a, ms = valid_args()
    a.sem_cls_scores = _lib.PcbStrided(None, 1, 1, 1, 1)
    assert fwd(a) == _lib.ERR_ARG and bwd(a) == _lib.ERR_ARG
    a, ms = valid_args()
    assert fwd(a, ws=_lib.lib.pcb_det_loss_ws_bytes(2, 16, 8, 4) - 1) == _lib.ERR_ARG           # short workspace
    assert fwd(a, sb=_lib.lib.pcb_det_loss_state_bytes(2, 16, 8, 4) - 1) == _lib.ERR_ARG        # short state
    assert bwd(a, sb=_lib.lib.pcb_det_loss_state_bytes(2, 16, 8, 4) - 1) == _lib.ERR_ARG
    assert _lib.lib.pcb_det_loss_backward(ctypes.byref(a), None, FAKE, FAKE, FAKE, FAKE, 1 << 20, *([None] * 9), None) == _lib.ERR_ARG
