"""Host checks of the training-step kernel tests (tests/exact_train_kernels.py): the argument checks of `pcb_ce_forward_backward` and
`pcb_gather_sum`, which return before anything touches a device, and the case lists and CPU generators."""
import torch

from tests import exact_train_kernels as X


def _lib():
    from pointcontrast_b200 import _lib
    return _lib


def test_ce_rejects_wide_rows_and_empty_batches():
    L = _lib()
    n, C = 9, 20
    x, t, loss, g = torch.zeros(n, 1025), torch.zeros(n, dtype=torch.int64), torch.zeros(1), torch.zeros(n, 1025)
    wsb = L.lib.pcb_ce_ws_bytes(n)
    ws = torch.zeros(wsb, dtype=torch.uint8)

    def call(n=n, C=C):
        return L.lib.pcb_ce_forward_backward(x.data_ptr(), t.data_ptr(), n, C, 255, 1.0, loss.data_ptr(), g.data_ptr(), ws.data_ptr(),
                                             wsb, None)
    for rc in (call(C=1025), call(n=0), call(C=0)):
        assert rc == L.ERR_ARG and b"bad argument" in L.lib.pcb_last_error()


def test_gather_sum_rejects_channels_not_a_multiple_of_4():
    L = _lib()
    x, y, cnt = torch.zeros(16, 32), torch.zeros(16, 32), torch.zeros(16)
    tbl = torch.zeros(1, 16, dtype=torch.int32)

    def call(C, ld=32):
        return L.lib.pcb_gather_sum(x.data_ptr(), ld, tbl.data_ptr(), 16, None, 1, 16, C, y.data_ptr(), ld, cnt.data_ptr(), None)
    for C in (1, 2, 6, 27, 30):
        assert call(C) == L.ERR_ARG and b"bad argument" in L.lib.pcb_last_error()


def test_case_lists_reach_every_row_geometry():
    classes = {"one partial CTA", "whole CTAs", "partial last CTA"}
    for C in X.CE_C:
        assert {X.ce_n_class(n) for n in X.ce_n_list(C)} == classes, C
    for C in X.L2_C:
        assert {X.ce_n_class(n) for n in X.l2_n_list(C)} == classes, C
    assert {20, 13} <= set(X.CE_C) and X.CE_BIG_N % 8 == 3 and abs(X.CE_BIG_N - 10 ** 6) < 8
    assert max(X.CE_C) == 1024 and any(32 < C < 64 for C in X.CE_C)                 # a second lane pass, the widest row
    assert {n % 4 for n in X.SGD_N} == {0, 1, 2, 3}
    big = [n for n in X.SGD_N if n > 2 ** 21]
    assert {n % 4 for n in big} == {1, 3} and all(abs(n - 2 ** 22) < 4 for n in big)


def test_ce_target_mixes_hold_their_kinds():
    for C in X.CE_C:
        for n in (9, 4099):
            for mix in X.CE_MIXES:
                gen = torch.Generator().manual_seed(C + n)
                t = X.ce_targets(mix, n, C, gen)
                ign = X.ce_ignore(mix, C)
                v = X.ce_valid(t, C, ign)
                if mix == "all ignored":
                    assert not bool(v.any())
                elif mix == "valid":
                    assert bool((v == (t != 255)).all())           # 255 is a class, and the ignore_index, when C > 255
                elif mix == "out of range":
                    assert {C, -1, -5} <= set(t.tolist()) and bool(v.any())
                else:
                    assert bool((t == ign).any()) and (bool(v.any()) or C == 1) and (mix == "ignore 255") == (ign == 255)
                    assert (ign < C) == (mix == "ignore inside" or C > 255)


def test_ce_dominated_rows_are_exactly_representable():
    for C in X.CE_C:
        for mix in X.CE_MIXES:
            gen = torch.Generator().manual_seed(C)
            t = X.ce_targets(mix, 64, C, gen)
            x, jmax = X.ce_dominated(t, C, gen)
            xd = x.double()
            fin = torch.isfinite(xd)
            assert bool((xd[fin] == xd[fin].round()).all() & (xd[fin].abs() <= X.XMAX).all())
            M = xd.max(1).values
            assert bool((xd[torch.arange(64), jmax] == M).all())
            rest = xd.clone()
            rest[torch.arange(64), jmax] = -float("inf")
            assert bool((rest <= (M - X.MARGIN)[:, None]).all())
            valid = (t >= 0) & (t < C)
            assert bool(torch.isfinite(xd[torch.arange(64)[valid], t[valid]]).all())
            if C > 1:
                assert bool((~fin).any())
