"""Host checks of the fused executor's unit schedule (`fused.schedule`, no GPU): it issues the units tests/exact_unit.py restates, in
order and with the same gradient modes, it refuses models not wired like Res16UNet, and every unit takes its neighbour tables from its
own kernel generator."""
import pytest
import torch

from pointcontrast_b200 import fused, me
from pointcontrast_b200.model import load_model, res16unet
from tests import exact_unit as XU
from tests.refload import default_config


def _meta_model(name="Res16UNet34C", in_channels=3):
    with torch.device("meta"):
        return load_model(name)(in_channels, 32, default_config(), D=3)


def _sig(sched, u):
    """exact_unit's signature of a schedule entry (fp16 off, training, two views)."""
    sliced = lambda b: isinstance(b, int) and sched.units[b].out is not None        # a column slice: row stride != width
    kind = "stem" if not u.tc else "up" if u.transpose else {27: "k27", 8: "down", 1: "k1"}[u.K]
    return XU.Sig(kind, u.K, u.Cin, u.Cout, u.relu, u.res is not None, u.need_f32, u.gres_mode, u.gin_mode, False, False, True,
                  sliced(u.x), u.out is not None, u.out is not None, u.gin_mode > 0 and sliced(u.x), u.gres_mode > 0 and sliced(u.res))


@pytest.mark.parametrize("name", XU.MODELS)
def test_schedule_issues_the_restated_units_in_order(name):
    m = _meta_model(name)
    sched = fused.schedule(m)
    assert sched is not None and fused.matches(m) and fused.schedule(m) is sched
    assert tuple(_sig(sched, u) for u in sched.units) == XU.model_units(name)
    assert sched.final.conv is m.final and sched.final.x == len(sched.units) - 1 and sched.final.tc
    # one plan per (levels, kernel generator, transpose): 5 3x3x3 + 5 1x1 + 4 down + 4 up + the stem
    assert len({u.plan_key for u in sched.units + (sched.final,)}) == 19


def _with_conv3(m):
    m.block2[0].conv3 = res16unet._conv(64, 64, 3, hybrid=True)


def _with_three_module_downsample(m):
    m.block2[0].downsample.append(me.MinkowskiReLU())


def _with_width_48(m):
    blk = m.block1[0]
    blk.conv1, blk.norm1 = res16unet._conv(32, 48, 3, hybrid=True), me.MinkowskiBatchNorm(48)
    blk.conv2 = res16unet._conv(48, 32, 3, hybrid=True)


def _with_k27_final(m):
    m.final = res16unet._conv(m.PLANES[7], 32, 3, bias=True)


def _without_bn3(m):
    del m.bn3


@pytest.mark.parametrize("variant", [_with_conv3, _with_three_module_downsample, _with_width_48, _with_k27_final, _without_bn3, None],
                         ids=["conv3", "downsample3", "width48", "final_k27", "no_bn3", "stem32"])
def test_schedule_refuses_other_wirings(variant):
    with torch.device("meta"):
        if variant is None:
            m = _meta_model(in_channels=32)          # a tensor-core stem: the executor's stem unit is the exact fp32 one
        else:
            m = _meta_model()
            variant(m)
    assert fused.schedule(m) is None and not fused.matches(m)


def test_each_unit_takes_the_tables_of_its_own_kernel_generator():
    """A block whose convolutions use HYPERCUBE generators among HYBRID ones: the same 27 offsets in another order, so the block's
    units need tables of their own."""
    m = _meta_model()
    with torch.device("meta"):
        blk = m.block3[1]
        blk.conv1, blk.conv2 = res16unet._conv(128, 128, 3), res16unet._conv(128, 128, 3)
    assert blk.conv1.kernel_generator.cache_key != m.block3[0].conv1.kernel_generator.cache_key
    sched = fused.schedule(m)
    assert sched is not None
    for u in sched.units + (sched.final,):
        assert u.plan_key == (u.level_in, u.level_out, u.conv.kernel_generator.cache_key, u.conv.is_transpose)
    cube = [u for u in sched.units if u.conv in (blk.conv1, blk.conv2)]
    assert len(cube) == 2 and all(u.plan_key[:2] == (3, 3) for u in cube)
    assert len({u.plan_key for u in sched.units + (sched.final,)}) == 20
