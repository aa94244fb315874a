"""tower.supports() admits exactly the nets.BoardNet nets the fused engine can run: every packed convolution image within
MAX_BOARD_ROWS rows (width x cells), and tower BatchNorms whose weight, bias, running buffers and momentum the engine reads."""
import pytest
import torch

from handyrl_b200 import nets, tower
from handyrl_b200._capi import MAX_BOARD_ROWS


@pytest.mark.parametrize('kw,D', [
    (dict(board=(3, 3), width=32), 288),             # cfg2
    (dict(board=(4, 4), width=18, planes=20, return_head=True, actions=32), 288),
    (dict(board=(2, 5), width=28, actions=32), 280),
    (dict(board=(3, 3), width=8, depth=9), 72),
])
def test_nets_within_the_packed_rows_are_admitted(kw, D):
    net = nets.BoardNet(**kw)
    assert net.stem.out_channels * kw['board'][0] * kw['board'][1] == D <= MAX_BOARD_ROWS
    assert tower.supports(net)


@pytest.mark.parametrize('kw,D', [
    (dict(board=(2, 2), width=73), 292),             # the first multiple of 4 past the limit
    (dict(board=(4, 4), width=32), 512),
    (dict(board=(3, 3), width=64), 576),
])
def test_nets_past_the_packed_rows_are_refused(kw, D):
    net = nets.BoardNet(**kw)
    assert net.stem.out_channels * kw['board'][0] * kw['board'][1] == D > MAX_BOARD_ROWS
    assert not tower.supports(net)


@pytest.mark.parametrize('variant', [dict(affine=False), dict(track_running_stats=False), dict(momentum=None)])
def test_batchnorm_variants_the_engine_cannot_run_are_refused(variant):
    net = nets.BoardNet()
    assert tower.supports(net)
    net.tower[1][1] = torch.nn.BatchNorm2d(net.stem.out_channels, **variant)
    assert not tower.supports(net)


def test_head_limits_stay():
    assert tower.supports(nets.BoardNet(board=(4, 4), width=8, policy_maps=3, value_maps=1))          # 64 squeeze outputs
    assert not tower.supports(nets.BoardNet(board=(4, 4), width=8, policy_maps=4, value_maps=1))      # 80
    assert not tower.supports(nets.BoardNet(actions=33))
    assert not tower.supports(nets.BoardNet(board=(3, 6), width=8))                                   # 18 cells
