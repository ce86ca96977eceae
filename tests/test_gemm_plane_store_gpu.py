"""The two ways of writing a GELU + two-bf16-plane output give the same bits.

Under the ping-pong schedule, whole tiles whose rows are consecutive output rows (plain GEMMs, and
convolutions whose tiles span whole image rows) stage each plane's 64 x 64 boxes in shared memory
and write them with TMA stores; everything else, and every tile of the cooperative schedule, takes
the register stores.  So each case runs under both schedules (TAPIR_B200_GEMM_SCHEDULE) into
NaN-filled buffers, at both tile widths, and the planes must match bit for bit, padding included.
The operands are tests/gemm_exact.py's GELU designs, whose accumulators are exact."""
import pytest
import torch

pytestmark = pytest.mark.gpu

from tests import gemm_exact as E  # noqa: E402
from tests import gpu_util as U  # noqa: E402

# name: (make_design arguments, ld_pad)
CASES = {
    # mixer `up`'s N and K
    'up': (dict(M=2048, N=2048, K=512), 0),
    # the last m-tile is partial and takes the register stores
    'ragged_m': (dict(M=1000, N=256, K=512), 0),
    # the ExtraConv GELU + planes layer at 32 x 32: tiles of four whole image rows
    'extra_conv_up': (dict(M=None, N=1024, K=None, conv=(1, 32, 32, 256)), 0),
    # tiles 8 pixels wide in a 40-pixel image: their rows are not consecutive, register stores
    'conv_narrow_tiles': (dict(M=None, N=128, K=None, conv=(2, 16, 40, 64)), 0),
    # plane leading dimension larger than N (still a multiple of 8 elements)
    'ld_pad': (dict(M=1024, N=256, K=256), 8),
    # several frames of whole-row tiles
    'frames': (dict(M=None, N=256, K=None, conv=(3, 16, 16, 64)), 0),
}


_designs = {}


def _design(name):
  if name not in _designs:
    kw, _ = CASES[name]
    d = E.make_design('G', sum(map(ord, name)), P=2, **kw)
    d.dev = dict(a=d.a_pl.cuda(), w=d.w_pl.cuda(), bias=d.bias.cuda())
    _designs[name] = d
  return _designs[name]


def _run(name, schedule, bn, bias):
  d = _design(name)
  _, ld_pad = CASES[name]
  with U.switches(TAPIR_B200_GEMM_SCHEDULE=schedule, TAPIR_B200_BLOCK_N=bn):
    res = U.gemm(d.dev['a'], d.dev['w'], d.dev['bias'] if bias else None, None, True, out_f32=False,
                 out_planes=2, conv=d.conv, ld_pad=ld_pad, details=True)
  assert res.launches == 1
  return res


@pytest.mark.parametrize('bias', [True, False], ids=['bias', 'nobias'])
@pytest.mark.parametrize('bn', [128, 64])
@pytest.mark.parametrize('name', sorted(CASES))
def test_tma_and_register_plane_stores_agree(name, bn, bias):
  regs = _run(name, 'coop', bn, bias)
  tma = _run(name, 'pingpong', bn, bias)
  assert torch.equal(regs.planes_buf.view(torch.int16), tma.planes_buf.view(torch.int16)), name
  assert U.untouched_padding(tma), name
  assert not torch.isnan(tma.planes.float()).any(), name
