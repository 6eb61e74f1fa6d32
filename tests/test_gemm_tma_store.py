"""The GEMM's shared-memory store path (gemm_sm90.cuh): tiles whose 128 rows all lie below the live row count leave through
two 8 KB slots per consumer warpgroup and TMA bulk stores; the tile that straddles the live count stores straight from the
fragment.  Every A_2D epilogue that takes the new path (f16, SiLU, GLU, f32, dual-A), and the residual one (in place and
not) that stays on the direct path, against float64 at live counts around the 128-row block inside a larger buffer, at
tile counts that make every slot serve many tiles, in a column window of a wider buffer (TMA-aligned and not), and bit
for bit against the direct path.  Every launch also asserts which store path it took.  Same bounds and sentinel
discipline as test_kernel_units.py, whose helpers this file uses."""
import math

import pytest
import torch

pytestmark = pytest.mark.gpu

from gigaam_b200 import synthetic  # noqa: E402
from gigaam_b200.engine import Engine, glu_row_permutation  # noqa: E402
from test_kernel_units import (SENT16, SENT32, _acc_ref, _assert_within, _epilogue_ref, _gemm, _gen, _i32,  # noqa: E402
                               _randn, _same_bits)

SCALE = 0.5
# (name, GemmKind, second A operand)
EPILOGUES = [("f16", 0, False), ("silu", 1, False), ("glu", 2, False), ("res", 3, False), ("res_in_place", 3, False),
             ("f32", 4, False), ("dual_a", 0, True)]


@pytest.fixture(scope="module")
def dev():
    assert torch.cuda.is_available(), "GPU tests need a CUDA device (there is no CPU fallback to test instead)"
    return torch.device("cuda", 0)


@pytest.fixture(scope="module")
def eng(dev):
    ck = synthetic.synthetic_checkpoint("v2_ctc", seed=0, n_layers=1)
    return Engine(ck["cfg"], ck["state_dict"], dev)


@pytest.fixture(scope="module")
def nsm(dev):
    return torch.cuda.get_device_properties(dev).multi_processor_count


class Case:
    """One GEMM of epilogue `name` over M rows (N = 512, so dual-A has one n-block per operand), stored into columns
    [col0, col0 + ncol) of a buffer of ldo columns filled with the sentinel."""

    def __init__(self, dev, name, M, K=128, seed=0):
        self.name, self.kind, self.dual = next((n, k, d) for n, k, d in EPILOGUES if n == name)
        self.dev, self.M, self.N, self.K = dev, M, 512, K
        g = _gen(dev, seed + 1000 * self.kind + M)
        self.A = _randn((M, K), g, dev, 0.5).half()
        self.A2 = _randn((M, K), g, dev, 0.5).half() if self.dual else None
        self.W = _randn((self.N, K), g, dev, 1.0 / math.sqrt(K)).half()
        self.bias = _randn((self.N,), g, dev)
        self.ncol = self.N // 2 if self.kind == 2 else self.N
        self.res = _randn((M, self.ncol), g, dev)
        self.f32 = self.kind >= 3
        self.sent = SENT32 if self.f32 else SENT16

    def run(self, eng, live, reverse=0, col0=0, ldo=None):
        """Returns the whole output buffer; live = None passes no device row count.  Asserts that the launch took the slot
        path exactly when the epilogue has one and the output window is 16-byte aligned."""
        ldo = self.ncol if ldo is None else ldo
        out = torch.full((self.M, ldo), self.sent, dtype=torch.float32 if self.f32 else torch.float16, device=self.dev)
        res = None
        if self.kind == 3:
            if self.name == "res_in_place":
                out[:, col0:col0 + self.ncol] = self.res
                res = out
            else:
                res = torch.full((self.M, ldo), SENT32, dtype=torch.float32, device=self.dev)
                res[:, col0:col0 + self.ncol] = self.res
        W, bias = self.W, self.bias
        if self.kind == 2:
            perm = glu_row_permutation(self.N // 2).to(self.dev)
            W, bias = W[perm].contiguous(), bias[perm].contiguous()
        _gemm(eng, self.kind, self.A, W, bias, out, self.M, self.N, self.K, A2=self.A2, n1=256 if self.dual else 0, res=res,
              ldo=ldo, col0=col0, scale=SCALE, reverse=reverse, m_dev=None if live is None else _i32([live], self.dev))
        esz = 4 if self.f32 else 2
        slots = self.kind != 3 and (col0 * esz) % 16 == 0 and (ldo * esz) % 16 == 0
        assert eng.lib.gam_test_gemm_used_slots(eng.handle) == int(slots), f"{self.name} col0={col0}: wrong store path"
        return out

    def check(self, out, live, col0=0, what=""):
        what = f"{self.name} M={self.M} live={live} col0={col0} {what}"
        if self.dual:
            acc1, d1 = _acc_ref(self.A[:live], self.W[:256], self.K)
            acc2, d2 = _acc_ref(self.A2[:live], self.W[256:], self.K)
            acc, dacc = torch.cat([acc1, acc2], 1), torch.cat([d1, d2], 1)
        else:
            acc, dacc = _acc_ref(self.A[:live], self.W, self.K)
        want, tol = _epilogue_ref(self.kind, acc, dacc, self.bias, self.res[:live], SCALE)
        if live:
            _assert_within(out[:live, col0:col0 + self.ncol], want, tol, what)
        if self.name == "res_in_place":   # rows past the live count keep their residual, the other columns their sentinel
            _same_bits(out[live:, col0:col0 + self.ncol], self.res[live:], f"{what}: rows past the live count")
        else:
            assert bool((out[live:] == self.sent).all()), f"{what}: rows at or past the live count were written"
        assert bool((out[:, :col0] == self.sent).all() and (out[:, col0 + self.ncol:] == self.sent).all()), \
            f"{what}: columns outside the window were written"


NAMES = [e[0] for e in EPILOGUES]


@pytest.mark.parametrize("reverse", [0, 1])
@pytest.mark.parametrize("live", [1, 127, 128, 129, 255, 256, 16064])
@pytest.mark.parametrize("name", NAMES)
def test_live_row_counts(eng, dev, name, live, reverse):
    """Live counts around the first two blocks and the bench's 64 x 251 rows, inside a padded M: full blocks go through the
    slots, the straddling block stores directly, nothing at or past the live count is written."""
    c = Case(dev, name, M=16384 if live > 256 else 640)
    c.check(c.run(eng, live, reverse), live, what=f"reverse={reverse}")


@pytest.mark.parametrize("rounds", [0.5, 1, 3.5])
@pytest.mark.parametrize("name", NAMES)
def test_tile_counts_around_one_round(eng, dev, nsm, name, rounds):
    """Tile counts below, at and above one round of the persistent grid: past one round every CTA reuses its slots for
    tile after tile while earlier bulk stores may still be reading them."""
    tiles = int(rounds * nsm)                 # N = 512: two n-blocks per 128-row block
    M = 128 * max(tiles // 2, 1)
    c = Case(dev, name, M=M, K=64, seed=3)
    c.check(c.run(eng, M, reverse=1), M, what=f"{tiles} tiles")


@pytest.mark.parametrize("name", NAMES)
def test_column_window(eng, dev, name):
    """A 16-byte-aligned window inside a wider buffer (the slot path, columns outside keep the sentinel) and a window
    TMA cannot address (col0 = 2: every tile stores directly)."""
    c = Case(dev, name, M=1000, seed=5)
    for col0 in (64, 2):
        ldo = c.ncol + 128
        c.check(c.run(eng, 777, reverse=col0 == 2, col0=col0, ldo=ldo), 777, col0=col0)


@pytest.mark.parametrize("name", NAMES)
def test_store_paths_give_the_same_bits(eng, dev, name):
    """The same rows once from a full tile (slot path) and once from a straddling tile (direct stores): rows 0..126 with
    live counts 128 and 127, row 128 with live counts 256 and 129."""
    c = Case(dev, name, M=512, seed=7)
    full, part = c.run(eng, 128), c.run(eng, 127)
    _same_bits(full[:127], part[:127], f"{name}: rows 0..126, full vs straddling tile")
    full, part = c.run(eng, 256), c.run(eng, 129)
    _same_bits(full[128:129], part[128:129], f"{name}: row 128, full vs straddling tile")
