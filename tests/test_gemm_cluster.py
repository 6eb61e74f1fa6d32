"""The GEMM's tile-pair scheduler (two-CTA clusters that share the W tile, gemm_sm90.cuh) against float64, at its edges:
block counts odd (the last pair has a phantom half) and even, device row counts whose live rows end in the first or the
second block of a pair, both walk directions, tile counts around twice the co-resident cluster count, and packed conv
batches where one block of a pair is live and its partner is dead or belongs to the next utterance.  Same bounds and
sentinel discipline as test_kernel_units.py, whose helpers this file uses."""
import math

import pytest
import torch
import torch.nn.functional as F

pytestmark = pytest.mark.gpu

from gigaam_b200 import synthetic  # noqa: E402
from gigaam_b200.engine import Engine, pack_conv1d_weight, pack_conv2_weight  # noqa: E402
from oracle import gigaam_oracle as orc  # noqa: E402
from test_kernel_units import (D, SENT16, SENT32, U, _acc_ref, _assert_within, _call, _conv_check, _epilogue_ref,  # noqa: E402
                               _f16_store, _gemm, _gemm_operands, _gen, _i32, _packing, _randn)


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


# live row counts in a buffer of 9 blocks (odd: pairs (0,1) .. (6,7) and (8, phantom)) or 10 blocks (even)
@pytest.mark.parametrize("reverse", [0, 1])
@pytest.mark.parametrize("blocks,live", [(9, 9 * 128), (9, 8 * 128 + 1), (9, 7 * 128 + 5), (9, 6 * 128 + 127),
                                         (10, 10 * 128), (10, 9 * 128 + 64), (10, 1), (10, 0)])
def test_pair_walk_device_row_count(eng, dev, reverse, blocks, live):
    """x += 0.5 (A W^T + b) in place with the row count on the device: the live rows end in the first block of a pair
    (its partner is past the count, or the phantom block of an odd count) or in the second.  Rows past the count keep
    the residual bit for bit."""
    M, N, K = blocks * 128, 768, 192
    A, W, bias, res = _gemm_operands(M, N, K, dev, 31 + blocks + live % 127 + reverse)
    x = res.clone()
    _gemm(eng, 3, A, W, bias, x, M, N, K, res=x, scale=0.5, reverse=reverse, m_dev=_i32([live], dev))
    if live:
        acc, dacc = _acc_ref(A[:live], W, K)
        want, tol = _epilogue_ref(3, acc, dacc, bias, res[:live], 0.5)
        _assert_within(x[:live], want, tol, f"blocks={blocks} live={live} reverse={reverse}")
    assert torch.equal(x[live:], res[live:]), "rows past the live count were written"


@pytest.mark.parametrize("reverse", [0, 1])
@pytest.mark.parametrize("offset", [-3, -2, -1, 0, 1, 2, 3])
def test_pair_walk_tile_counts_around_twice_the_clusters(eng, dev, nsm, reverse, offset):
    """N = 256 (one n-block), so tiles = m-blocks: counts around 2 x nsm / 2 (every SM in a cluster, one round) and
    2 x nsm (two rounds).  A bound on the co-resident cluster count is all the test can know from here: counts around
    both ends of its range leave some CTAs without a pair, walk several pairs per cluster, or a phantom half."""
    for tiles in (nsm + offset, 2 * nsm + offset):
        M, N, K = 128 * tiles - 7, 256, 128
        A, W, bias, _ = _gemm_operands(M, N, K, dev, 71 + tiles + reverse)
        out = torch.full((M + 9, N), SENT16, dtype=torch.float16, device=dev)
        _gemm(eng, 0, A, W, bias, out, M, N, K, reverse=reverse)
        acc, dacc = _acc_ref(A, W, K)
        want, tol = _epilogue_ref(0, acc, dacc, bias)
        _assert_within(out[:M], want, tol, f"tiles={tiles} reverse={reverse}")
        assert bool((out[M:] == SENT16).all())


@pytest.mark.parametrize("plen", [[17, 0, 21, 9, 8], [9, 21, 0, 0, 1], [0, 0, 0, 0, 21], [21, 21, 21, 21, 21]])
def test_pair_walk_packed_conv2d(eng, dev, plen):
    """A_CONV with 3 blocks of 8 frames per utterance (T2 = 21): pairs straddle utterances, the 15 blocks of 5
    utterances leave a phantom half, and the lengths make pairs of a live and a dead block, of two dead blocks (skipped)
    and of blocks from two utterances."""
    B, T1, F1, Cc, N = 5, 41, 32, D, D
    T2 = int(orc.sub_out_len(torch.tensor([T1]), 3, 1)[0])
    assert (T2 + 7) // 8 == 3
    len2 = [min(p, T2 - 2) for p in plen]
    g = _gen(dev, 23 + sum(plen))
    x = torch.rand((B, T1, F1, Cc), generator=g, device=dev).half()
    w2 = _randn((N, Cc, 3, 3), g, dev, 1.0 / math.sqrt(9 * Cc)).half()
    bias = _randn((N,), g, dev, 0.1)
    Wp = pack_conv2_weight(w2.float()).half().contiguous()
    xin = x.double().permute(0, 3, 1, 2)
    acc = F.conv2d(xin, w2.double(), stride=2, padding=1) + bias.double()[None, :, None, None]
    dacc = F.conv2d(xin.abs(), w2.double().abs(), stride=2, padding=1) * (9 * Cc * U) + U * acc.abs()
    live = (torch.arange(T2, device=dev)[None, :] < torch.tensor(len2, device=dev)[:, None])[:, None, :, None]
    want = torch.where(live, acc.clamp_min(0), torch.zeros_like(acc)).permute(0, 2, 3, 1)
    tol = (dacc + _f16_store(acc)).permute(0, 2, 3, 1)
    cu, frames = _packing(plen, 1, 2)
    out = torch.full((frames * 16, N), SENT16, dtype=torch.float16, device=dev)
    _call(eng, "gam_test_gemm_conv", 0, x, Wp, bias, _i32(len2, dev), _i32(cu, dev), _i32(plen, dev), out, frames,
          B, T1, F1, Cc, 9, N, 0)
    _conv_check(out, want, tol, len2, plen, cu, T2, 16, SENT16, f"A_CONV plen={plen}")


@pytest.mark.parametrize("plen", [[130, 0, 300], [300, 1, 0], [0, 0, 257]])
def test_pair_walk_packed_conv1d(eng, dev, plen):
    """A_CONV1D with 3 blocks of 128 frames per utterance (T_out = 300), 9 blocks in all: the same pair cases as the
    conv2d test, fp32 out."""
    B, T_in, taps, c_in, N = 3, 600, 5, D, D
    pad = (taps - 1) // 2
    T_out = int(orc.sub_out_len(torch.tensor([T_in]), taps, 1)[0])
    assert (T_out + 127) // 128 == 3
    lens = [max(p - 3, 0) for p in plen]
    g = _gen(dev, 41 + sum(plen))
    x = _randn((B, T_in, c_in), g, dev).half()
    w = _randn((N, c_in, taps), g, dev, 1.0 / math.sqrt(taps * c_in)).half()
    bias = _randn((N,), g, dev, 0.1)
    Wp = pack_conv1d_weight(w.float()).half().contiguous()
    xin = x.double().transpose(1, 2)
    acc = F.conv1d(xin, w.double(), stride=2, padding=pad) + bias.double()[None, :, None]
    dacc = F.conv1d(xin.abs(), w.double().abs(), stride=2, padding=pad) * (taps * c_in * U) + U * acc.abs()
    live = (torch.arange(T_out, device=dev)[None, :] < torch.tensor(lens, device=dev)[:, None])[:, None, :]
    want = torch.where(live, acc.clamp_min(0), torch.zeros_like(acc)).transpose(1, 2)
    tol = dacc.transpose(1, 2)
    cu, frames = _packing(plen, 2, 5)
    out = torch.full((frames, N), SENT32, dtype=torch.float32, device=dev)
    _call(eng, "gam_test_gemm_conv", 1, x, Wp, bias, _i32(lens, dev), _i32(cu, dev), _i32(plen, dev), out, frames,
          B, T_in, 0, c_in, taps, N, 1)
    _conv_check(out, want, tol, lens, plen, cu, T_out, 1, SENT32, f"A_CONV1D plen={plen}")
