"""How the learner's GEMMs are put on the machine, checked without a GPU: the split-K rule (sized to the device's SMs:
with fewer output tiles than SMs, the most slices that still run in one wave) and the work items of the persistent wgmma
kernel (CTA b of a grid of g runs items b, b + g, ...: every (tile, slice) exactly once, the slices covering k)."""
import pytest

from sample_factory_b200 import ops

# (M rows reduced over, N, K) of sfb200_linear_backward -- dW is [N, K] -- and the SMs of the device
CASES = [(32768, 512, 512, 132), (32768, 512, 64, 132), (32768, 512, 512, 148), (32768, 512, 64, 148), (1000, 72, 200, 132),
         (100, 128, 64, 132), (17000, 512, 128, 132), (65536, 1024, 2048, 132), (32768, 1536, 1408, 132),
         (4096, 2048, 512, 114), (300000, 32, 288, 132), (64, 512, 512, 132)]


def ceil_div(a, b):
    return (a + b - 1) // b


@pytest.mark.parametrize("M,N,K,sms", CASES)
def test_split_k_fills_one_wave(M, N, K, sms):
    tiles = ceil_div(N, 128) * ceil_div(K, 128)
    s = ops.linear_backward_splits(M, N, K, sms)
    assert 1 <= s <= 64
    if tiles >= sms:
        assert s == 1
    else:
        assert tiles * s <= sms
        # no larger count would do: the next one overflows the wave, the k cap (128 k per slice) or the 64 cap
        assert tiles * (s + 1) > sms or s == 64 or s + 1 > max(M // 128, 1)


def test_split_k_at_the_headline_shapes():
    assert ops.linear_backward_splits(32768, 512, 512, 132) == 8     # dW2: 16 tiles -> 128 CTAs
    assert ops.linear_backward_splits(32768, 512, 64, 132) == 33     # dW1: 4 tiles -> at most 132 CTAs


@pytest.mark.parametrize("M,N,K,sms", CASES)
def test_workspace_covers_the_slices(M, N, K, sms):
    # (the current device's rule, or the 132-SM one when there is no device)
    s = ops.linear_backward_splits(M, N, K)
    assert ops.linear_backward_workspace_bytes(M, N, K) >= s * N * K * 4


@pytest.mark.parametrize("M,N,K,sms", CASES)
def test_every_work_item_once(M, N, K, sms):
    """the dW GEMM: output [N, K] reduced over M in the slices the rule gives"""
    splits = ops.linear_backward_splits(M, N, K, sms)
    rows, cols, red = N, K, M
    items = ops.gemm_work_item(0, rows, cols, red, splits)[5]
    assert items % (ceil_div(rows, 128) * ceil_div(cols, 128)) == 0
    assert items // (ceil_div(rows, 128) * ceil_div(cols, 128)) <= splits
    grid = min(items, sms)
    seen = {}
    for b in range(grid):
        for item in range(b, items, grid):
            m0, n0, k0, k_len, z, n_items = ops.gemm_work_item(item, rows, cols, red, splits)
            assert n_items == items and m0 % 128 == 0 and n0 % 128 == 0 and m0 < rows and n0 < cols and k_len > 0
            assert (m0, n0, z) not in seen
            seen[(m0, n0, z)] = (k0, k_len)
    assert len(seen) == items
    # consecutive items walk n first: the CTAs running together share their A rows
    if cols > 128:
        assert ops.gemm_work_item(1, rows, cols, red, splits)[1] == 128
    # the slices of one tile tile k: contiguous, whole 32-k stages, the last one reaching the end
    for m0 in range(0, rows, 128):
        for n0 in range(0, cols, 128):
            ks = sorted(v for (m, n, _), v in seen.items() if (m, n) == (m0, n0))
            assert ks[0][0] == 0
            for (a0, al), (b0, _) in zip(ks, ks[1:]):
                assert a0 + al == b0 and al % 32 == 0
            assert ks[-1][0] < red <= ks[-1][0] + ks[-1][1] < red + 32
