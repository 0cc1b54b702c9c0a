"""CPU-only: the shapes the tensor-core tokeniser accepts (K = 256 m, m = 1..8) and its prepared-state size, through
host-only calls of the C ABI (include/rqb200.h)."""
import pytest

RQB_MAX_LEVELS = 8
TC_HEADER_BYTES = RQB_MAX_LEVELS * 8 * 4 + 4 * RQB_MAX_LEVELS * 4     # TcLevelConst[8] + four scratch words per level


def _round_up(v, a):
    return (v + a - 1) // a * a


def state_bytes(D, K, L):
    """The layout of csrc/tc_common.cuh: header | cc [L][K] | hcc [L][K] | Gram [L(L-1)/2][K][K] | codebook pointers |
    fp32 codebooks [L][K][D] | fp16 blob [L][K/128][D/64][16 KB]."""
    cc = _round_up(TC_HEADER_BYTES, 256)
    hcc = cc + _round_up(L * K * 4, 256)
    gram = hcc + _round_up(L * K * 4, 256)
    cbptr = gram + L * (L - 1) // 2 * K * K * 4
    cbf = _round_up(cbptr + RQB_MAX_LEVELS * 8, 256)
    blob = _round_up(cbf + L * K * D * 4, 1024)
    return blob + L * (K // 128) * (D // 64) * 16384


@pytest.fixture(scope="module")
def lib():
    from rq_vae_recommender_b200 import _lib
    _lib.build()
    return _lib.load()


def test_supported_codebook_sizes(lib):
    for m in range(1, 9):
        for D, L in ((64, 1), (128, 3), (768, 3), (768, 8)):
            assert lib.rqb200_tokenize_tc_supported(D, 256 * m, L) == 1, (D, 256 * m, L)
    for K in (0, 128, 255, 300, 2304, 4096, -256):
        assert lib.rqb200_tokenize_tc_supported(768, K, 3) == 0, K
    assert lib.rqb200_tokenize_tc_supported(832, 1024, 3) == 0
    assert lib.rqb200_tokenize_tc_supported(768, 1024, 9) == 0


@pytest.mark.parametrize("D", [64, 128, 768])
@pytest.mark.parametrize("K", [256, 512, 1024, 1792, 2048])
@pytest.mark.parametrize("L", [1, 3, 8])
def test_state_bytes_follow_the_layout(lib, D, K, L):
    assert lib.rqb200_tokenize_tc_state_bytes(D, K, L) == state_bytes(D, K, L)


def test_state_bytes_of_unsupported_shapes_is_zero(lib):
    assert lib.rqb200_tokenize_tc_state_bytes(768, 2304, 3) == 0
    assert lib.rqb200_tokenize_tc_state_bytes(768, 384, 3) == 0


def test_documented_state_sizes(lib):
    """The sizes INTEGRATION.md / README state: ~80 MB at K = 2048, L = 3, D = 768 and ~0.55 GB at L = 8."""
    assert 75e6 < lib.rqb200_tokenize_tc_state_bytes(768, 2048, 3) < 85e6
    assert 0.53e9 < lib.rqb200_tokenize_tc_state_bytes(768, 2048, 8) < 0.57e9
