"""Every context create of the C ABI refuses bad arguments before it selects a device: the same code and message for each
input, and `*out` left null.  CPU-only: the shapes are refused by arithmetic alone, so nothing is allocated, and the device
argument names no device, which a create that got as far as selecting it would report instead."""
import ctypes

import pytest

from torchnmf_b200 import _capi

ERR_INVALID = 1
NO_DEVICE = -1
SENTINEL = 0x5EED
MAX_RANK_MSG = "rank must be at most 65535 x 256 = 16776960"
I32 = 2**31 - 1

_i64 = ctypes.c_int64


def _arr(vals):
    return None if vals is None else (_i64 * len(vals))(*vals)


def _nmf(N, C, R, precision=_capi.PREC_F32):
    return "nmfb200_nmf_create", (NO_DEVICE, N, C, R, precision)


def _nmf_batched(B, N, C, R):
    return "nmfb200_nmf_batched_create", (NO_DEVICE, B, N, C, R)


def _nmf_ragged(B, N, C, R, lengths):
    return "nmfb200_nmf_batched_create_ragged", (NO_DEVICE, B, N, C, R, _arr(lengths))


def _nmfnd(B, C, vdims, R, kdims, precision=_capi.PREC_F32, ndim=None):
    nd = len(vdims) if ndim is None else ndim
    return "nmfb200_nmfnd_create", (NO_DEVICE, B, C, nd, _arr(vdims), R, _arr(kdims), precision)


def _nmfnd_batched(P, B, C, vdims, R, kdims, ndim=None):
    nd = len(vdims) if ndim is None else ndim
    return "nmfb200_nmfnd_batched_create", (NO_DEVICE, P, B, C, nd, _arr(vdims), R, _arr(kdims))


def _nmfnd_ragged(P, B, C, vdims, R, kdims, lengths, ndim=None):
    nd = len(vdims) if ndim is None else ndim
    return "nmfb200_nmfnd_batched_create_ragged", (NO_DEVICE, P, B, C, nd, _arr(vdims), R, _arr(kdims), _arr(lengths))


def _plca_sparse(N, C, R, nnz):
    return "nmfb200_plca_sparse_create", (NO_DEVICE, N, C, R, nnz)


BAD_NMFD = "bad NMFD sizes"
NMFD_AXES = "1 to 3 convolved axes are supported"
P_LOSS = "batched NMFD: P x loss partials per problem must be below 2^31"

# (id, (symbol, arguments after `out`), message)
CASES = [
    # nmfb200_nmf_create
    ("nmf-n0", _nmf(0, 8, 2), "N, C, R must be positive"),
    ("nmf-c0", _nmf(8, 0, 2), "N, C, R must be positive"),
    ("nmf-r0", _nmf(8, 8, 0), "N, C, R must be positive"),
    ("nmf-rank", _nmf(8, 8, 65535 * 256 + 1), MAX_RANK_MSG),
    ("nmf-prec-low", _nmf(8, 8, 2, _capi.PREC_AUTO - 1), "unknown precision mode"),
    ("nmf-prec-high", _nmf(8, 8, 2, _capi.PREC_F16_SPLIT + 1), "unknown precision mode"),
    # nmfb200_nmf_batched_create
    ("batched-b0", _nmf_batched(0, 8, 8, 2), "B, N, C, R must be positive"),
    ("batched-n0", _nmf_batched(2, 0, 8, 2), "B, N, C, R must be positive"),
    ("batched-rank", _nmf_batched(2, 8, 8, 257), "batched fits support rank <= 256"),
    ("batched-grid-rows", _nmf_batched(2**30, 256, 256, 1), "batch too large for the launch grids"),
    ("batched-grid-rank", _nmf_batched(2**30, 8, 8, 256), "batch too large for the launch grids"),
    # nmfb200_nmf_batched_create_ragged
    ("ragged-b0", _nmf_ragged(0, 8, 8, 2, [1]), "B, N, C, R must be positive"),
    ("ragged-r0", _nmf_ragged(1, 8, 8, 0, [1]), "B, N, C, R must be positive"),
    ("ragged-rank", _nmf_ragged(1, 8, 8, 257, [1]), "batched fits support rank <= 256"),
    ("ragged-lengths-null", _nmf_ragged(2, 8, 8, 2, None), "lengths is null"),
    ("ragged-b-grid", _nmf_ragged(2**31, 8, 8, 2, [1]),
     "ragged batch: B must be below 2^31 (one block per problem and launch)"),
    ("ragged-length-0", _nmf_ragged(3, 8, 8, 2, [8, 0, 1]), "lengths[1] = 0 is outside [1, N]"),
    ("ragged-length-above-n", _nmf_ragged(3, 8, 8, 2, [8, 1, 9]), "lengths[2] = 9 is outside [1, N]"),
    ("ragged-grid-x", _nmf_ragged(1, 4, 2**40, 1, [4]),
     "ragged batch: the problems' blocks of one launch pass grid x (2^31 - 1)"),
    ("ragged-shared-grids", _nmf_ragged(128, 2**33, 1, 1, [1] * 128), "batch too large for the launch grids"),
    # nmfb200_nmfnd_create
    ("nmfd-ndim0", _nmfnd(1, 4, [10], 2, [3], ndim=0), NMFD_AXES),
    ("nmfd-ndim4", _nmfnd(1, 4, [10, 10, 10, 10], 2, [3, 3, 3, 3]), NMFD_AXES),
    ("nmfd-vdims-null", ("nmfb200_nmfnd_create", (NO_DEVICE, 1, 4, 1, None, 2, _arr([3]), _capi.PREC_F32)), NMFD_AXES),
    ("nmfd-b0", _nmfnd(0, 4, [10], 2, [3]), BAD_NMFD),
    ("nmfd-r0", _nmfnd(1, 4, [10], 0, [3]), BAD_NMFD),
    ("nmfd-kernel-above-target", _nmfnd(1, 4, [10], 2, [11]), BAD_NMFD),
    ("nmfd2d-kernel-above-target", _nmfnd(1, 4, [3, 10], 2, [4, 3]), BAD_NMFD),
    ("nmfd-kernel-0", _nmfnd(1, 4, [10], 2, [0]), BAD_NMFD),
    ("nmfd-rank", _nmfnd(1, 4, [10], 257, [3]), "rank > 256 is not supported"),
    ("nmfd-target-size", _nmfnd(2**21, 2**20, [1], 1, [1]), "NMFD target too large"),
    ("nmfd-channels", _nmfnd(1, 65535 * 64 + 1, [1], 1, [1]),
     "NMFD supports at most 65535 x 64 = 4194240 channels (grid.y of the reconstruction)"),
    ("nmfd-line-index", _nmfnd(2**31, 1, [1], 1, [1]),
     "NMFD batch x outer activation lines must be below 2^31 (the W gradient's line index)"),
    ("nmfd-contraction-index", _nmfnd(1, 2**21, [32, 64, 1], 1, [32, 64, 1]),
     "NMFD channels (or rank) x outer kernel offsets must be below 2^31 (the contraction index)"),
    ("nmfd-f16-split", _nmfnd(1, 4, [10], 2, [3], _capi.PREC_F16_SPLIT), "NMFD precision must be auto, f32 or f16"),
    # nmfb200_nmfnd_batched_create
    ("nmfd-batched-p0", _nmfnd_batched(0, 1, 4, [10], 2, [3]), "P must be positive"),
    ("nmfd-batched-ndim0", _nmfnd_batched(2, 1, 4, [10], 2, [3], ndim=0), NMFD_AXES),
    ("nmfd-batched-kernel", _nmfnd_batched(2, 1, 4, [10], 2, [11]), BAD_NMFD),
    ("nmfd-batched-rank", _nmfnd_batched(2, 1, 4, [10], 257, [3]), "rank > 256 is not supported"),
    ("nmfd-batched-lines", _nmfnd_batched(2**30, 4, 1, [4], 1, [1]),
     "batched NMFD: P x B must be below 2^31 (the line index of the fp32 kernels)"),
    ("nmfd-batched-loss", _nmfnd_batched(I32, 1, 1024, [1024], 1, [1]), P_LOSS),
    ("nmfd-batched-colsum", _nmfnd_batched(2**30 + 1, 1, 1, [1], 128, [1]),
     "batched NMFD: P x column-sum blocks must be below 2^31 (grid x of the column sums)"),
    # nmfb200_nmfnd_batched_create_ragged
    ("nmfd-ragged-p0", _nmfnd_ragged(0, 1, 4, [10], 2, [3], [10]), "P must be positive"),
    ("nmfd-ragged-ndim4", _nmfnd_ragged(1, 1, 4, [10] * 4, 2, [3] * 4, [10]), NMFD_AXES),
    ("nmfd-ragged-rank", _nmfnd_ragged(1, 1, 4, [10], 257, [3], [10]), "rank > 256 is not supported"),
    ("nmfd-ragged-loss", _nmfnd_ragged(I32, 1, 1024, [1024], 1, [1], [1024]), P_LOSS),
    ("nmfd-ragged-lengths-null", _nmfnd_ragged(2, 1, 4, [10], 2, [3], None), "lengths is null"),
    ("nmfd-ragged-colsum-grid", _nmfnd_ragged(2**16, 2**8, 1, [1], 2**8, [1], [1]),
     "ragged NMFD batch: P x B x R must be below 2^31 (grid x of the column sums of H)"),
    ("nmfd-ragged-length-below-kernel", _nmfnd_ragged(3, 1, 4, [10], 2, [3], [10, 2, 5]),
     "lengths[1] = 2 is outside [3, 10] (the last kernel and target sizes)"),
    ("nmfd-ragged-length-above-target", _nmfnd_ragged(3, 1, 4, [10], 2, [3], [10, 3, 11]),
     "lengths[2] = 11 is outside [3, 10] (the last kernel and target sizes)"),
    ("nmfd2d-ragged-length", _nmfnd_ragged(2, 1, 4, [5, 10], 2, [2, 4], [3, 10]),
     "lengths[0] = 3 is outside [4, 10] (the last kernel and target sizes)"),
    # nmfb200_plca_sparse_create
    ("plca-sparse-n0", _plca_sparse(0, 8, 2, 4), "N, C, R must be positive and nnz >= 0"),
    ("plca-sparse-r0", _plca_sparse(8, 8, 0, 4), "N, C, R must be positive and nnz >= 0"),
    ("plca-sparse-nnz", _plca_sparse(8, 8, 2, -1), "N, C, R must be positive and nnz >= 0"),
    ("plca-sparse-rank", _plca_sparse(8, 8, 65535 * 256 + 1, 4), MAX_RANK_MSG),
    ("plca-sparse-gather", _plca_sparse(8 * 2**31, 8, 2, 4),
     "sparse PLCA: ceil(max(N, C) / 8) gather blocks pass grid x (2^31 - 1)"),
    ("plca-sparse-gather-c", _plca_sparse(8, 8 * 2**31, 2, 4),
     "sparse PLCA: ceil(max(N, C) / 8) gather blocks pass grid x (2^31 - 1)"),
]

CREATES = {
    "nmfb200_nmf_create": _nmf(8, 8, 2),
    "nmfb200_nmf_batched_create": _nmf_batched(2, 8, 8, 2),
    "nmfb200_nmf_batched_create_ragged": _nmf_ragged(2, 8, 8, 2, [8, 3]),
    "nmfb200_nmfnd_create": _nmfnd(1, 4, [10], 2, [3]),
    "nmfb200_nmfnd_batched_create": _nmfnd_batched(2, 1, 4, [10], 2, [3]),
    "nmfb200_nmfnd_batched_create_ragged": _nmfnd_ragged(2, 1, 4, [10], 2, [3], [10, 3]),
    "nmfb200_plca_sparse_create": _plca_sparse(8, 8, 2, 4),
}


@pytest.fixture(scope="module")
def lib():
    return _capi.load()


def _refused(lib, call, message):
    symbol, args = call
    out = ctypes.c_void_p(SENTINEL)
    rc = getattr(lib, symbol)(ctypes.byref(out), *args)
    assert rc == ERR_INVALID, (symbol, rc, lib.nmfb200_last_error())
    assert lib.nmfb200_last_error().decode() == message
    assert out.value is None


@pytest.mark.parametrize("name,call,message", CASES, ids=[c[0] for c in CASES])
def test_create_refuses_before_device_selection(lib, name, call, message):
    _refused(lib, call, message)


@pytest.mark.parametrize("symbol", sorted(CREATES))
def test_create_refuses_a_null_out(lib, symbol):
    sym, args = CREATES[symbol]
    assert getattr(lib, sym)(None, *args) == ERR_INVALID
    assert lib.nmfb200_last_error().decode() == "out is null"


def test_every_create_is_covered():
    covered = {call[0] for _, call, _ in CASES}
    assert covered == set(CREATES)
    assert {s for s in _capi.SIGNATURES if s.endswith("_create") or s.endswith("_create_ragged")} == set(CREATES)
