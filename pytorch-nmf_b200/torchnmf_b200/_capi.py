"""ctypes binding of libnmf_b200.so (include/nmf_b200.h).

This is the stub a torchnmf maintainer would add next to torchnmf/nmf.py (see INTEGRATION.md): it
exposes the C ABI with plain pointers and sizes, taking device pointers from ``Tensor.data_ptr()``.
There is NO fallback: if the library is missing or fails to load, every product entry point raises.
"""
import ctypes
import os

import torch

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.environ.get("NMFB200_LIB") or os.path.join(os.path.dirname(_HERE), "lib", "libnmf_b200.so")   # override: tuning builds

PREC_AUTO, PREC_F32, PREC_F16, PREC_F16_SPLIT = -1, 0, 1, 2
PRECISIONS = {"auto": PREC_AUTO, "f32": PREC_F32, "f16": PREC_F16, "f16_split": PREC_F16_SPLIT}
PRECISION_NAMES = {v: k for k, v in PRECISIONS.items()}

# element types a dense target may have (NMFB200_DTYPE_*); the factors are always fp32
DTYPE_F32, DTYPE_F16, DTYPE_BF16 = 0, 1, 2
DTYPES = {torch.float32: DTYPE_F32, torch.float16: DTYPE_F16, torch.bfloat16: DTYPE_BF16}

_c = ctypes
_vp, _i64, _dbl, _int = _c.c_void_p, _c.c_int64, _c.c_double, _c.c_int

# symbol -> (restype, argtypes); must list every function include/nmf_b200.h declares
SIGNATURES = {
    "nmfb200_abi_version": (_int, []),
    "nmfb200_last_error": (_c.c_char_p, []),
    "nmfb200_build_info": (_c.c_char_p, []),
    "nmfb200_launch_count": (_i64, []),
    "nmfb200_ctx_check_health": (_int, [_vp, _vp]),
    "nmfb200_nmf_create": (_int, [_c.POINTER(_vp), _int, _i64, _i64, _i64, _int]),
    "nmfb200_destroy": (None, [_vp]),
    "nmfb200_precision": (_int, [_vp]),
    "nmfb200_precision_for_beta": (_int, [_vp, _dbl]),
    "nmfb200_nmf_set_target": (_int, [_vp, _vp, _i64, _int, _vp]),
    "nmfb200_target_minmax": (_int, [_vp, _c.POINTER(_c.c_float), _c.POINTER(_c.c_float), _vp]),
    "nmfb200_nmf_iterate": (_int, [_vp, _vp, _vp, _dbl, _dbl, _dbl, _dbl, _int, _vp]),
    "nmfb200_nmf_loss_prefetch_w": (_int, [_vp, _vp, _vp, _dbl, _vp, _vp]),
    "nmfb200_nmf_contract_only": (_int, [_vp, _vp, _vp, _int, _dbl, _vp]),
    "nmfb200_nmf_cd_update": (_int, [_vp, _vp, _vp, _int, _dbl, _dbl, _vp]),
    "nmfb200_nmf_cd_iterate": (_int, [_vp, _vp, _vp, _dbl, _dbl, _int, _vp]),
    "nmfb200_nmf_batched_create": (_int, [_c.POINTER(_vp), _int, _i64, _i64, _i64, _i64]),
    "nmfb200_nmf_batched_create_ragged": (_int, [_c.POINTER(_vp), _int, _i64, _i64, _i64, _i64, _c.POINTER(_i64)]),
    "nmfb200_nmf_batched_set_target": (_int, [_vp, _vp, _i64, _i64, _int, _vp]),
    "nmfb200_nmf_batched_set_active": (_int, [_vp, _vp, _vp]),
    "nmfb200_nmf_batched_cd_update": (_int, [_vp, _vp, _vp, _int, _dbl, _dbl, _vp]),
    "nmfb200_nmf_batched_cd_iterate": (_int, [_vp, _vp, _vp, _dbl, _dbl, _int, _vp]),
    "nmfb200_nmf_observed_cd_update": (_int, [_vp, _vp, _vp, _int, _dbl, _dbl, _vp]),
    "nmfb200_nmf_observed_cd_iterate": (_int, [_vp, _vp, _vp, _dbl, _dbl, _int, _vp]),
    "nmfb200_nmf_set_target_sparse": (_int, [_vp, _i64, _vp, _vp, _vp, _vp, _vp, _vp, _dbl, _dbl, _vp]),
    "nmfb200_nmf_set_target_sparse_any_beta": (_int, [_vp, _i64, _vp, _vp, _vp, _vp, _vp, _vp, _dbl, _dbl, _vp]),
    "nmfb200_nmf_set_target_observed": (_int, [_vp, _i64, _vp, _vp, _vp, _vp, _vp, _vp, _vp]),
    "nmfb200_nmf_set_target_observed_weighted": (_int, [_vp, _i64, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _vp]),
    "nmfb200_nmf_peer_supported": (_int, [_vp, _dbl]),
    "nmfb200_nmf_peer_alloc": (_int, [_vp, _vp]),
    "nmfb200_nmf_peer_connect": (_int, [_vp, _int, _int, _vp]),
    "nmfb200_nmf_peer_world": (_int, [_vp]),
    "nmfb200_nmf_peer_release": (_int, [_vp]),
    "nmfb200_nmf_update_w_peer": (_int, [_vp, _vp, _vp, _dbl, _dbl, _dbl, _dbl, _vp]),
    "nmfb200_nmfnd_create": (_int, [_c.POINTER(_vp), _int, _i64, _i64, _int, _c.POINTER(_i64), _i64, _c.POINTER(_i64), _int]),
    "nmfb200_nmfd_set_target": (_int, [_vp, _vp, _int, _vp]),
    "nmfb200_nmfnd_batched_create": (_int, [_c.POINTER(_vp), _int, _i64, _i64, _i64, _int, _c.POINTER(_i64), _i64,
                                            _c.POINTER(_i64)]),
    "nmfb200_nmfnd_batched_create_ragged": (_int, [_c.POINTER(_vp), _int, _i64, _i64, _i64, _int, _c.POINTER(_i64), _i64,
                                                   _c.POINTER(_i64), _c.POINTER(_i64)]),
    "nmfb200_nmfd_batched_set_target": (_int, [_vp, _vp, _i64, _int, _vp]),
    "nmfb200_nmfd_batched_set_active": (_int, [_vp, _vp, _vp]),
    "nmfb200_plca_work_numel": (_i64, [_vp]),
    "nmfb200_plca_iterate": (_int, [_vp, _vp, _vp, _vp, _vp, _vp, _int, _vp, _vp, _vp, _int, _vp]),
    "nmfb200_plca_loss": (_int, [_vp, _vp, _vp, _vp, _vp, _vp]),
    "nmfb200_plca_masked_terms": (_int, [_vp, _vp, _vp, _int, _vp, _vp, _vp]),
    "nmfb200_plca_sparse_create": (_int, [_c.POINTER(_vp), _int, _i64, _i64, _i64, _i64]),
    "nmfb200_plca_sparse_set_target": (_int, [_vp, _vp, _vp, _vp, _vp, _vp, _vp, _vp]),
    "nmfb200_plca_sparse_terms": (_int, [_vp, _vp, _vp, _vp, _c.c_float, _vp, _vp]),
    "nmfb200_plca_sparse_device_bytes": (_i64, [_vp]),
    "nmfb200_sync_factors": (_int, [_vp]),
    "nmfb200_update_w": (_int, [_vp, _vp, _vp, _dbl, _dbl, _dbl, _dbl, _vp]),
    "nmfb200_update_h": (_int, [_vp, _vp, _vp, _dbl, _dbl, _dbl, _dbl, _vp]),
    "nmfb200_loss": (_int, [_vp, _vp, _vp, _dbl, _vp, _vp]),
    "nmfb200_raw_terms_numel": (_i64, [_vp, _int, _dbl]),
    "nmfb200_raw_terms": (_int, [_vp, _vp, _vp, _int, _dbl, _vp, _vp]),
    "nmfb200_w_apply": (_int, [_vp, _vp, _vp, _dbl, _dbl, _dbl, _dbl, _vp]),
    "nmfb200_set_mask": (_int, [_vp, _vp, _vp]),
    "nmfb200_set_weight": (_int, [_vp, _vp, _vp]),
    "nmfb200_set_fixed_w": (_int, [_vp, _vp, _vp]),
    "nmfb200_set_ard": (_int, [_vp, _vp, _vp, _dbl, _dbl, _dbl, _vp]),
    "nmfb200_ard_update": (_int, [_vp, _vp, _vp, _vp]),
    "nmfb200_ard_read": (_int, [_vp, _vp, _vp, _vp, _vp]),
    "nmfb200_hoyer_project": (_int, [_int, _vp, _i64, _i64, _i64, _vp, _vp, _vp, _vp]),
    "nmfb200_nmf_plan": (_int, [_i64, _i64, _i64, _c.POINTER(_i64), _int]),
    "nmfb200_nmfd_plan": (_int, [_i64, _i64, _int, _c.POINTER(_i64), _i64, _c.POINTER(_i64), _c.POINTER(_i64), _int]),
    "nmfb200_nmf_sparse_plan": (_int, [_i64, _i64, _i64, _c.POINTER(_i64), _int]),
    "nmfb200_nmfnd_tc_plan": (_int, [_i64, _i64, _int, _c.POINTER(_i64), _i64, _c.POINTER(_i64), _c.POINTER(_i64), _int]),
    "nmfb200_nmf_tc_plan": (_int, [_i64, _i64, _i64, _int, _int, _c.POINTER(_i64), _int]),
}
NMF_PLAN_LEN, NMFD_PLAN_LEN, SPARSE_PLAN_LEN, NMFND_TC_PLAN_LEN = 9, 19, 8, 31         # include/nmf_b200.h
NMF_TC_PLAN_LEN = 15                                                                    # include/nmf_b200.h
PLCA_TRAIN_W, PLCA_TRAIN_H, PLCA_TRAIN_Z = 1, 2, 4                                       # include/nmf_b200.h

_lib = None


class NmfB200Error(RuntimeError):
    pass


def load():
    """Load the shared library once; raise loudly if it is absent (no CPU fallback exists)."""
    global _lib
    if _lib is not None:
        return _lib
    if not os.path.exists(LIB_PATH):
        raise NmfB200Error(
            f"{LIB_PATH} not found: build it with `python -c 'import __graft_entry__ as g; g.build()'` "
            "(needs nvcc). torchnmf_b200 has no CPU fallback.")
    lib = ctypes.CDLL(LIB_PATH)
    for name, (res, args) in SIGNATURES.items():
        fn = getattr(lib, name)          # AttributeError here == ABI mismatch
        fn.restype = res
        fn.argtypes = args
    if lib.nmfb200_abi_version() != 2:
        raise NmfB200Error("libnmf_b200.so ABI version mismatch")
    _lib = lib
    return lib


def check(rc):
    if rc != 0:
        msg = load().nmfb200_last_error()
        raise NmfB200Error(f"libnmf_b200 error {rc}: {msg.decode() if msg else '?'}")


def build_info():
    """The library's build stamp: source hash, nvcc version, target architecture, build time."""
    return load().nmfb200_build_info().decode()


def launch_count():
    return int(load().nmfb200_launch_count())


def nmf_plan(N, C, R):
    """The fp32 kernels' tile plan of an (N, C) rank-R NMF context (nmfb200_nmf_plan), as a dict; no device needed."""
    out = (_i64 * NMF_PLAN_LEN)()
    check(load().nmfb200_nmf_plan(N, C, R, out, NMF_PLAN_LEN))
    keys = ("nch_w", "nch_h", "tpc_w", "tpc_h", "rb", "loss_chunks", "loss_tpc", "colsum_blocks_n", "colsum_blocks_c")
    return dict(zip(keys, out))


def sparse_plan(N, C, R):
    """The sparse-target kernels' launch plan of an (N, C) rank-R context (nmfb200_nmf_sparse_plan), as a dict; no device
    needed.  Gram plans: `rpb_n` / `nb_n` over the N rows of H, `rpb_c` / `nb_c` over the C rows of W."""
    out = (_i64 * SPARSE_PLAN_LEN)()
    check(load().nmfb200_nmf_sparse_plan(N, C, R, out, SPARSE_PLAN_LEN))
    keys = ("rpl", "gram_passes", "rpb_n", "nb_n", "rpb_c", "nb_c", "gather_blocks_n", "gather_blocks_c")
    return dict(zip(keys, out))


def nmfd_plan(B, C, vdims, R, kdims):
    """The fp32 kernels' tile plan of an NMFD / NMF2D / NMF3D context (nmfb200_nmfd_plan), as a dict; no device needed."""
    nd = len(vdims)
    out = (_i64 * NMFD_PLAN_LEN)()
    check(load().nmfb200_nmfd_plan(B, C, nd, (_i64 * nd)(*vdims), R, (_i64 * nd)(*kdims), out, NMFD_PLAN_LEN))
    v = list(out)
    return {"recon_mt": v[0], "recon_grid": tuple(v[1:4]), "dgrad_mt": v[4], "dgrad_nsplit": v[5],
            "dgrad_grid": tuple(v[6:9]), "wgrad": dict(zip(("mt", "tp", "nr", "no", "ntt", "nrg", "nog"), v[9:16])),
            "wgrad_nsplit": v[16], "vec4_w": bool(v[17]), "vec4_h": bool(v[18])}


def nmfnd_tc_plan(B, C, vdims, R, kdims):
    """The tensor-core kernels' launch plan of an NMFD / NMF2D / NMF3D context (nmfb200_nmfnd_tc_plan), as a dict; no
    device needed.  `bslice` / `slices` count target lines (b, x1, x2) per recon launch, `hslice` / `hslices` activation
    lines (b, j1, j2) per dgrad launch.  Raises NmfB200Error naming the limit for a shape the f16 path does not take."""
    nd = len(vdims)
    out = (_i64 * NMFND_TC_PLAN_LEN)()
    check(load().nmfb200_nmfnd_tc_plan(B, C, nd, (_i64 * nd)(*vdims), R, (_i64 * nd)(*kdims), out, NMFND_TC_PLAN_LEN))
    v = list(out)
    return {"prep_w": tuple(v[0:3]), "prep_h": tuple(v[3:6]), "recon": tuple(v[6:9]), "wgrad": tuple(v[9:12]),
            "dgrad": tuple(v[12:15]), "bslice": v[15], "slices": v[16], "dgrad_rblocks": v[17], "loss_blocks": v[18],
            "ws_w": v[19], "kbs_w": v[20], "ws_h": v[21], "kbs_h": v[22], "hslice": v[23], "hslices": v[24],
            "Tp": v[25], "padl": v[26], "Lp": v[27], "Lq": v[28], "Cpad": v[29], "nch": v[30]}


def nmf_tc_plan(N, C, R, precision, num_sms):
    """The tensor-core contraction's layout and launch plan of an (N, C) rank-R NMF context on a device with `num_sms` SMs
    (nmfb200_nmf_tc_plan), as a dict; no device needed.  `tn`, `ns`, `nf`: tile width, ring stages, F slots; then per
    orientation (`_w`: rows C over N, `_h`: rows N over C) `row_blocks`, `tiles`, `nchunks`, `tpc`, `items`, `grid`.
    `precision` is a name of PRECISIONS or its value; raises NmfB200Error for f32 and for shapes the f16 path refuses."""
    prec = PRECISIONS[precision] if isinstance(precision, str) else int(precision)
    out = (_i64 * NMF_TC_PLAN_LEN)()
    check(load().nmfb200_nmf_tc_plan(N, C, R, prec, num_sms, out, NMF_TC_PLAN_LEN))
    v = list(out)
    keys = ("row_blocks", "tiles", "nchunks", "tpc", "items", "grid")
    plan = {"tn": v[0], "ns": v[1], "nf": v[2]}
    plan.update({f"{k}_w": x for k, x in zip(keys, v[3:9])})
    plan.update({f"{k}_h": x for k, x in zip(keys, v[9:15])})
    return plan
