"""ctypes binding of libsnarkb200.so (include/snarkb200.h).  The library is CUDA-only: if it is missing or no
device is present every entry point raises — there is no CPU fallback on the product path."""
from __future__ import annotations

import ctypes
import os
import subprocess

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_HERE, "libsnarkb200.so")
_lib = None

SB_BN254, SB_BLS12_381 = 0, 1
SB_G1, SB_G2 = 1, 2

u8p = ctypes.c_char_p
u64 = ctypes.c_uint64
u32 = ctypes.c_uint32
vp = ctypes.c_void_p

_SIGNATURES = {
    # name: (restype, [argtypes])
    "sb_create": (ctypes.c_int, [ctypes.c_int, ctypes.c_int, ctypes.POINTER(vp)]),
    "sb_destroy": (None, [vp]),
    "sb_last_error": (ctypes.c_char_p, [vp]),
    "sb_version": (ctypes.c_char_p, []),
    "sb_launch_count": (u64, [vp]),
    "sb_msm_g1_affine": (ctypes.c_int, [vp, vp, vp, u32, u64, vp]),
    "sb_msm_g2_affine": (ctypes.c_int, [vp, vp, vp, u32, u64, vp]),
    "sb_bases_register": (ctypes.c_int, [vp, ctypes.c_int, vp, u64, ctypes.POINTER(u64)]),
    "sb_bases_release": (ctypes.c_int, [vp, u64]),
    "sb_msm_registered": (ctypes.c_int, [vp, u64, u64, vp, u32, u64, vp]),
    "sb_msm_registered_partial": (ctypes.c_int, [vp, u64, u64, vp, u32, u64, vp]),
    "sb_msm_registered_batch": (ctypes.c_int, [vp, u64, u64, vp, u32, u64, u32, vp]),
    "sb_msm_sum_partials": (ctypes.c_int, [vp, ctypes.c_int, vp, ctypes.c_int, vp]),
    "sb_msm_partial_bytes": (u32, [vp, ctypes.c_int]),
    "sb_ntt_fr": (ctypes.c_int, [vp, vp, u64, ctypes.c_int, vp]),
    "sb_fr_batch_apply_key": (ctypes.c_int, [vp, vp, u64, vp, vp, vp]),
    "sb_fr_batch_to_montgomery": (ctypes.c_int, [vp, vp, u64, vp]),
    "sb_fr_batch_from_montgomery": (ctypes.c_int, [vp, vp, u64, vp]),
    "sb_qap_join_abc": (ctypes.c_int, [vp, vp, vp, vp, u64, vp]),
    "sb_fr_root": (ctypes.c_int, [vp, ctypes.c_int, vp]),
    "sb_group_fft": (ctypes.c_int, [vp, ctypes.c_int, vp, ctypes.c_int, u64, ctypes.c_int, ctypes.c_int, vp]),
    "sb_group_batch_apply_key": (ctypes.c_int, [vp, ctypes.c_int, vp, ctypes.c_int, u64, vp, vp, ctypes.c_int, vp]),
    "sb_groth16_load": (ctypes.c_int, [vp, vp, u64, ctypes.POINTER(u64)]),
    "sb_groth16_load_sharded": (ctypes.c_int, [vp, vp, u64, ctypes.c_int, ctypes.c_int, ctypes.POINTER(u64)]),
    "sb_groth16_load_file": (ctypes.c_int, [vp, ctypes.c_char_p, ctypes.POINTER(u64)]),
    "sb_groth16_info": (ctypes.c_int, [vp, u64, ctypes.POINTER(u32), ctypes.POINTER(u32), ctypes.POINTER(u32)]),
    "sb_groth16_prove": (ctypes.c_int, [vp, u64, vp, u64, vp, vp, vp]),
    "sb_groth16_prove_wtns": (ctypes.c_int, [vp, u64, vp, u64, vp, vp, vp]),
    "sb_groth16_prove_batch": (ctypes.c_int, [vp, u64, vp, u64, u32, vp, vp, vp]),
    "sb_groth16_release": (ctypes.c_int, [vp, u64]),
    "sb_groth16_verify_batch": (ctypes.c_int, [vp, vp, u64, u32, vp, vp, u32, vp]),
    "sb_plonk_verify_batch": (ctypes.c_int, [vp, vp, u64, u32, u32, vp, vp, u32, vp]),
    "sb_fflonk_verify_batch": (ctypes.c_int, [vp, vp, u64, u32, u32, vp, vp, u32, vp]),
    "sb_pairing_eval": (ctypes.c_int, [vp, ctypes.c_int, vp, u64, vp]),
    "sb_plonk_load": (ctypes.c_int, [vp, vp, u64, ctypes.POINTER(u64)]),
    "sb_plonk_load_file": (ctypes.c_int, [vp, ctypes.c_char_p, ctypes.POINTER(u64)]),
    "sb_plonk_info": (ctypes.c_int, [vp, u64, ctypes.POINTER(u32), ctypes.POINTER(u32), ctypes.POINTER(u32), ctypes.POINTER(u32)]),
    "sb_plonk_proof_bytes": (u32, [vp]),
    "sb_plonk_prove": (ctypes.c_int, [vp, u64, vp, u64, ctypes.c_char_p, vp]),
    "sb_plonk_prove_batch": (ctypes.c_int, [vp, u64, vp, u64, u32, vp, vp, vp]),
    "sb_plonk_prove_resident": (ctypes.c_int, [vp, u64, ctypes.c_char_p, vp]),
    "sb_plonk_release": (ctypes.c_int, [vp, u64]),
    "sb_fflonk_load": (ctypes.c_int, [vp, vp, u64, ctypes.POINTER(u64)]),
    "sb_fflonk_load_file": (ctypes.c_int, [vp, ctypes.c_char_p, ctypes.POINTER(u64)]),
    "sb_fflonk_info": (ctypes.c_int, [vp, u64, ctypes.POINTER(u32), ctypes.POINTER(u32), ctypes.POINTER(u32), ctypes.POINTER(u32)]),
    "sb_fflonk_proof_bytes": (u32, [vp]),
    "sb_fflonk_prove": (ctypes.c_int, [vp, u64, vp, u64, ctypes.c_char_p, vp]),
    "sb_fflonk_prove_resident": (ctypes.c_int, [vp, u64, ctypes.c_char_p, vp]),
    "sb_fflonk_prove_batch": (ctypes.c_int, [vp, u64, vp, u64, u32, vp, vp, vp]),
    "sb_fflonk_release": (ctypes.c_int, [vp, u64]),
    "sb_plonk_load_multi": (ctypes.c_int, [ctypes.POINTER(vp), ctypes.c_int, vp, u64, ctypes.POINTER(u64)]),
    "sb_plonk_prove_multi": (ctypes.c_int, [ctypes.POINTER(vp), ctypes.POINTER(u64), ctypes.c_int, vp, u64, ctypes.c_char_p, vp]),
    "sb_fflonk_load_multi": (ctypes.c_int, [ctypes.POINTER(vp), ctypes.c_int, vp, u64, ctypes.POINTER(u64)]),
    "sb_fflonk_prove_multi": (ctypes.c_int, [ctypes.POINTER(vp), ctypes.POINTER(u64), ctypes.c_int, vp, u64, ctypes.c_char_p, vp]),
    "sb_groth16_load_replicas": (ctypes.c_int, [ctypes.POINTER(vp), ctypes.c_int, vp, u64, ctypes.POINTER(u64)]),
    "sb_plonk_load_replicas": (ctypes.c_int, [ctypes.POINTER(vp), ctypes.c_int, vp, u64, ctypes.POINTER(u64)]),
    "sb_fflonk_load_replicas": (ctypes.c_int, [ctypes.POINTER(vp), ctypes.c_int, vp, u64, ctypes.POINTER(u64)]),
    "sb_groth16_prove_batch_multi": (ctypes.c_int, [ctypes.POINTER(vp), ctypes.POINTER(u64), ctypes.c_int, vp, u64, u32, vp, vp, vp]),
    "sb_plonk_prove_batch_multi": (ctypes.c_int, [ctypes.POINTER(vp), ctypes.POINTER(u64), ctypes.c_int, vp, u64, u32, vp, vp, vp]),
    "sb_fflonk_prove_batch_multi": (ctypes.c_int, [ctypes.POINTER(vp), ctypes.POINTER(u64), ctypes.c_int, vp, u64, u32, vp, vp, vp]),
    "sb_groth16_prove_resident": (ctypes.c_int, [vp, u64, vp, vp, vp]),
    "sb_last_stat": (ctypes.c_double, [vp, ctypes.c_int]),
    "sb_calibrate": (ctypes.c_double, [vp, ctypes.c_int]),
    "sb_set_tuning": (ctypes.c_int, [ctypes.c_int, ctypes.c_int]),
    "sb_gen_points": (ctypes.c_int, [vp, ctypes.c_int, u64, u64, vp]),
    "sb_generator": (ctypes.c_int, [vp, ctypes.c_int, vp]),
    "sb_field_eval": (ctypes.c_int, [vp, ctypes.c_int, ctypes.c_int, vp, u64, vp]),
    "sb_ntt_eval": (ctypes.c_int, [vp, ctypes.c_int, ctypes.c_int, ctypes.c_int, ctypes.c_int, vp, vp, vp, vp, vp]),
    "sb_groth16_prove_shard": (ctypes.c_int, [vp, u64, vp, u64, ctypes.c_int, ctypes.c_int, vp]),
    "sb_groth16_partials_bytes": (u32, [vp]),
    "sb_groth16_finish": (ctypes.c_int, [vp, u64, vp, ctypes.c_int, vp, vp, vp]),
    "sb_comm_unique_id": (ctypes.c_int, [vp]),
    "sb_comm_init_rank": (ctypes.c_int, [vp, ctypes.c_int, ctypes.c_int, vp]),
    "sb_comm_info": (ctypes.c_int, [vp, ctypes.POINTER(ctypes.c_int), ctypes.POINTER(ctypes.c_int)]),
    "sb_comm_destroy": (ctypes.c_int, [vp]),
    "sb_dist_chain_owner": (ctypes.c_int, [ctypes.c_int, ctypes.c_int]),
    "sb_groth16_prove_dist": (ctypes.c_int, [vp, u64, vp, u64, vp, vp, vp]),
    "sb_create_multi": (ctypes.c_int, [ctypes.c_int, ctypes.POINTER(ctypes.c_int), ctypes.c_int, ctypes.POINTER(vp)]),
    "sb_groth16_load_multi": (ctypes.c_int, [ctypes.POINTER(vp), ctypes.c_int, vp, u64, ctypes.POINTER(u64)]),
    "sb_groth16_prove_multi": (ctypes.c_int, [ctypes.POINTER(vp), ctypes.POINTER(u64), ctypes.c_int, vp, u64, vp, vp, vp]),
    "sb_host_sum_partials": (ctypes.c_int, [ctypes.c_int, ctypes.c_int, vp, ctypes.c_int, vp]),
    "sb_host_partial_from_affine": (ctypes.c_int, [ctypes.c_int, ctypes.c_int, vp, vp]),
    "sb_host_partial_bytes": (u32, [ctypes.c_int, ctypes.c_int]),
    "sb_host_groth16_finish": (ctypes.c_int, [ctypes.c_int, vp, vp, vp, vp, vp, vp, ctypes.c_int, vp, vp, vp]),
    "sb_shard_range": (None, [u64, ctypes.c_int, ctypes.c_int, ctypes.POINTER(u64), ctypes.POINTER(u64)]),
    "sb_msm_dev": (ctypes.c_int, [vp, ctypes.c_int, vp, vp, u32, u64, vp]),
    "sb_ntt_fr_dev": (ctypes.c_int, [vp, vp, vp, u64, ctypes.c_int, ctypes.POINTER(vp)]),
    "sb_dev_alloc": (vp, [vp, u64]),
    "sb_dev_free": (ctypes.c_int, [vp, vp]),
    "sb_dev_upload": (ctypes.c_int, [vp, vp, vp, u64]),
    "sb_dev_download": (ctypes.c_int, [vp, vp, vp, u64]),
    "sb_last_ms": (ctypes.c_float, [vp, ctypes.c_int]),
    "sb_sync": (ctypes.c_int, [vp]),
}

EXPORTED_SYMBOLS = tuple(_SIGNATURES)


def build(verbose: bool = False) -> str:
    """Compile libsnarkb200.so in-tree for sm_90a (nvcc cross-compiles without a GPU)."""
    cmd = ["make", "-C", os.path.join(_HERE, "csrc"), "-j8"]
    subprocess.check_call(cmd, stdout=None if verbose else subprocess.DEVNULL)
    return LIB_PATH


def _prefer_bundled_nccl():
    """libsnarkb200 dlopens libnccl.so.2 on first multi-GPU use (SB_NCCL_LIB first).  In a Python process that also imports
    torch, torch's bundled libnccl (a newer build under the same soname) must be the copy in the process: the first one
    loaded wins, and torch cannot import against an older system copy.  Point the library at the bundled file unless the
    caller chose one; a Node host has no torch and uses the system libnccl."""
    if os.environ.get("SB_NCCL_LIB"):
        return
    try:
        import importlib.util
        spec = importlib.util.find_spec("nvidia.nccl")
        for base in (spec.submodule_search_locations if spec else []):
            cand = os.path.join(base, "lib", "libnccl.so.2")
            if os.path.exists(cand):
                os.environ["SB_NCCL_LIB"] = cand
                return
    except Exception:
        pass


def lib():
    global _lib
    if _lib is None:
        if not os.path.exists(LIB_PATH):
            raise RuntimeError(f"{LIB_PATH} is missing: build it with `make -C snarkjs_b200/csrc` "
                               "(there is no CPU fallback)")
        _prefer_bundled_nccl()
        L = ctypes.CDLL(LIB_PATH)
        for name, (res, args) in _SIGNATURES.items():
            fn = getattr(L, name)           # raises AttributeError if a declared symbol is not exported
            fn.restype = res
            fn.argtypes = args
        _lib = L
        # profiling and test switches without code changes: SB_TUNE="key=value,key=value" -> sb_set_tuning (keys in
        # include/snarkb200.h; every setting computes the same bytes, an unknown key is an error)
        for kv in filter(None, os.environ.get("SB_TUNE", "").split(",")):
            k, v = kv.split("=")
            if L.sb_set_tuning(int(k), int(v)) != 0:
                raise RuntimeError(f"SB_TUNE: sb_set_tuning({k}, {v}) rejected")
    return _lib
