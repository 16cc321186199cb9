"""ctypes binding of include/b2kyber.h -- the same C ABI a Go adapter binds with cgo.

There is no CPU fallback: importing this without the built library, or creating an Engine
without an sm_90 device, raises.
"""
from __future__ import annotations
import ctypes as C
import os

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_HERE, "libb2kyber.so")

B2K_OK, ERR_CUDA, ERR_ARG, ERR_SCALAR_RANGE, ERR_NO_DEVICE, ERR_POINT, ERR_COMM = 0, -1, -2, -3, -4, -5, -6
COMM_BLOB_BYTES, MAX_RANKS = 128, 16


class B2KError(RuntimeError):
    def __init__(self, code: int, msg: str):
        super().__init__(f"b2kyber error {code}: {msg}")
        self.code = code


def load_library() -> C.CDLL:
    if not os.path.exists(LIB_PATH):
        raise ImportError(f"{LIB_PATH} is missing: build it with `python -m kyber_b200.build` "
                          "(there is no CPU fallback)")
    lib = C.CDLL(LIB_PATH)
    vp, sz, u8p = C.c_void_p, C.c_size_t, C.c_char_p
    sigs = {
        "b2k_create": (C.c_int, [C.c_int, C.POINTER(vp)]),
        "b2k_destroy": (None, [vp]),
        "b2k_last_error": (C.c_char_p, [vp]),
        "b2k_version": (C.c_char_p, []),
        "b2k_set_stream": (C.c_int, [vp, vp]),
        "b2k_synchronize": (C.c_int, [vp]),
        "b2k_wait": (C.c_int, [vp]),
        "b2k_last_timings": (C.c_int, [vp, C.POINTER(C.c_float), C.c_int]),
        "b2k_set_msm_window": (C.c_int, [vp, C.c_int]),
        "b2k_launch_count": (C.c_uint64, [vp]),
        "b2k_set_msm_slice": (C.c_int, [vp, C.c_int]),
        "b2k_set_msm_variant": (C.c_int, [vp, C.c_int]),
        "b2k_set_msm_glv": (C.c_int, [vp, C.c_int]),
        "b2k_set_pairing_variant": (C.c_int, [vp, C.c_int]),
        "b2k_set_pairing_coop": (C.c_int, [vp, C.c_int]),
        "b2k_set_msm_groups": (C.c_int, [vp, C.c_int]),
        "b2k_set_msm_occupancy": (C.c_int, [vp, C.c_int]),
        "b2k_set_msm_chunk": (C.c_int, [vp, C.c_int]),
        "b2k_set_msm_reduce": (C.c_int, [vp, C.c_int, C.c_int, C.c_int]),
        "b2k_set_msm_affine": (C.c_int, [vp, C.c_int, C.c_int]),
        "b2k_last_msm_plan": (C.c_int, [vp, C.POINTER(C.c_int), C.c_int]),
        "b2k_set_msm_affine_split": (C.c_int, [vp, C.c_int]),
        "b2k_set_msm_staging": (C.c_int, [vp, C.c_int]),
        "b2k_set_mul_occupancy": (C.c_int, [vp, C.c_int]),
        "b2k_set_msm_layout": (C.c_int, [vp, C.c_int]),
    }
    sigs["b2k_bls12381_pair"] = (C.c_int, [vp, sz, vp, vp, vp])
    sigs["b2k_bls12381_pair_dev"] = (C.c_int, [vp, sz, vp, vp, vp])
    sigs["b2k_bls12381_pairing_check"] = (C.c_int, [vp, sz, vp, vp, vp, vp, vp])
    sigs["b2k_bls12381_pairing_check_dev"] = (C.c_int, [vp, sz, vp, vp, vp, vp, vp])
    sigs["b2k_bls12381_pair_fixed_g2"] = (C.c_int, [vp, sz, vp, vp, vp])
    for g in ("g1", "g2"):
        sigs[f"b2k_bls12381_ibe_decrypt_cca_{g}"] = (C.c_int, [vp, vp, sz, vp, sz, vp, vp, vp, vp])
        sigs[f"b2k_bls12381_ibe_encrypt_cca_{g}"] = (C.c_int, [vp, vp, vp, sz, vp, sz, sz, sz, vp, vp, vp, vp, vp])
    sigs["b2k_bls12381_hash_to_g1"] = (C.c_int, [vp, sz, vp, vp, vp, C.c_uint32, vp])
    sigs["b2k_bls12381_hash_to_g1_dev"] = (C.c_int, [vp, sz, vp, vp, vp, C.c_uint32, vp])
    sigs["b2k_bls12381_hash_to_g2"] = (C.c_int, [vp, sz, vp, vp, vp, C.c_uint32, vp])
    sigs["b2k_bls12381_hash_to_g2_dev"] = (C.c_int, [vp, sz, vp, vp, vp, C.c_uint32, vp])
    sigs["b2k_bls12381_verify_g2sig"] = (C.c_int, [vp, sz, vp, vp, vp, vp, C.c_uint32, vp, vp])
    sigs["b2k_bls12381_verify_g2sig_dev"] = (C.c_int, [vp, sz, vp, vp, vp, vp, C.c_uint32, vp, vp])
    sigs["b2k_bls12381_verify_g1sig"] = (C.c_int, [vp, sz, vp, vp, vp, vp, C.c_uint32, vp, vp])
    sigs["b2k_bls12381_verify_g1sig_dev"] = (C.c_int, [vp, sz, vp, vp, vp, vp, C.c_uint32, vp, vp])
    sigs["b2k_ed25519_verify"] = (C.c_int, [vp, sz, vp, vp, vp, vp, vp])
    sigs["b2k_ed25519_verify_dev"] = (C.c_int, [vp, sz, vp, vp, vp, vp, vp])
    sigs["b2k_ed25519_recover_commit"] = (C.c_int, [vp, sz, vp, vp, vp])
    sigs["b2k_ed25519_pubpoly_eval"] = (C.c_int, [vp, sz, vp, sz, vp, vp])
    sigs["b2k_ed25519_pubpoly_check"] = (C.c_int, [vp, sz, sz, vp, sz, vp, vp, vp])
    sigs["b2k_ed25519_dleq_verify"] = (C.c_int, [vp, sz, vp, vp, vp, vp, vp, vp])
    sigs["b2k_ed25519_dleq_verify_dev"] = (C.c_int, [vp, sz, vp, vp, vp, vp, vp, vp])
    sigs["b2k_ed25519_pvss_verify_enc_shares"] = (C.c_int, [vp, sz, sz, sz, vp, vp, vp, vp, vp, vp, vp])
    sigs["b2k_ed25519_pvss_verify_dec_shares"] = (C.c_int, [vp, sz, vp, vp, vp, vp, vp, vp])
    sigs["b2k_ed25519_shuffle_verify"] = (C.c_int, [vp, sz, sz, vp, vp, vp, vp, vp, vp, vp, vp, C.c_uint32, vp])
    sigs["b2k_ed25519_shuffle_sequence_verifiable"] = (C.c_int, [vp, sz, sz, vp, vp, vp, vp, vp, vp, vp, vp, vp])
    sigs["b2k_ed25519_anon_verify"] = (C.c_int, [vp, sz, vp, C.c_int, vp, sz, sz, vp, vp, vp, vp, vp])
    sigs["b2k_ed25519_ecies_decrypt"] = (C.c_int, [vp, vp, sz, sz, vp, vp, vp])
    sigs["b2k_ed25519_ecies_encrypt"] = (C.c_int, [vp, sz, vp, vp, sz, vp, vp, vp])
    sigs["b2k_bn254_pairing_check"] = (C.c_int, [vp, sz, vp, vp, vp, vp, vp])
    sigs["b2k_bn256_pairing_check"] = (C.c_int, [vp, sz, vp, vp, vp, vp, vp])
    sigs["b2k_bn254_recover_commit"] = (C.c_int, [vp, sz, vp, vp, vp])
    sigs["b2k_bls12381_g1_recover_commit"] = (C.c_int, [vp, sz, vp, vp, vp])
    sigs["b2k_bls12381_g2_recover_commit"] = (C.c_int, [vp, sz, vp, vp, vp])
    sigs["b2k_bls12381_g1_pubpoly_eval"] = (C.c_int, [vp, sz, vp, sz, vp, vp])
    sigs["b2k_bls12381_g2_pubpoly_eval"] = (C.c_int, [vp, sz, vp, sz, vp, vp])
    for nm in ("b2k_bn254_g1_unmarshal_check", "b2k_bn254_g2_unmarshal_check", "b2k_bn256_g1_unmarshal_check", "b2k_bn256_g2_unmarshal_check"):
        sigs[nm] = (C.c_int, [vp, sz, vp, vp])
    for nm in ("b2k_bls12381_g1_pubpoly_check", "b2k_bls12381_g2_pubpoly_check", "b2k_bn254_pubpoly_check"):
        sigs[nm] = (C.c_int, [vp, sz, sz, vp, sz, vp, vp, vp])
    sigs["b2k_bls12381_g1_msm_bucket_plan"] = (C.c_int, [vp, sz, C.POINTER(C.c_int)])
    sigs["b2k_bls12381_g1_msm_buckets_dev"] = (C.c_int, [vp, sz, vp, vp, vp, sz, C.POINTER(C.c_int)])
    sigs["b2k_bls12381_g1_msm_reduce_windows_dev"] = (C.c_int, [vp, C.c_int, C.c_int, C.c_int, vp, vp])
    sigs["b2k_bls12381_g1_msm_finish_dev"] = (C.c_int, [vp, C.c_int, C.c_int, vp, vp, C.c_int])
    for cv in ("bls12381", "bn254"):
        sigs[f"b2k_{cv}_gt_mul"] = (C.c_int, [vp, sz, vp, vp, vp])
        sigs[f"b2k_{cv}_gt_inv"] = (C.c_int, [vp, sz, vp, vp])
        sigs[f"b2k_{cv}_gt_exp"] = (C.c_int, [vp, sz, vp, vp, vp])
    for nm in ("b2k_bls12381_miller", "b2k_bn254_miller", "b2k_bn256_miller", "b2k_bls12381_pairing_product_check",
               "b2k_bls12381_pairing_product", "b2k_bn254_pairing_product_check", "b2k_bn256_pairing_product_check"):
        sigs[nm] = (C.c_int, [vp, sz, vp, vp, vp])
    for nm in ("b2k_bls12381_final_exp", "b2k_bn254_finalize", "b2k_bn256_finalize"):
        sigs[nm] = (C.c_int, [vp, sz, vp, vp])
    for nm in ("b2k_bls12381_g1_add_batch", "b2k_bls12381_g2_add_batch"):
        sigs[nm] = (C.c_int, [vp, sz, vp, vp, C.c_int, vp])
    for nm in ("b2k_bls12381_g1_recover_pubpoly", "b2k_bls12381_g2_recover_pubpoly", "b2k_bn254_recover_pubpoly",
               "b2k_bls12381_g1_commit_batch", "b2k_bls12381_g2_commit_batch", "b2k_bn254_commit_batch"):
        sigs[nm] = (C.c_int, [vp, sz, vp, vp, vp])
    sigs["b2k_bn256_hash_g1"] = (C.c_int, [vp, sz, vp, vp, vp, C.c_uint32, vp])
    sigs["b2k_bn256_hash_g1_dev"] = (C.c_int, [vp, sz, vp, vp, vp, C.c_uint32, vp])
    sigs["b2k_comm_create"] = (C.c_int, [vp, C.c_int, C.c_int, C.POINTER(vp)])
    sigs["b2k_comm_export"] = (C.c_int, [vp, vp])
    sigs["b2k_comm_connect"] = (C.c_int, [vp, vp])
    sigs["b2k_comm_connect_local"] = (C.c_int, [C.POINTER(vp), C.c_int])
    sigs["b2k_nccl_unique_id"] = (C.c_int, [vp])
    sigs["b2k_comm_use_nccl"] = (C.c_int, [vp, vp])
    sigs["b2k_comm_destroy"] = (None, [vp])
    sigs["b2k_comm_last_plan"] = (C.c_int, [vp, C.POINTER(C.c_int)])
    sigs["b2k_bls12381_g1_msm_sharded_dev"] = (C.c_int, [vp, sz, vp, vp, vp, C.c_int])
    sigs["b2k_bls12381_g1_msm_sharded_async"] = (C.c_int, [vp, sz, vp, vp, vp])
    sigs["b2k_bls12381_g1_msm_multi_gpu"] = (C.c_int, [C.POINTER(vp), C.c_int, sz, vp, vp, vp])
    host3 = (C.c_int, [vp, sz, vp, vp, vp])
    for name in HOST_FUNCS + DEV_FUNCS:
        sigs[name] = host3
    for name, (res, args) in sigs.items():
        fn = getattr(lib, name)      # AttributeError here = ABI drift between header and library
        fn.restype, fn.argtypes = res, args
    return lib


HOST_FUNCS = [
    "b2k_bn254_pair", "b2k_bn254_g2_mul_batch", "b2k_bn254_g2_msm", "b2k_bn256_pair",
    "b2k_bn256_g1_mul_batch", "b2k_bn256_g1_msm", "b2k_bn256_g2_mul_batch", "b2k_bn256_g2_msm",
    "b2k_bls12381_g1_msm_affine", "b2k_bls12381_g2_msm_affine",
    "b2k_bls12381_g2_mul_batch", "b2k_bls12381_g2_mul_batch_affine", "b2k_bls12381_g2_msm",
    "b2k_bls12381_g1_decompress", "b2k_bls12381_g2_decompress",
    "b2k_bls12381_g1_mul_batch", "b2k_bls12381_g1_mul_batch_affine", "b2k_bls12381_g1_msm",
    "b2k_bn254_g1_mul_batch", "b2k_bn254_g1_msm", "b2k_ed25519_mul_batch", "b2k_ed25519_msm",
]
DEV_FUNCS = [
    "b2k_bls12381_g2_mul_batch_affine_dev", "b2k_bls12381_g2_msm_dev",
    "b2k_bls12381_g1_decompress_dev", "b2k_bls12381_g2_decompress_dev",
    "b2k_bls12381_g1_mul_batch_dev", "b2k_bls12381_g1_mul_batch_affine_dev", "b2k_bls12381_g1_msm_dev",
    "b2k_bls12381_g1_msm_affine_dev", "b2k_bn254_g1_msm_dev", "b2k_ed25519_mul_batch_dev", "b2k_ed25519_msm_dev",
]


def _buf(b):
    """bytes-like -> (ctypes pointer, keepalive)."""
    if isinstance(b, (bytes, bytearray)):
        arr = (C.c_char * len(b)).from_buffer_copy(b) if isinstance(b, bytes) else (C.c_char * len(b)).from_buffer(b)
        return C.cast(arr, C.c_void_p), arr
    if isinstance(b, int):
        return C.c_void_p(b), None
    mv = memoryview(b)
    arr = (C.c_char * mv.nbytes).from_buffer(mv)
    return C.cast(arr, C.c_void_p), arr


class Engine:
    """One b2k context (one CUDA stream + scratch arena) on one device."""

    def __init__(self, device: int = 0):
        self.lib = load_library()
        h = C.c_void_p()
        rc = self.lib.b2k_create(device, C.byref(h))
        if rc != 0:
            raise B2KError(rc, "b2k_create failed (no sm_90 device? there is no CPU fallback)")
        self.h = h
        self.device = device

    def close(self):
        if getattr(self, "h", None):
            self.lib.b2k_destroy(self.h)
            self.h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def _check(self, rc: int):
        if rc != 0:
            raise B2KError(rc, (self.lib.b2k_last_error(self.h) or b"").decode())

    # -- generic calls ---------------------------------------------------------------------------
    def call_host(self, name: str, n: int, scalars, points, out_len: int) -> bytes:
        out = bytearray(out_len)
        ps, k1 = _buf(scalars); pp, k2 = _buf(points); po, k3 = _buf(out)
        self._check(getattr(self.lib, name)(self.h, n, ps, pp, po))
        return bytes(out)

    def call_dev(self, name: str, n: int, d_scalars: int, d_points: int, d_out: int):
        self._check(getattr(self.lib, name)(self.h, n, C.c_void_p(d_scalars), C.c_void_p(d_points), C.c_void_p(d_out)))

    def set_stream(self, cuda_stream: int):
        self._check(self.lib.b2k_set_stream(self.h, C.c_void_p(cuda_stream)))

    def wait(self):
        """synchronise and raise the deferred status (scalar range / malformed point) of everything enqueued since the last wait"""
        self._check(self.lib.b2k_wait(self.h))

    def synchronize(self):
        self._check(self.lib.b2k_synchronize(self.h))

    def set_msm_window(self, c: int):
        self._check(self.lib.b2k_set_msm_window(self.h, c))

    def set_msm_slice(self, L: int):
        self._check(self.lib.b2k_set_msm_slice(self.h, L))

    def set_msm_groups(self, groups: int):
        """window groups of the overlapped MSM tail; 1 = serial pipeline (per-stage timings meaningful)"""
        self._check(self.lib.b2k_set_msm_groups(self.h, groups))

    def set_msm_variant(self, one_thread_per_bucket: bool):
        self._check(self.lib.b2k_set_msm_variant(self.h, int(one_thread_per_bucket)))

    def set_msm_glv(self, on: bool):
        """BLS12-381 G1 MSM: endomorphism split on (default) / off (plain 255-bit pipeline)"""
        self._check(self.lib.b2k_set_msm_glv(self.h, int(on)))

    def set_msm_affine(self, rounds: int = -1, batch: int = 0):
        """affine pair-tree rounds of the BLS12-381 G1 MSM: -1 automatic, 0 off, 1..8 forced; batch = additions per thread"""
        self._check(self.lib.b2k_set_msm_affine(self.h, int(rounds), int(batch)))

    def set_pairing_coop(self, max_n: int):
        """batches of at most max_n BLS12-381 pairings / checks run one per warp (coop_pairing.cuh); 0 = never"""
        self._check(self.lib.b2k_set_pairing_coop(self.h, int(max_n)))

    def set_msm_affine_split(self, split: bool):
        """affine rounds as three kernels each (True, default) or one fused kernel (False)"""
        self._check(self.lib.b2k_set_msm_affine_split(self.h, int(split)))

    def set_mul_occupancy(self, blocks_per_sm: int):
        self._check(self.lib.b2k_set_mul_occupancy(self.h, int(blocks_per_sm)))

    def set_msm_reduce(self, levels: int = 0, m1: int = 0, m2: int = 0):
        """bucket reduction in one or two levels (0 = automatic); A/B and tuning aid"""
        self._check(self.lib.b2k_set_msm_reduce(self.h, int(levels), int(m1), int(m2)))

    def last_msm_plan(self) -> dict:
        """parameters of the last MSM: window bits, windows, chunk, slice length, affine rounds and their batch widths"""
        arr = (C.c_int * 20)()
        n = self.lib.b2k_last_msm_plan(self.h, arr, 20)
        if n < 0:
            self._check(n)
        return {"c": arr[0], "W": arr[1], "buckets_per_window": arr[2], "chunk": arr[3], "slice_len": arr[4],
                "affine_rounds": arr[5], "affine_batch": [arr[6 + r] for r in range(arr[5])], "glv": bool(arr[14]),
                "affine_split": bool(arr[15]), "reduce_levels": arr[16], "reduce_chunks": [arr[17], arr[18]] if arr[16] == 2 else [arr[17]]}

    def last_timings(self):
        arr = (C.c_float * 16)()
        n = self.lib.b2k_last_timings(self.h, arr, 16)
        if n < 0:
            self._check(n)
        return [float(arr[i]) for i in range(n)]

    def launch_count(self) -> int:
        return int(self.lib.b2k_launch_count(self.h))

    # -- multi-GPU MSM by partial-bucket exchange (device pointers; see kyber_b200/multi.py) ---------
    def bls12381_g1_msm_bucket_plan(self, n: int) -> dict:
        arr = (C.c_int * 4)()
        self._check(self.lib.b2k_bls12381_g1_msm_bucket_plan(self.h, n, arr))
        return {"c": arr[0], "W": arr[1], "buckets_per_window": arr[2], "bucket_bytes": arr[3]}

    def bls12381_g1_msm_buckets_dev(self, n: int, d_scalars: int, d_points: int, d_buckets: int, cap_bytes: int):
        self._check(self.lib.b2k_bls12381_g1_msm_buckets_dev(self.h, n, C.c_void_p(d_scalars), C.c_void_p(d_points),
                                                             C.c_void_p(d_buckets), cap_bytes, None))

    def bls12381_g1_msm_reduce_windows_dev(self, c: int, w_cnt: int, parts: int, d_recv: int, d_wsum: int):
        self._check(self.lib.b2k_bls12381_g1_msm_reduce_windows_dev(self.h, c, w_cnt, parts, C.c_void_p(d_recv), C.c_void_p(d_wsum)))

    def bls12381_g1_msm_finish_dev(self, c: int, W: int, d_wsum: int, d_out: int, affine_out: bool = False):
        self._check(self.lib.b2k_bls12381_g1_msm_finish_dev(self.h, c, W, C.c_void_p(d_wsum), C.c_void_p(d_out), 1 if affine_out else 0))

    # -- BLS12-381 G1 -----------------------------------------------------------------------------
    def bls12381_g1_mul_batch(self, scalars: bytes, points: bytes) -> bytes:
        n = len(scalars) // 32
        assert len(scalars) == 32 * n and len(points) == 96 * n
        return self.call_host("b2k_bls12381_g1_mul_batch", n, scalars, points, 48 * n)

    def bls12381_g1_mul_batch_affine(self, scalars: bytes, points: bytes) -> bytes:
        n = len(scalars) // 32
        assert len(scalars) == 32 * n and len(points) == 96 * n
        return self.call_host("b2k_bls12381_g1_mul_batch_affine", n, scalars, points, 96 * n)

    def bls12381_g1_msm(self, scalars: bytes, points: bytes) -> bytes:
        n = len(scalars) // 32
        assert len(scalars) == 32 * n and len(points) == 96 * n
        return self.call_host("b2k_bls12381_g1_msm", n, scalars, points, 48)

    # -- BLS12-381 G2 -----------------------------------------------------------------------------------
    def bls12381_g2_mul_batch(self, scalars: bytes, points: bytes) -> bytes:
        n = len(scalars) // 32
        assert len(scalars) == 32 * n and len(points) == 192 * n
        return self.call_host("b2k_bls12381_g2_mul_batch", n, scalars, points, 96 * n)

    def bls12381_g2_mul_batch_affine(self, scalars: bytes, points: bytes) -> bytes:
        n = len(scalars) // 32
        assert len(scalars) == 32 * n and len(points) == 192 * n
        return self.call_host("b2k_bls12381_g2_mul_batch_affine", n, scalars, points, 192 * n)

    def bls12381_g2_msm(self, scalars: bytes, points: bytes) -> bytes:
        n = len(scalars) // 32
        assert len(scalars) == 32 * n and len(points) == 192 * n
        return self.call_host("b2k_bls12381_g2_msm", n, scalars, points, 96)

    # -- UnmarshalBinary batches ------------------------------------------------------------------------
    def _decompress(self, name: str, data: bytes, in_len: int, out_len: int):
        n = len(data) // in_len
        assert len(data) == in_len * n
        out, ok = bytearray(out_len * n), bytearray(n)
        bufs = [_buf(x) for x in (data, out, ok)]
        self._check(getattr(self.lib, name)(self.h, n, *[b[0] for b in bufs]))
        return bytes(out), bytes(ok)

    def bls12381_g1_decompress(self, data: bytes):
        """-> (operand bytes [n][96], ok flags [n])"""
        return self._decompress("b2k_bls12381_g1_decompress", data, 48, 96)

    def bls12381_g2_decompress(self, data: bytes):
        return self._decompress("b2k_bls12381_g2_decompress", data, 96, 192)

    # -- hash-to-G1 / BLS verify -------------------------------------------------------------------------
    @staticmethod
    def _pack_msgs(msgs):
        import struct
        offs, blob, pos = [0], b"", 0
        for m in msgs:
            pos += len(m)
            offs.append(pos)
        blob = b"".join(msgs) or b"\x00"
        return blob, struct.pack("<%dI" % len(offs), *offs)

    def bls12381_hash_to_g1(self, msgs, dst: bytes) -> bytes:
        """msgs: list of bytes -> operand bytes [n][96]"""
        n = len(msgs)
        blob, offs = self._pack_msgs(msgs)
        out = bytearray(96 * n)
        bufs = [_buf(x) for x in (blob, offs, dst, out)]
        self._check(self.lib.b2k_bls12381_hash_to_g1(self.h, n, bufs[0][0], bufs[1][0], bufs[2][0], len(dst), bufs[3][0]))
        return bytes(out)

    def bn254_hash_to_g1(self, msgs, dst: bytes = b"BN254G1_XMD:KECCAK-256_SVDW_RO_") -> bytes:
        """bn254 pointG1.Hash (Keccak-256 XMD + SvdW) for a list of messages -> [n][64] x||y"""
        n = len(msgs)
        blob, offs = self._pack_msgs(msgs)
        out = bytearray(64 * n)
        bufs = [_buf(x) for x in (blob, offs, dst, out)]
        self.lib.b2k_bn254_hash_to_g1.restype = C.c_int
        self.lib.b2k_bn254_hash_to_g1.argtypes = [C.c_void_p, C.c_size_t, C.c_void_p, C.c_void_p, C.c_void_p, C.c_uint32, C.c_void_p]
        self._check(self.lib.b2k_bn254_hash_to_g1(self.h, n, bufs[0][0], bufs[1][0], bufs[2][0], len(dst), bufs[3][0]))
        return bytes(out)

    def bn256_hash_to_g1(self, msgs) -> bytes:
        """bn256 pointG1.Hash (SHA-256 try-and-increment) for a list of messages -> [n][64] x||y"""
        n = len(msgs)
        blob, offs = self._pack_msgs(msgs)
        out = bytearray(64 * n)
        bufs = [_buf(x) for x in (blob, offs, out)]
        self.lib.b2k_bn256_hash_to_g1.restype = C.c_int
        self.lib.b2k_bn256_hash_to_g1.argtypes = [C.c_void_p, C.c_size_t, C.c_void_p, C.c_void_p, C.c_void_p]
        self._check(self.lib.b2k_bn256_hash_to_g1(self.h, n, bufs[0][0], bufs[1][0], bufs[2][0]))
        return bytes(out)

    def bn256_hash_g1(self, msgs, dst: bytes = b"") -> bytes:
        """bn256 HashG1 (HKDF-SHA256 + SvdW, pairing/bn256/hash.go:10-110) for a list of messages -> [n][64] x||y"""
        n = len(msgs)
        blob, offs = self._pack_msgs(msgs)
        out = bytearray(64 * n)
        bufs = [_buf(x) for x in (blob, offs, dst or b"\x00", out)]
        self._check(self.lib.b2k_bn256_hash_g1(self.h, n, bufs[0][0], bufs[1][0], bufs[2][0] if dst else None, len(dst), bufs[3][0]))
        return bytes(out)

    def bls12381_hash_to_g2(self, msgs, dst: bytes) -> bytes:
        """msgs: list of bytes -> operand bytes [n][192]"""
        n = len(msgs)
        blob, offs = self._pack_msgs(msgs)
        out = bytearray(192 * n)
        bufs = [_buf(x) for x in (blob, offs, dst, out)]
        self._check(self.lib.b2k_bls12381_hash_to_g2(self.h, n, bufs[0][0], bufs[1][0], bufs[2][0], len(dst), bufs[3][0]))
        return bytes(out)

    def bls12381_verify_g2sig(self, pks: bytes, msgs, dst: bytes, sigs: bytes) -> bytes:
        """n x bls.Verify (sigs on G2): pks [n][48] compressed G1, sigs [n][96] compressed G2 -> ok flags [n]"""
        n = len(msgs)
        assert len(pks) == 48 * n and len(sigs) == 96 * n
        blob, offs = self._pack_msgs(msgs)
        ok = bytearray(n)
        bufs = [_buf(x) for x in (pks, blob, offs, dst, sigs, ok)]
        self._check(self.lib.b2k_bls12381_verify_g2sig(self.h, n, bufs[0][0], bufs[1][0], bufs[2][0], bufs[3][0], len(dst),
                                                       bufs[4][0], bufs[5][0]))
        return bytes(ok)

    def bls12381_verify_g1sig(self, pks: bytes, msgs, dst: bytes, sigs: bytes) -> bytes:
        """n x bls.Verify (sigs on G1): pks [n][96] compressed G2, sigs [n][48] compressed G1 -> ok flags [n]"""
        n = len(msgs)
        assert len(pks) == 96 * n and len(sigs) == 48 * n
        blob, offs = self._pack_msgs(msgs)
        ok = bytearray(n)
        bufs = [_buf(x) for x in (pks, blob, offs, dst, sigs, ok)]
        self._check(self.lib.b2k_bls12381_verify_g1sig(self.h, n, bufs[0][0], bufs[1][0], bufs[2][0], bufs[3][0], len(dst),
                                                       bufs[4][0], bufs[5][0]))
        return bytes(ok)

    # -- BLS12-381 pairings ---------------------------------------------------------------------------
    def bls12381_pair(self, g1: bytes, g2: bytes) -> bytes:
        n = len(g1) // 96
        assert len(g1) == 96 * n and len(g2) == 192 * n
        return self.call_host("b2k_bls12381_pair", n, g1, g2, 576 * n)

    def bls12381_pair_fixed_g2(self, g1: bytes, g2: bytes) -> bytes:
        """gt[i] = e(g1[i], g2) for one g2 operand [192] (its Miller-loop lines shared by every element)"""
        n = len(g1) // 96
        assert len(g1) == 96 * n and len(g2) == 192
        return self.call_host("b2k_bls12381_pair_fixed_g2", n, g1, g2, 576 * n)

    # -- encrypt/ibe: Boneh-Franklin CCA ---------------------------------------------------------------
    def bls12381_ibe_decrypt(self, on: int, priv: bytes, u: bytes, v, w):
        """n x DecryptCCAonG1 (on = 1: priv [96] on G2, u [n][48]) / DecryptCCAonG2 (on = 2: priv [48] on G1, u [n][96]); v, w lists
        of n byte strings of one length <= 32 -> (list of n messages, status bytes [n] B2K_IBE_*: 0 OK, 1 PROOF, 2 POINT)"""
        assert on in (1, 2) and len(priv) == 144 - 48 * on
        n = len(v)
        ln = len(v[0]) if n else 0
        assert len(u) == 48 * on * n and len(w) == n and all(len(x) == ln for x in list(v) + list(w))
        msg, status = bytearray(max(n * ln, 1)), bytearray(max(n, 1))
        bufs = [_buf(x) for x in (priv, u or b"\x00", b"".join(v) or b"\x00", b"".join(w) or b"\x00", msg, status)]
        self._check(getattr(self.lib, f"b2k_bls12381_ibe_decrypt_cca_g{on}")(self.h, bufs[0][0], n, bufs[1][0], ln, bufs[2][0], bufs[3][0],
                                                                            bufs[4][0], bufs[5][0]))
        return [bytes(msg[ln * i:ln * (i + 1)]) for i in range(n)], bytes(status[:n])

    def bls12381_ibe_encrypt(self, on: int, master: bytes, ident: bytes, msgs, sigmas, dst: bytes = None):
        """n x EncryptCCAonG1 (on = 1: master [48] on G1, U [n][48]) / EncryptCCAonG2 (on = 2: master [96] on G2, U [n][96]) towards
        one identity; msgs, sigmas lists of n byte strings of one length <= 32; dst None = the default DST of the identity's hash
        -> (u bytes [n][48 on], list of n V, list of n W)"""
        assert on in (1, 2) and len(master) == 48 * on
        n = len(msgs)
        ln = len(msgs[0]) if n else 0
        assert len(sigmas) == n and all(len(x) == ln for x in list(msgs) + list(sigmas))
        u, v, w = bytearray(max(48 * on * n, 1)), bytearray(max(n * ln, 1)), bytearray(max(n * ln, 1))
        bufs = [_buf(x) for x in (master, ident or b"\x00", dst or b"\x00", b"".join(msgs) or b"\x00", b"".join(sigmas) or b"\x00",
                                  u, v, w)]
        self._check(getattr(self.lib, f"b2k_bls12381_ibe_encrypt_cca_g{on}")(
            self.h, bufs[0][0], bufs[1][0], len(ident), bufs[2][0] if dst is not None else None, len(dst) if dst is not None else 0,
            n, ln, bufs[3][0], bufs[4][0], bufs[5][0], bufs[6][0], bufs[7][0]))
        return bytes(u[:48 * on * n]), [bytes(v[ln * i:ln * (i + 1)]) for i in range(n)], [bytes(w[ln * i:ln * (i + 1)]) for i in range(n)]

    def bls12381_pairing_check(self, a1: bytes, a2: bytes, b1: bytes, b2: bytes) -> bytes:
        n = len(a1) // 96
        assert len(a1) == len(b1) == 96 * n and len(a2) == len(b2) == 192 * n
        out = bytearray(n)
        bufs = [_buf(x) for x in (a1, a2, b1, b2, out)]
        self._check(self.lib.b2k_bls12381_pairing_check(self.h, n, *[b[0] for b in bufs]))
        return bytes(out)

    # -- bn254 G1 ---------------------------------------------------------------------------------
    def bn254_g1_mul_batch(self, scalars: bytes, points: bytes) -> bytes:
        n = len(scalars) // 32
        assert len(scalars) == 32 * n and len(points) == 64 * n
        return self.call_host("b2k_bn254_g1_mul_batch", n, scalars, points, 64 * n)

    # -- bn256 (G1 64 B, G2 128 B operands and results) ------------------------------------------------------
    def bn256_call(self, name: str, scalars: bytes, points: bytes, point_len: int, out_len: int) -> bytes:
        n = len(scalars) // 32
        assert len(scalars) == 32 * n and len(points) == point_len * n
        return self.call_host(name, n, scalars, points, out_len)

    def bn256_g1_mul_batch(self, s, p): return self.bn256_call("b2k_bn256_g1_mul_batch", s, p, 64, 64 * (len(s) // 32))
    def bn256_g1_msm(self, s, p): return self.bn256_call("b2k_bn256_g1_msm", s, p, 64, 64)
    def bn256_g2_mul_batch(self, s, p): return self.bn256_call("b2k_bn256_g2_mul_batch", s, p, 128, 128 * (len(s) // 32))
    def bn256_g2_msm(self, s, p): return self.bn256_call("b2k_bn256_g2_msm", s, p, 128, 128)

    def bn256_pair(self, g1: bytes, g2: bytes) -> bytes:
        n = len(g1) // 64
        return self.call_host("b2k_bn256_pair", n, g1, g2, 384 * n)

    def bn256_pairing_check(self, a1: bytes, a2: bytes, b1: bytes, b2: bytes) -> bytes:
        n = len(a1) // 64
        out = bytearray(n)
        bufs = [_buf(x) for x in (a1, a2, b1, b2, out)]
        self._check(self.lib.b2k_bn256_pairing_check(self.h, n, *[b[0] for b in bufs]))
        return bytes(out)

    # -- target group, Miller / Finalize, products of pairings, point additions (b2k_gt.cu) --------------------------------------
    GT_BYTES = {"bls12381": 576, "bn254": 384, "bn256": 384}
    G1_BYTES = {"bls12381": 96, "bn254": 64, "bn256": 64}
    G2_BYTES = {"bls12381": 192, "bn254": 128, "bn256": 128}

    def _call_bufs(self, name: str, n: int, ins, out_len: int, extra=()) -> bytes:
        out = bytearray(out_len)
        keep = [_buf(b) for b in ins]
        po, ko = _buf(out)
        self._check(getattr(self.lib, name)(self.h, n, *[k[0] for k in keep], *extra, po))
        return bytes(out)

    def gt_mul(self, curve: str, a: bytes, b: bytes) -> bytes:
        n = len(a) // self.GT_BYTES[curve]
        return self._call_bufs(f"b2k_{curve}_gt_mul", n, (a, b), len(a))

    def gt_inv(self, curve: str, a: bytes) -> bytes:
        n = len(a) // self.GT_BYTES[curve]
        return self._call_bufs(f"b2k_{curve}_gt_inv", n, (a,), len(a))

    def gt_exp(self, curve: str, scalars: bytes, a: bytes) -> bytes:
        n = len(a) // self.GT_BYTES[curve]
        return self._call_bufs(f"b2k_{curve}_gt_exp", n, (scalars, a), len(a))

    def miller(self, curve: str, g1: bytes, g2: bytes) -> bytes:
        n = len(g1) // self.G1_BYTES[curve]
        return self._call_bufs(f"b2k_{curve}_miller", n, (g1, g2), n * self.GT_BYTES[curve])

    def final_exp(self, curve: str, f: bytes) -> bytes:
        n = len(f) // self.GT_BYTES[curve]
        return self._call_bufs("b2k_bls12381_final_exp" if curve == "bls12381" else f"b2k_{curve}_finalize", n, (f,), len(f))

    def pairing_product_check(self, curve: str, g1: bytes, g2: bytes) -> bool:
        n = len(g1) // self.G1_BYTES[curve]
        return self._call_bufs(f"b2k_{curve}_pairing_product_check", n, (g1, g2), 1) == b"\x01"

    def bls12381_pairing_product(self, g1: bytes, g2: bytes) -> bytes:
        return self._call_bufs("b2k_bls12381_pairing_product", len(g1) // 96, (g1, g2), 576)

    def bls12381_add_batch(self, group: int, a: bytes, b: bytes, negate_b: bool = False) -> bytes:
        pb = 96 if group == 1 else 192
        out = bytearray(len(a))
        pa, k1 = _buf(a); pbb, k2 = _buf(b); po, k3 = _buf(out)
        self._check(getattr(self.lib, f"b2k_bls12381_g{group}_add_batch")(self.h, len(a) // pb, pa, pbb, 1 if negate_b else 0, po))
        return bytes(out)

    @staticmethod
    def bdn_coefficients(pubs: bytes, pub_len: int, add_one: bool = False) -> bytes:
        """sign/bdn hashPointToR (bdn.go:29-63) over the marshalled public keys -> n x 32-byte big-endian c_i (+1).
        Host function of the library (no device work); static: needs no context."""
        lib = load_library()
        n = len(pubs) // pub_len
        assert len(pubs) == n * pub_len
        out = C.create_string_buffer(32 * n)
        lib.b2k_bdn_coefficients.restype = C.c_int
        lib.b2k_bdn_coefficients.argtypes = [C.c_size_t, C.c_char_p, C.c_size_t, C.c_int, C.c_char_p]
        rc = lib.b2k_bdn_coefficients(n, pubs, pub_len, 1 if add_one else 0, out)
        if rc != 0:
            raise ValueError("b2k_bdn_coefficients: rc=%d" % rc)
        return out.raw

    def ed25519_mul_batch(self, scalars_le: bytes, points: bytes) -> bytes:
        """n x edwards25519 Point.Mul: raw little-endian 32-byte scalars, 32-byte compressed points -> 32 B each"""
        n = len(scalars_le) // 32
        assert len(scalars_le) == 32 * n and len(points) == 32 * n
        return self.call_host("b2k_ed25519_mul_batch", n, scalars_le, points, 32 * n)

    def ed25519_msm(self, scalars_le: bytes, points: bytes) -> bytes:
        """sum_i k_i P_i on edwards25519: little-endian 32-byte scalars read as Point.Mul reads them, 32-byte compressed
        points -> the 32-byte encoding of the sum"""
        n = len(scalars_le) // 32
        assert len(scalars_le) == 32 * n and len(points) == 32 * n
        return self.call_host("b2k_ed25519_msm", n, scalars_le, points, 32)

    def ed25519_msm_dev(self, n: int, d_scalars: int, d_points: int, d_out: int):
        """the same on device pointers ([n][32], [n][32], [32]); enqueue only, data errors at wait()"""
        self.call_dev("b2k_ed25519_msm_dev", n, d_scalars, d_points, d_out)

    def ed25519_recover_commit(self, indices, points: bytes) -> bytes:
        """share.RecoverCommit over edwards25519: share indices I_i (x_i = I_i + 1), points [t][32] -> 32 B"""
        import struct
        t = len(indices)
        assert len(points) == 32 * t
        return self.call_host("b2k_ed25519_recover_commit", t, struct.pack("<%dI" % t, *indices), points, 32)

    def ed25519_pubpoly_eval(self, commits: bytes, indices) -> bytes:
        """PubPoly.Eval for every index: sum_j (I+1)^j C_j; commits [t][32] -> [n][32]"""
        import struct
        t, n = len(commits) // 32, len(indices)
        out = bytearray(32 * n)
        bufs = [_buf(x) for x in (commits, struct.pack("<%dI" % n, *indices), out)]
        self._check(self.lib.b2k_ed25519_pubpoly_eval(self.h, t, bufs[0][0], n, bufs[1][0], bufs[2][0]))
        return bytes(out)

    def ed25519_pubpoly_check(self, commits: bytes, t: int, indices, shares_le: bytes) -> bytes:
        """PubPoly.Check for m dealers x n shares: commits [m][t][32], indices m rows of n, shares [m][n][32] little-endian
        -> m*n bytes (1 = the share matches the dealer's commitments)"""
        import struct
        m = len(commits) // (32 * t)
        flat = [i for row in indices for i in row]
        n = len(flat) // m
        assert len(commits) == m * t * 32 and len(flat) == m * n and len(shares_le) == 32 * m * n
        out = bytearray(m * n)
        bufs = [_buf(x) for x in (commits, struct.pack("<%dI" % (m * n), *flat), shares_le, out)]
        self._check(self.lib.b2k_ed25519_pubpoly_check(self.h, m, t, bufs[0][0], n, bufs[1][0], bufs[2][0], bufs[3][0]))
        return bytes(out)

    def ed25519_verify(self, pks: bytes, msgs, sigs: bytes) -> bytes:
        """n x eddsa.VerifyWithChecks: pks [n][32], msgs list of bytes, sigs [n][64] R || s -> one status byte each
        (0 = valid, else the first failing check, B2K_ED_* of include/b2kyber.h)"""
        n = len(msgs)
        assert len(pks) == 32 * n and len(sigs) == 64 * n
        blob, offs = self._pack_msgs(msgs)
        status = bytearray(n)
        bufs = [_buf(x) for x in (pks, blob, offs, sigs, status)]
        self._check(self.lib.b2k_ed25519_verify(self.h, n, *[b[0] for b in bufs]))
        return bytes(status)

    def ed25519_verify_dev(self, n: int, d_pks: int, d_msgs: int, d_offsets: int, d_sigs: int, d_status: int):
        """the same on device pointers ([n][32], message bytes, [n+1] uint32 offsets, [n][64], [n] status); enqueue only"""
        self._check(self.lib.b2k_ed25519_verify_dev(self.h, n, C.c_void_p(d_pks), C.c_void_p(d_msgs), C.c_void_p(d_offsets),
                                                    C.c_void_p(d_sigs), C.c_void_p(d_status)))

    def _status_call(self, name: str, n: int, sizes, ins, out_len: int) -> bytes:
        status = bytearray(out_len)
        bufs = [_buf(x) for x in (*ins, status)]
        self._check(getattr(self.lib, name)(self.h, *sizes, *[b[0] for b in bufs]))
        return bytes(status)

    def ed25519_dleq_verify(self, g: bytes, h: bytes, xg: bytes, xh: bytes, proofs: bytes) -> bytes:
        """n x dleq.Proof.Verify(G, H, xG, xH): points [n][32], proofs [n][128] C || R || VG || VH -> one status byte each
        (B2K_DLEQ_*: 0 OK, 2 INVALID, 3 POINT)"""
        n = len(g) // 32
        assert len(g) == len(h) == len(xg) == len(xh) == 32 * n and len(proofs) == 128 * n
        return self._status_call("b2k_ed25519_dleq_verify", n, (n,), (g, h, xg, xh, proofs), n)

    def ed25519_dleq_verify_dev(self, n: int, d_g: int, d_h: int, d_xg: int, d_xh: int, d_proofs: int, d_status: int):
        """the same on device pointers; enqueue only"""
        self._check(self.lib.b2k_ed25519_dleq_verify_dev(self.h, n, *[C.c_void_p(p) for p in (d_g, d_h, d_xg, d_xh, d_proofs, d_status)]))

    def ed25519_pvss_verify_enc_shares(self, h: bytes, commits: bytes, t: int, x: bytes, sh: bytes, v: bytes, proofs: bytes) -> bytes:
        """pvss.VerifyEncShareBatch for m deals: h [m][32], commits [m][t][32], x, sh, v [m][n][32], proofs [m][n][128]
        -> m*n status bytes (B2K_DLEQ_*)"""
        m = len(h) // 32
        n = len(x) // (32 * m)
        assert len(h) == 32 * m and len(commits) == 32 * m * t
        assert len(x) == len(sh) == len(v) == 32 * m * n and len(proofs) == 128 * m * n
        return self._status_call("b2k_ed25519_pvss_verify_enc_shares", m * n, (m, t, n), (h, commits, x, sh, v, proofs), m * n)

    def ed25519_pvss_verify_dec_shares(self, g: bytes, x: bytes, enc_v: bytes, dec_v: bytes, proofs: bytes) -> bytes:
        """pvss.VerifyDecShareBatch: g [32], x, enc_v, dec_v [n][32], proofs [n][128] -> n status bytes (B2K_DLEQ_*)"""
        n = len(x) // 32
        assert len(g) == 32 and len(x) == len(enc_v) == len(dec_v) == 32 * n and len(proofs) == 128 * n
        return self._status_call("b2k_ed25519_pvss_verify_dec_shares", n, (n,), (g, x, enc_v, dec_v, proofs), n)

    def ed25519_pvss_recover_secret(self, g: bytes, indices, x: bytes, enc_v: bytes, dec_v: bytes, proofs: bytes, t: int):
        """pvss.RecoverSecret (pvss.go:303-323): VerifyDecShareBatch, then RecoverCommit over the valid shares (sorted by index,
        the first t, as xyCommit selects them) -> the 32-byte secret commitment, or None below t valid shares (ErrTooFewShares)"""
        status = self.ed25519_pvss_verify_dec_shares(g, x, enc_v, dec_v, proofs)
        good = sorted((indices[i], i) for i in range(len(status)) if status[i] == 0)[:t]
        if len(good) < t or t == 0:
            return None
        return self.ed25519_recover_commit([idx for idx, _ in good], b"".join(dec_v[32 * i:32 * i + 32] for _, i in good))

    def ed25519_shuffle_verify(self, k: int, x: bytes, y: bytes, xbar: bytes, ybar: bytes, proofs: bytes,
                               proto: bytes = b"", g: bytes = None, h: bytes = None) -> bytes:
        """m x proof.HashVerify(suite, proto, shuffle.Verifier(suite, G, H, X, Y, Xbar, Ybar), proof): x, y, xbar, ybar
        [m][k][32], proofs [m][32 (12k + 3)], g / h None (the base point) or [m][32] -> m status bytes (B2K_SHUFFLE_*: 0 OK,
        1 SIMPLE, 2 PAIR, 3 POINT)"""
        m = len(x) // (32 * k)
        assert m > 0 and len(x) == len(y) == len(xbar) == len(ybar) == 32 * m * k and len(proofs) == 32 * (12 * k + 3) * m
        assert (g is None or len(g) == 32 * m) and (h is None or len(h) == 32 * m)
        status = bytearray(m)
        bufs = [_buf(b) if b is not None else (None, None) for b in (g, h, x, y, xbar, ybar, proofs, bytes(proto), status)]
        self._check(self.lib.b2k_ed25519_shuffle_verify(self.h, m, k, *[b[0] for b in bufs[:8]], len(proto), bufs[8][0]))
        return bytes(status)

    def ed25519_shuffle_sequence_verifiable(self, nq: int, x: bytes, y: bytes, xbar: bytes, ybar: bytes, e: bytes):
        """shuffle.GetSequenceVerifiable: x, y, xbar, ybar [nq][k][32], e [nq][32] little-endian (raw) -> (xUp, yUp, xDown,
        yDown), each [k][32] canonical encodings"""
        k = len(x) // (32 * nq)
        assert k > 0 and len(x) == len(y) == len(xbar) == len(ybar) == 32 * nq * k and len(e) == 32 * nq
        outs = [bytearray(32 * k) for _ in range(4)]
        bufs = [_buf(b) for b in (x, y, xbar, ybar, e, *outs)]
        self._check(self.lib.b2k_ed25519_shuffle_sequence_verifiable(self.h, nq, k, *[b[0] for b in bufs]))
        return tuple(bytes(o) for o in outs)

    def ed25519_anon_verify(self, ring: bytes, msgs, sigs, scope: bytes = None):
        """m x anon.Verify(suite, msgs[j], ring, scope, sigs[j]) over one ring [n][32]: scope None = unlinkable, b"" = linkable
        with an empty scope; sigs: list of m signatures of exactly 32 (n + 1 + linkable) bytes -> (m status bytes (B2K_ANON_*:
        0 OK, 1 INVALID, 2 POINT), [m][32] tags: the canonical Tag of every OK linkable signature, zero otherwise)"""
        n, m, linkable = len(ring) // 32, len(msgs), scope is not None
        siglen = 32 * (n + 1 + linkable)
        assert len(ring) == 32 * n and len(sigs) == m and all(len(s) == siglen for s in sigs)
        blob, offs = self._pack_msgs(msgs)
        status, tags = bytearray(m), bytearray(32 * m)
        sc = bytes(scope or b"")
        bufs = [_buf(x) if len(x) else (None, None) for x in (bytes(ring), sc, blob, offs, b"".join(sigs) or b"\x00", status, tags)]
        self._check(self.lib.b2k_ed25519_anon_verify(self.h, n, bufs[0][0], int(linkable), bufs[1][0], len(sc), m,
                                                     *[b[0] for b in bufs[2:]]))
        return bytes(status), bytes(tags)

    # -- encrypt/ecies on edwards25519 (SHA-256) --------------------------------------------------------
    def ed25519_ecies_decrypt(self, priv: bytes, ctxts, length: int):
        """n x ecies.Decrypt(edwards25519, priv, ctxts[i], sha256.New); every ciphertext is 32 + length bytes (length =
        body + tag, >= 16) -> ([n] messages of length - 16 bytes, zero unless OK; n status bytes (B2K_ECIES_*: 0 OK, 1 POINT,
        2 AUTH))"""
        n = len(ctxts)
        assert len(priv) == 32 and all(len(c) == 32 + length for c in ctxts)
        msg, status = bytearray(max(n * (length - 16), 1)), bytearray(n)
        bufs = [_buf(x) for x in (bytes(priv), b"".join(ctxts) or b"\x00", msg, status)]
        self._check(self.lib.b2k_ed25519_ecies_decrypt(self.h, bufs[0][0], n, length, *[b[0] for b in bufs[1:]]))
        w = length - 16
        return [bytes(msg[w * i:w * i + w]) for i in range(n)], bytes(status)

    def ed25519_ecies_encrypt(self, pubs, rs, msgs):
        """n x ecies.Encrypt(edwards25519, pubs[i], msgs[i], sha256.New) with the ephemeral scalars rs[i] (32 bytes LE); all
        messages of one length -> ([n] ciphertexts R || C || tag, zero unless OK; n status bytes (0 OK, 1 POINT))"""
        n = len(msgs)
        length = len(msgs[0]) if n else 0
        assert len(pubs) == n and len(rs) == n and all(len(m) == length for m in msgs)
        out, status = bytearray(max(n * (length + 48), 1)), bytearray(n)
        bufs = [_buf(x) for x in (b"".join(pubs) or b"\x00", b"".join(rs) or b"\x00", b"".join(msgs) or b"\x00", out, status)]
        self._check(self.lib.b2k_ed25519_ecies_encrypt(self.h, n, bufs[0][0], bufs[1][0], length, *[b[0] for b in bufs[2:]]))
        w = length + 48
        return [bytes(out[w * i:w * i + w]) for i in range(n)], bytes(status)

    def bn254_pair(self, g1: bytes, g2: bytes) -> bytes:
        n = len(g1) // 64
        assert len(g1) == 64 * n and len(g2) == 128 * n
        return self.call_host("b2k_bn254_pair", n, g1, g2, 384 * n)

    def bn254_pairing_check(self, a1: bytes, a2: bytes, b1: bytes, b2: bytes) -> bytes:
        n = len(a1) // 64
        out = bytearray(n)
        bufs = [_buf(x) for x in (a1, a2, b1, b2, out)]
        self._check(self.lib.b2k_bn254_pairing_check(self.h, n, *[b[0] for b in bufs]))
        return bytes(out)

    def bn254_g2_mul_batch(self, s, p): return self.call_host("b2k_bn254_g2_mul_batch", len(s) // 32, s, p, 128 * (len(s) // 32))
    def bn254_g2_msm(self, s, p): return self.call_host("b2k_bn254_g2_msm", len(s) // 32, s, p, 128)

    def recover_pubpoly(self, name: str, indices, points: bytes) -> bytes:
        """share.RecoverPubPoly: name in bls12381_g1 / bls12381_g2 / bn254; returns t commitments in operand form"""
        import struct
        t = len(indices)
        return self.call_host(f"b2k_{name}_recover_pubpoly", t, struct.pack("<%dI" % t, *indices), points, len(points))

    def commit_batch(self, name: str, scalars: bytes, base: bytes = None) -> bytes:
        """PriPoly.Commit: out[i] = scalars[i] * base (None = generator), operand form"""
        n = len(scalars) // 32
        pb = {"bls12381_g1": 96, "bls12381_g2": 192, "bn254": 64}[name]
        out = bytearray(n * pb)
        ps, k1 = _buf(scalars); po, k3 = _buf(out)
        pbase, k2 = _buf(base) if base else (None, None)
        self._check(getattr(self.lib, f"b2k_{name}_commit_batch")(self.h, n, ps, pbase, po))
        return bytes(out)

    def bn254_recover_commit(self, indices, points: bytes) -> bytes:
        """share.RecoverCommit over bn254 G1: indices = share indices I_i (x_i = I_i + 1), points [t][64] -> 64 B"""
        import struct
        t = len(indices)
        assert len(points) == 64 * t
        return self.call_host("b2k_bn254_recover_commit", t, struct.pack("<%dI" % t, *indices), points, 64)

    def bls12381_recover_commit(self, group: int, indices, points: bytes) -> bytes:
        """share.RecoverCommit over BLS12-381 G1 (group=1, points [t][96] -> 48 B) or G2 (group=2, [t][192] -> 96 B)"""
        import struct
        t = len(indices)
        plen, olen = (96, 48) if group == 1 else (192, 96)
        assert len(points) == plen * t
        return self.call_host(f"b2k_bls12381_g{group}_recover_commit", t, struct.pack("<%dI" % t, *indices), points, olen)

    def bls12381_pubpoly_eval(self, group: int, commits: bytes, indices) -> bytes:
        """PubPoly.Eval for every index: sum_j (I+1)^j C_j; commits [t][96|192] operand form -> [n][96|192]"""
        import struct
        plen = 96 if group == 1 else 192
        t, n = len(commits) // plen, len(indices)
        out = bytearray(plen * n)
        bufs = [_buf(x) for x in (commits, struct.pack("<%dI" % n, *indices), out)]
        self._check(getattr(self.lib, f"b2k_bls12381_g{group}_pubpoly_eval")(self.h, t, bufs[0][0], n, bufs[1][0], bufs[2][0]))
        return bytes(out)

    def bn_unmarshal_check(self, curve: str, group: int, data: bytes) -> bytes:
        """UnmarshalBinary validation of a batch: curve in {"bn254", "bn256"}, group 1 ([n][64]) or 2 ([n][128]) -> n bytes"""
        plen = 64 if group == 1 else 128
        n = len(data) // plen
        assert n * plen == len(data)
        out = bytearray(n)
        bufs = [_buf(x) for x in (data, out)]
        self._check(getattr(self.lib, f"b2k_{curve}_g{group}_unmarshal_check")(self.h, n, bufs[0][0], bufs[1][0]))
        return bytes(out)

    def pubpoly_check(self, curve: str, commits: bytes, t: int, indices, shares: bytes) -> bytes:
        """PubPoly.Check for m dealers x n shares (share/poly.go:405-409, the DKG/VSS verification loops): curve in
        {"bls12381_g1", "bls12381_g2", "bn254"}; commits [m][t][96|192|64], indices m rows of n, shares [m][n][32] BE
        -> m*n bytes (1 = the share matches the dealer's commitments)"""
        import struct
        plen = {"bls12381_g1": 96, "bls12381_g2": 192, "bn254": 64}[curve]
        m = len(commits) // (plen * t)
        flat = [i for row in indices for i in row]
        n = len(flat) // m
        assert len(commits) == m * t * plen and len(flat) == m * n and len(shares) == 32 * m * n
        out = bytearray(m * n)
        bufs = [_buf(x) for x in (commits, struct.pack("<%dI" % (m * n), *flat), shares, out)]
        self._check(getattr(self.lib, f"b2k_{curve}_pubpoly_check")(self.h, m, t, bufs[0][0], n, bufs[1][0], bufs[2][0], bufs[3][0]))
        return bytes(out)

    def bn254_g1_msm(self, scalars: bytes, points: bytes) -> bytes:
        n = len(scalars) // 32
        assert len(scalars) == 32 * n and len(points) == 64 * n
        return self.call_host("b2k_bn254_g1_msm", n, scalars, points, 64)


class Comm:
    """One rank of the sharded MSM (include/b2kyber.h: b2k_comm_*): owns the rank's exchange slab on the engine's device.

    Wiring, one process per GPU:   c = Comm(eng, world, rank); blobs = all_gather(c.export()); c.connect(b"".join(blobs))
    one process, several engines:  comms = [Comm(e, n, r) ...]; Comm.connect_local(comms)
    """

    def __init__(self, eng: Engine, nranks: int, rank: int):
        self.eng, self.nranks, self.rank = eng, nranks, rank
        h = C.c_void_p()
        eng._check(eng.lib.b2k_comm_create(eng.h, nranks, rank, C.byref(h)))
        self.h = h

    def export(self) -> bytes:
        buf = C.create_string_buffer(COMM_BLOB_BYTES)
        self.eng._check(self.eng.lib.b2k_comm_export(self.h, C.cast(buf, C.c_void_p)))
        return buf.raw

    def connect(self, blobs: bytes):
        assert len(blobs) == self.nranks * COMM_BLOB_BYTES
        p, keep = _buf(blobs)
        self.eng._check(self.eng.lib.b2k_comm_connect(self.h, p))

    @staticmethod
    def connect_local(comms):
        arr = (C.c_void_p * len(comms))(*[c.h for c in comms])
        comms[0].eng._check(comms[0].eng.lib.b2k_comm_connect_local(arr, len(comms)))

    def use_nccl(self, unique_id: bytes):
        p, keep = _buf(unique_id)
        self.eng._check(self.eng.lib.b2k_comm_use_nccl(self.h, p))

    @staticmethod
    def nccl_unique_id(lib=None) -> bytes:
        lib = lib or load_library()
        buf = C.create_string_buffer(128)
        if lib.b2k_nccl_unique_id(C.cast(buf, C.c_void_p)) != 0:
            raise B2KError(-1, "b2k_nccl_unique_id failed (libnccl.so.2 not loadable)")
        return buf.raw

    def last_plan(self):
        a = (C.c_int * 4)()
        self.eng._check(self.eng.lib.b2k_comm_last_plan(self.h, a))
        return {"c": a[0], "W": a[1], "buckets_per_window": a[2], "bucket_bytes": a[3]}

    def msm_sharded_dev(self, n: int, d_scalars: int, d_points: int, d_out: int, shape: int = 0):
        """this rank's n resident pairs -> 48-byte sum over all ranks at d_out (enqueue only)"""
        self.eng._check(self.eng.lib.b2k_bls12381_g1_msm_sharded_dev(self.h, n, C.c_void_p(d_scalars), C.c_void_p(d_points),
                                                                   C.c_void_p(d_out), shape))

    def msm_sharded_async(self, n: int, h_scalars: int, h_points: int, h_out: int):
        """host pointers (page-locked); collect with eng.wait()"""
        self.eng._check(self.eng.lib.b2k_bls12381_g1_msm_sharded_async(self.h, n, C.c_void_p(h_scalars), C.c_void_p(h_points),
                                                                     C.c_void_p(h_out)))

    @staticmethod
    def msm_multi_gpu(comms, scalars: bytes, points: bytes) -> bytes:
        """one process, len(comms) GPUs: the whole sharded MSM from host buffers (b2k_bls12381_g1_msm_multi_gpu)"""
        n = len(scalars) // 32
        arr = (C.c_void_p * len(comms))(*[c.h for c in comms])
        ps, k1 = _buf(scalars)
        pp, k2 = _buf(points)
        out = C.create_string_buffer(48)
        rc = comms[0].eng.lib.b2k_bls12381_g1_msm_multi_gpu(arr, len(comms), n, ps, pp, C.cast(out, C.c_void_p))
        for c in comms:
            if rc == 0:
                break
            c.eng._check(rc)
        return out.raw

    def close(self):
        if getattr(self, "h", None):
            self.eng.lib.b2k_comm_destroy(self.h)
            self.h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass
