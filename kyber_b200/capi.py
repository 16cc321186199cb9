"""ctypes binding of include/b2kyber.h -- the same C ABI a Go adapter binds with cgo.

Every signature is read from the header, so the binding cannot drift from it.  There is no CPU fallback: importing this
without the built library, or creating an Engine without an sm_90 device, raises.
"""
from __future__ import annotations
import ctypes as C
import functools
import os
import re
import struct

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_HERE, "libb2kyber.so")
HEADER_PATH = os.path.join(os.path.dirname(_HERE), "include", "b2kyber.h")

B2K_OK, ERR_CUDA, ERR_ARG, ERR_SCALAR_RANGE, ERR_NO_DEVICE, ERR_POINT, ERR_COMM = 0, -1, -2, -3, -4, -5, -6
COMM_BLOB_BYTES, MAX_RANKS = 128, 16

_VALUE_TYPES = {"int": C.c_int, "size_t": C.c_size_t, "uint32_t": C.c_uint32, "uint64_t": C.c_uint64}
_RESULT_TYPES = {**_VALUE_TYPES, "void": None, "const char *": C.c_char_p}


class B2KError(RuntimeError):
    def __init__(self, code: int, msg: str):
        super().__init__(f"b2kyber error {code}: {msg}")
        self.code = code


def header_signatures(path: str = HEADER_PATH) -> dict:
    """{name: (restype, argtypes)} of every b2k_* prototype in the C header.  Every pointer parameter is a c_void_p (it takes
    bytes, ctypes arrays, byref(...), int addresses and None); a const char* result is a c_char_p (bytes).  Any other type
    raises, so that a new header type cannot bind silently wrong."""
    with open(path) as f:
        src = re.sub(r"/\*.*?\*/|//[^\n]*", " ", f.read(), flags=re.S)
    sigs = {}
    for ret, name, params in re.findall(r"([A-Za-z_][\w \t*]*?)\s*\b(b2k_\w+)\s*\(([^()]*)\)\s*;", src):
        ret = " ".join(ret.replace("*", " * ").split())
        if ret not in _RESULT_TYPES:
            raise ValueError(f"{name}: no ctypes mapping for the result type {ret!r}")
        args = []
        for p in [] if params.strip() in ("", "void") else params.split(","):
            m = re.fullmatch(r"(?:const\s+)?(\w+)\s+\w+", p.strip())
            if "*" in p:
                args.append(C.c_void_p)
            elif m and m.group(1) in _VALUE_TYPES:
                args.append(_VALUE_TYPES[m.group(1)])
            else:
                raise ValueError(f"{name}: no ctypes mapping for the parameter {p.strip()!r}")
        sigs[name] = (_RESULT_TYPES[ret], args)
    return sigs


@functools.cache
def load_library() -> C.CDLL:
    """the library with every signature of the header bound, loaded once per process"""
    if not os.path.exists(LIB_PATH):
        raise ImportError(f"{LIB_PATH} is missing: build it with `python -m kyber_b200.build` "
                          "(there is no CPU fallback)")
    lib = C.CDLL(LIB_PATH)
    for name, (res, args) in header_signatures().items():
        fn = getattr(lib, name)      # AttributeError here = ABI drift between header and library
        fn.restype, fn.argtypes = res, args
    return lib


def _buf(b):
    """argument -> (what a pointer parameter takes, keepalive): a bytearray or memoryview becomes a ctypes array over its
    memory; bytes, ints, None and ctypes objects pass unchanged"""
    if isinstance(b, (bytearray, memoryview)):
        arr = (C.c_char * memoryview(b).nbytes).from_buffer(b)
        return arr, arr
    return b, None


def _u32(xs) -> bytes:
    return struct.pack("<%dI" % len(xs), *xs)


class Engine:
    """One b2k context (one CUDA stream + scratch arena) on one device."""

    GT_BYTES = {"bls12381": 576, "bn254": 384, "bn256": 384}
    G1_BYTES = {"bls12381": 96, "bn254": 64, "bn256": 64}
    G2_BYTES = {"bls12381": 192, "bn254": 128, "bn256": 128}
    # (operand, result) bytes of a point, by the prefix of the group's entry points; bn254's share calls are on G1 and omit "_g1"
    POINT_BYTES = {"bls12381_g1": (96, 48), "bls12381_g2": (192, 96), "bn254_g1": (64, 64), "bn254": (64, 64),
                   "bn254_g2": (128, 128), "bn256_g1": (64, 64), "bn256_g2": (128, 128), "ed25519": (32, 32)}

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

    def _call(self, name: str, *args, out: int | None = None, h=None):
        """lib.<name>(h, *args), raising B2KError on a non-zero status.  h is this context unless given (a communicator, or
        an array of them).  With `out`, a zeroed buffer of that many bytes goes last and its bytes are returned.  Arguments
        pass through _buf."""
        res = None if out is None else bytearray(out)
        ptrs = [_buf(a)[0] for a in (args if res is None else (*args, res))]
        self._check(getattr(self.lib, name)(self.h if h is None else h, *ptrs))
        return None if res is None else bytes(res)

    # -- generic calls ---------------------------------------------------------------------------
    def call_host(self, name: str, n: int, scalars, points, out_len: int) -> bytes:
        return self._call(name, n, scalars, points, out=out_len)

    def call_dev(self, name: str, n: int, d_scalars: int, d_points: int, d_out: int):
        self._call(name, n, d_scalars, d_points, d_out)

    def set_stream(self, cuda_stream: int):
        self._call("b2k_set_stream", cuda_stream)

    def wait(self):
        """synchronise and raise the deferred status (scalar range / malformed point) of everything enqueued since the last wait"""
        self._call("b2k_wait")

    def synchronize(self):
        self._call("b2k_synchronize")

    def set_msm_window(self, c: int):
        self._call("b2k_set_msm_window", c)

    def set_msm_slice(self, L: int):
        self._call("b2k_set_msm_slice", L)

    def set_msm_groups(self, groups: int):
        """window groups of the overlapped MSM tail; 1 = serial pipeline (per-stage timings meaningful)"""
        self._call("b2k_set_msm_groups", groups)

    def set_msm_variant(self, one_thread_per_bucket: bool):
        self._call("b2k_set_msm_variant", int(one_thread_per_bucket))

    def set_msm_glv(self, on: bool):
        """BLS12-381 G1 MSM: endomorphism split on (default) / off (plain 255-bit pipeline)"""
        self._call("b2k_set_msm_glv", int(on))

    def set_msm_affine(self, rounds: int = -1, batch: int = 0):
        """affine pair-tree rounds of the BLS12-381 G1 MSM: -1 automatic, 0 off, 1..8 forced; batch = additions per thread"""
        self._call("b2k_set_msm_affine", int(rounds), int(batch))

    def set_pairing_coop(self, max_n: int):
        """batches of at most max_n BLS12-381 pairings / checks run one per warp (coop_pairing.cuh); 0 = never"""
        self._call("b2k_set_pairing_coop", int(max_n))

    def set_msm_affine_split(self, split: bool):
        """affine rounds as three kernels each (True, default) or one fused kernel (False)"""
        self._call("b2k_set_msm_affine_split", int(split))

    def set_mul_occupancy(self, blocks_per_sm: int):
        self._call("b2k_set_mul_occupancy", int(blocks_per_sm))

    def set_msm_reduce(self, levels: int = 0, m1: int = 0, m2: int = 0):
        """bucket reduction in one or two levels (0 = automatic); A/B and tuning aid"""
        self._call("b2k_set_msm_reduce", int(levels), int(m1), int(m2))

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
        self._call("b2k_bls12381_g1_msm_bucket_plan", n, arr)
        return {"c": arr[0], "W": arr[1], "buckets_per_window": arr[2], "bucket_bytes": arr[3]}

    def bls12381_g1_msm_buckets_dev(self, n: int, d_scalars: int, d_points: int, d_buckets: int, cap_bytes: int):
        self._call("b2k_bls12381_g1_msm_buckets_dev", n, d_scalars, d_points, d_buckets, cap_bytes, None)

    def bls12381_g1_msm_reduce_windows_dev(self, c: int, w_cnt: int, parts: int, d_recv: int, d_wsum: int):
        self._call("b2k_bls12381_g1_msm_reduce_windows_dev", c, w_cnt, parts, d_recv, d_wsum)

    def bls12381_g1_msm_finish_dev(self, c: int, W: int, d_wsum: int, d_out: int, affine_out: bool = False):
        self._call("b2k_bls12381_g1_msm_finish_dev", c, W, d_wsum, d_out, 1 if affine_out else 0)

    # -- Point.Mul batches and MSMs of every group ----------------------------------------------------
    def _mul(self, group: str, op: str, scalars: bytes, points: bytes) -> bytes:
        """b2k_<group>_<op>: mul_batch (n results), mul_batch_affine (n operands) or msm (one result)"""
        operand, result = self.POINT_BYTES[group]
        n = len(scalars) // 32
        assert len(scalars) == 32 * n and len(points) == operand * n
        size = operand if op == "mul_batch_affine" else result
        return self.call_host(f"b2k_{group}_{op}", n, scalars, points, size if op == "msm" else size * n)

    def bls12381_g1_mul_batch(self, scalars: bytes, points: bytes) -> bytes:
        return self._mul("bls12381_g1", "mul_batch", scalars, points)

    def bls12381_g1_mul_batch_affine(self, scalars: bytes, points: bytes) -> bytes:
        return self._mul("bls12381_g1", "mul_batch_affine", scalars, points)

    def bls12381_g1_msm(self, scalars: bytes, points: bytes) -> bytes:
        return self._mul("bls12381_g1", "msm", scalars, points)

    def bls12381_g2_mul_batch(self, scalars: bytes, points: bytes) -> bytes:
        return self._mul("bls12381_g2", "mul_batch", scalars, points)

    def bls12381_g2_mul_batch_affine(self, scalars: bytes, points: bytes) -> bytes:
        return self._mul("bls12381_g2", "mul_batch_affine", scalars, points)

    def bls12381_g2_msm(self, scalars: bytes, points: bytes) -> bytes:
        return self._mul("bls12381_g2", "msm", scalars, points)

    def bn254_g1_mul_batch(self, scalars: bytes, points: bytes) -> bytes:
        return self._mul("bn254_g1", "mul_batch", scalars, points)

    def bn254_g1_msm(self, scalars: bytes, points: bytes) -> bytes:
        return self._mul("bn254_g1", "msm", scalars, points)

    def bn254_g2_mul_batch(self, s, p): return self._mul("bn254_g2", "mul_batch", s, p)
    def bn254_g2_msm(self, s, p): return self._mul("bn254_g2", "msm", s, p)
    def bn256_g1_mul_batch(self, s, p): return self._mul("bn256_g1", "mul_batch", s, p)
    def bn256_g1_msm(self, s, p): return self._mul("bn256_g1", "msm", s, p)
    def bn256_g2_mul_batch(self, s, p): return self._mul("bn256_g2", "mul_batch", s, p)
    def bn256_g2_msm(self, s, p): return self._mul("bn256_g2", "msm", s, p)

    def ed25519_mul_batch(self, scalars_le: bytes, points: bytes) -> bytes:
        """n x edwards25519 Point.Mul: raw little-endian 32-byte scalars, 32-byte compressed points -> 32 B each"""
        return self._mul("ed25519", "mul_batch", scalars_le, points)

    def ed25519_msm(self, scalars_le: bytes, points: bytes) -> bytes:
        """sum_i k_i P_i on edwards25519: little-endian 32-byte scalars read as Point.Mul reads them, 32-byte compressed
        points -> the 32-byte encoding of the sum"""
        return self._mul("ed25519", "msm", scalars_le, points)

    def ed25519_msm_dev(self, n: int, d_scalars: int, d_points: int, d_out: int):
        """the same on device pointers ([n][32], [n][32], [32]); enqueue only, data errors at wait()"""
        self.call_dev("b2k_ed25519_msm_dev", n, d_scalars, d_points, d_out)

    # -- UnmarshalBinary batches ------------------------------------------------------------------------
    def bls12381_g1_decompress(self, data: bytes):
        """-> (operand bytes [n][96], ok flags [n])"""
        n = len(data) // 48
        assert len(data) == 48 * n
        out = bytearray(96 * n)
        ok = self._call("b2k_bls12381_g1_decompress", n, data, out, out=n)
        return bytes(out), ok

    def bls12381_g2_decompress(self, data: bytes):
        n = len(data) // 96
        assert len(data) == 96 * n
        out = bytearray(192 * n)
        ok = self._call("b2k_bls12381_g2_decompress", n, data, out, out=n)
        return bytes(out), ok

    def bn_unmarshal_check(self, curve: str, group: int, data: bytes) -> bytes:
        """UnmarshalBinary validation of a batch: curve in {"bn254", "bn256"}, group 1 ([n][64]) or 2 ([n][128]) -> n bytes"""
        plen = self.POINT_BYTES[f"{curve}_g{group}"][0]
        n = len(data) // plen
        assert n * plen == len(data)
        return self._call(f"b2k_{curve}_g{group}_unmarshal_check", n, data, out=n)

    # -- hash-to-G1 / BLS verify -------------------------------------------------------------------------
    @staticmethod
    def _pack_msgs(msgs):
        offs = [0]
        for m in msgs:
            offs.append(offs[-1] + len(m))
        return b"".join(msgs), _u32(offs)

    def bls12381_hash_to_g1(self, msgs, dst: bytes) -> bytes:
        """msgs: list of bytes -> operand bytes [n][96]"""
        blob, offs = self._pack_msgs(msgs)
        return self._call("b2k_bls12381_hash_to_g1", len(msgs), blob, offs, dst, len(dst), out=96 * len(msgs))

    def bn254_hash_to_g1(self, msgs, dst: bytes = b"BN254G1_XMD:KECCAK-256_SVDW_RO_") -> bytes:
        """bn254 pointG1.Hash (Keccak-256 XMD + SvdW) for a list of messages -> [n][64] x||y"""
        blob, offs = self._pack_msgs(msgs)
        return self._call("b2k_bn254_hash_to_g1", len(msgs), blob, offs, dst, len(dst), out=64 * len(msgs))

    def bn256_hash_to_g1(self, msgs) -> bytes:
        """bn256 pointG1.Hash (SHA-256 try-and-increment) for a list of messages -> [n][64] x||y"""
        blob, offs = self._pack_msgs(msgs)
        return self._call("b2k_bn256_hash_to_g1", len(msgs), blob, offs, out=64 * len(msgs))

    def bn256_hash_g1(self, msgs, dst: bytes = b"") -> bytes:
        """bn256 HashG1 (HKDF-SHA256 + SvdW, pairing/bn256/hash.go:10-110) for a list of messages -> [n][64] x||y"""
        blob, offs = self._pack_msgs(msgs)
        return self._call("b2k_bn256_hash_g1", len(msgs), blob, offs, dst or None, len(dst), out=64 * len(msgs))

    def bls12381_hash_to_g2(self, msgs, dst: bytes) -> bytes:
        """msgs: list of bytes -> operand bytes [n][192]"""
        blob, offs = self._pack_msgs(msgs)
        return self._call("b2k_bls12381_hash_to_g2", len(msgs), blob, offs, dst, len(dst), out=192 * len(msgs))

    def bls12381_verify_g2sig(self, pks: bytes, msgs, dst: bytes, sigs: bytes) -> bytes:
        """n x bls.Verify (sigs on G2): pks [n][48] compressed G1, sigs [n][96] compressed G2 -> ok flags [n]"""
        n = len(msgs)
        assert len(pks) == 48 * n and len(sigs) == 96 * n
        blob, offs = self._pack_msgs(msgs)
        return self._call("b2k_bls12381_verify_g2sig", n, pks, blob, offs, dst, len(dst), sigs, out=n)

    def bls12381_verify_g1sig(self, pks: bytes, msgs, dst: bytes, sigs: bytes) -> bytes:
        """n x bls.Verify (sigs on G1): pks [n][96] compressed G2, sigs [n][48] compressed G1 -> ok flags [n]"""
        n = len(msgs)
        assert len(pks) == 96 * n and len(sigs) == 48 * n
        blob, offs = self._pack_msgs(msgs)
        return self._call("b2k_bls12381_verify_g1sig", n, pks, blob, offs, dst, len(dst), sigs, out=n)

    # -- pairings --------------------------------------------------------------------------------------
    def bls12381_pair(self, g1: bytes, g2: bytes) -> bytes:
        n = len(g1) // 96
        assert len(g1) == 96 * n and len(g2) == 192 * n
        return self.call_host("b2k_bls12381_pair", n, g1, g2, 576 * n)

    def bls12381_pair_fixed_g2(self, g1: bytes, g2: bytes) -> bytes:
        """gt[i] = e(g1[i], g2) for one g2 operand [192] (its Miller-loop lines shared by every element)"""
        n = len(g1) // 96
        assert len(g1) == 96 * n and len(g2) == 192
        return self.call_host("b2k_bls12381_pair_fixed_g2", n, g1, g2, 576 * n)

    def bls12381_pairing_check(self, a1: bytes, a2: bytes, b1: bytes, b2: bytes) -> bytes:
        n = len(a1) // 96
        assert len(a1) == len(b1) == 96 * n and len(a2) == len(b2) == 192 * n
        return self._call("b2k_bls12381_pairing_check", n, a1, a2, b1, b2, out=n)

    def bn254_pair(self, g1: bytes, g2: bytes) -> bytes:
        n = len(g1) // 64
        assert len(g1) == 64 * n and len(g2) == 128 * n
        return self.call_host("b2k_bn254_pair", n, g1, g2, 384 * n)

    def bn254_pairing_check(self, a1: bytes, a2: bytes, b1: bytes, b2: bytes) -> bytes:
        return self._call("b2k_bn254_pairing_check", len(a1) // 64, a1, a2, b1, b2, out=len(a1) // 64)

    def bn256_pair(self, g1: bytes, g2: bytes) -> bytes:
        n = len(g1) // 64
        return self.call_host("b2k_bn256_pair", n, g1, g2, 384 * n)

    def bn256_pairing_check(self, a1: bytes, a2: bytes, b1: bytes, b2: bytes) -> bytes:
        return self._call("b2k_bn256_pairing_check", len(a1) // 64, a1, a2, b1, b2, out=len(a1) // 64)

    # -- encrypt/ibe: Boneh-Franklin CCA ---------------------------------------------------------------
    def bls12381_ibe_decrypt(self, on: int, priv: bytes, u: bytes, v, w):
        """n x DecryptCCAonG1 (on = 1: priv [96] on G2, u [n][48]) / DecryptCCAonG2 (on = 2: priv [48] on G1, u [n][96]); v, w lists
        of n byte strings of one length <= 32 -> (list of n messages, status bytes [n] B2K_IBE_*: 0 OK, 1 PROOF, 2 POINT)"""
        assert on in (1, 2) and len(priv) == 144 - 48 * on
        n = len(v)
        ln = len(v[0]) if n else 0
        assert len(u) == 48 * on * n and len(w) == n and all(len(x) == ln for x in list(v) + list(w))
        msg, status = bytearray(max(n * ln, 1)), bytearray(max(n, 1))
        self._call(f"b2k_bls12381_ibe_decrypt_cca_g{on}", priv, n, u, ln, b"".join(v), b"".join(w), msg, status)
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
        self._call(f"b2k_bls12381_ibe_encrypt_cca_g{on}", master, ident, len(ident), dst, 0 if dst is None else len(dst), n, ln,
                   b"".join(msgs), b"".join(sigmas), u, v, w)
        return bytes(u[:48 * on * n]), [bytes(v[ln * i:ln * (i + 1)]) for i in range(n)], [bytes(w[ln * i:ln * (i + 1)]) for i in range(n)]

    # -- target group, Miller / Finalize, products of pairings, point additions (b2k_gt.cu) --------------------------------------
    def gt_mul(self, curve: str, a: bytes, b: bytes) -> bytes:
        return self._call(f"b2k_{curve}_gt_mul", len(a) // self.GT_BYTES[curve], a, b, out=len(a))

    def gt_inv(self, curve: str, a: bytes) -> bytes:
        return self._call(f"b2k_{curve}_gt_inv", len(a) // self.GT_BYTES[curve], a, out=len(a))

    def gt_exp(self, curve: str, scalars: bytes, a: bytes) -> bytes:
        return self._call(f"b2k_{curve}_gt_exp", len(a) // self.GT_BYTES[curve], scalars, a, out=len(a))

    def miller(self, curve: str, g1: bytes, g2: bytes) -> bytes:
        n = len(g1) // self.G1_BYTES[curve]
        return self._call(f"b2k_{curve}_miller", n, g1, g2, out=n * self.GT_BYTES[curve])

    def final_exp(self, curve: str, f: bytes) -> bytes:
        name = "b2k_bls12381_final_exp" if curve == "bls12381" else f"b2k_{curve}_finalize"
        return self._call(name, len(f) // self.GT_BYTES[curve], f, out=len(f))

    def pairing_product_check(self, curve: str, g1: bytes, g2: bytes) -> bool:
        return self._call(f"b2k_{curve}_pairing_product_check", len(g1) // self.G1_BYTES[curve], g1, g2, out=1) == b"\x01"

    def bls12381_pairing_product(self, g1: bytes, g2: bytes) -> bytes:
        return self._call("b2k_bls12381_pairing_product", len(g1) // 96, g1, g2, out=576)

    def bls12381_add_batch(self, group: int, a: bytes, b: bytes, negate_b: bool = False) -> bytes:
        n = len(a) // self.POINT_BYTES[f"bls12381_g{group}"][0]
        return self._call(f"b2k_bls12381_g{group}_add_batch", n, a, b, 1 if negate_b else 0, out=len(a))

    @staticmethod
    def bdn_coefficients(pubs: bytes, pub_len: int, add_one: bool = False) -> bytes:
        """sign/bdn hashPointToR (bdn.go:29-63) over the marshalled public keys -> n x 32-byte big-endian c_i (+1).
        Host function of the library (no device work); static: needs no context."""
        n = len(pubs) // pub_len
        assert len(pubs) == n * pub_len
        out = C.create_string_buffer(32 * n)
        rc = load_library().b2k_bdn_coefficients(n, pubs, pub_len, 1 if add_one else 0, out)
        if rc != 0:
            raise ValueError("b2k_bdn_coefficients: rc=%d" % rc)
        return out.raw

    # -- sign/bdn: a roster's terms once, then aggregate keys / verification for many masks ----------------------------------
    # key group -> the scheme whose signatures it verifies, that scheme's signature bytes and its default domain separation tag
    # (the signature group's, kilic/g1.go:17 and g2.go:18; bn256 hashes without one)
    BDN_SCHEMES = {"bls12381_g2": ("bls12381_bdn_verify_g1sig", 48, b"BLS_SIG_BLS12381G1_XMD:SHA-256_SSWU_RO_NUL_"),
                   "bls12381_g1": ("bls12381_bdn_verify_g2sig", 96, b"BLS_SIG_BLS12381G2_XMD:SHA-256_SSWU_RO_NUL_"),
                   "bn256_g2": ("bn256_bdn_verify_g1sig", 64, None)}

    def bdn_terms(self, group: str, pubs: bytes) -> bytes:
        """NewMask's terms (c_i + 1) PK_i of a roster: group in BDN_SCHEMES, pubs [n][MarshalBinary] -> [n][operand]"""
        operand, wire = self.POINT_BYTES[group]
        n = len(pubs) // wire
        assert len(pubs) == n * wire
        return self._call(f"b2k_{group}_bdn_terms", n, pubs, out=n * operand)

    def bdn_aggregate_keys(self, group: str, terms: bytes, masks) -> bytes:
        """AggregatePublicKeys for every mask (list of (n + 7) / 8 mask bytes) -> [m][operand]"""
        operand = self.POINT_BYTES[group][0]
        n = len(terms) // operand
        assert masks and all(len(k) == (n + 7) // 8 for k in masks)
        return self._call(f"b2k_{group}_bdn_aggregate_keys", n, terms, len(masks), b"".join(masks), out=len(masks) * operand)

    def bdn_aggregate_keys_dev(self, group: str, n: int, d_terms: int, m: int, d_masks: int, d_out: int):
        self._call(f"b2k_{group}_bdn_aggregate_keys_dev", n, d_terms, m, d_masks, d_out)

    def bdn_verify(self, group: str, terms: bytes, masks, msgs, sigs: bytes, dst: bytes = None) -> bytes:
        """bls.Verify under each mask's aggregate key -> statuses [m] (B2K_BDN_OK / _SIG / _INVALID).  dst: BLS12-381 only, the
        signature group's default when left out"""
        name, sig_bytes, default_dst = self.BDN_SCHEMES[group]
        n, m = len(terms) // self.POINT_BYTES[group][0], len(masks)
        assert len(msgs) == m and len(sigs) == sig_bytes * m and all(len(k) == (n + 7) // 8 for k in masks)
        blob, offs = self._pack_msgs(msgs)
        if group == "bn256_g2":
            if dst is not None:
                raise ValueError("bn256 hashes with try-and-increment: it takes no dst")
            return self._call(f"b2k_{name}", n, terms, m, b"".join(masks), blob, offs, sigs, out=m)
        dst = default_dst if dst is None else dst
        return self._call(f"b2k_{name}", n, terms, m, b"".join(masks), blob, offs, dst, len(dst), sigs, out=m)

    def bdn_verify_dev(self, group: str, n: int, d_terms: int, m: int, d_masks: int, d_msgs: int, d_offsets: int, d_dst: int,
                       dst_len: int, d_sigs: int, d_status: int):
        self._call(f"b2k_{self.BDN_SCHEMES[group][0]}_dev", n, d_terms, m, d_masks, d_msgs, d_offsets, d_dst, dst_len, d_sigs, d_status)

    # -- share/poly: RecoverCommit, RecoverPubPoly, PubPoly.Eval / Check, PriPoly.Commit ---------------------------------------
    def _recover_commit(self, group: str, indices, points: bytes) -> bytes:
        operand, result = self.POINT_BYTES[group]
        assert len(points) == operand * len(indices)
        return self.call_host(f"b2k_{group}_recover_commit", len(indices), _u32(indices), points, result)

    def ed25519_recover_commit(self, indices, points: bytes) -> bytes:
        """share.RecoverCommit over edwards25519: share indices I_i (x_i = I_i + 1), points [t][32] -> 32 B"""
        return self._recover_commit("ed25519", indices, points)

    def bn254_recover_commit(self, indices, points: bytes) -> bytes:
        """share.RecoverCommit over bn254 G1: indices = share indices I_i (x_i = I_i + 1), points [t][64] -> 64 B"""
        return self._recover_commit("bn254", indices, points)

    def bls12381_recover_commit(self, group: int, indices, points: bytes) -> bytes:
        """share.RecoverCommit over BLS12-381 G1 (group=1, points [t][96] -> 48 B) or G2 (group=2, [t][192] -> 96 B)"""
        return self._recover_commit(f"bls12381_g{group}", indices, points)

    def recover_pubpoly(self, name: str, indices, points: bytes) -> bytes:
        """share.RecoverPubPoly: name in bls12381_g1 / bls12381_g2 / bn254; returns t commitments in operand form"""
        return self.call_host(f"b2k_{name}_recover_pubpoly", len(indices), _u32(indices), points, len(points))

    def commit_batch(self, name: str, scalars: bytes, base: bytes = None) -> bytes:
        """PriPoly.Commit: out[i] = scalars[i] * base (None = generator), operand form"""
        n = len(scalars) // 32
        return self._call(f"b2k_{name}_commit_batch", n, scalars, base or None, out=n * self.POINT_BYTES[name][0])

    def _pubpoly_eval(self, group: str, commits: bytes, indices) -> bytes:
        plen = self.POINT_BYTES[group][0]
        n = len(indices)
        return self._call(f"b2k_{group}_pubpoly_eval", len(commits) // plen, commits, n, _u32(indices), out=plen * n)

    def ed25519_pubpoly_eval(self, commits: bytes, indices) -> bytes:
        """PubPoly.Eval for every index: sum_j (I+1)^j C_j; commits [t][32] -> [n][32]"""
        return self._pubpoly_eval("ed25519", commits, indices)

    def bls12381_pubpoly_eval(self, group: int, commits: bytes, indices) -> bytes:
        """PubPoly.Eval for every index: sum_j (I+1)^j C_j; commits [t][96|192] operand form -> [n][96|192]"""
        return self._pubpoly_eval(f"bls12381_g{group}", commits, indices)

    def pubpoly_check(self, curve: str, commits: bytes, t: int, indices, shares: bytes) -> bytes:
        """PubPoly.Check for m dealers x n shares (share/poly.go:405-409, the DKG/VSS verification loops): curve in
        {"bls12381_g1", "bls12381_g2", "bn254", "ed25519"}; commits [m][t][96|192|64|32], indices m rows of n, shares [m][n][32]
        (big-endian; little-endian on ed25519) -> m*n bytes (1 = the share matches the dealer's commitments)"""
        plen = self.POINT_BYTES[curve][0]
        m = len(commits) // (plen * t)
        flat = [i for row in indices for i in row]
        n = len(flat) // m
        assert len(commits) == m * t * plen and len(flat) == m * n and len(shares) == 32 * m * n
        return self._call(f"b2k_{curve}_pubpoly_check", m, t, commits, n, _u32(flat), shares, out=m * n)

    def ed25519_pubpoly_check(self, commits: bytes, t: int, indices, shares_le: bytes) -> bytes:
        """PubPoly.Check for m dealers x n shares: commits [m][t][32], indices m rows of n, shares [m][n][32] little-endian
        -> m*n bytes (1 = the share matches the dealer's commitments)"""
        return self.pubpoly_check("ed25519", commits, t, indices, shares_le)

    # -- edwards25519 protocols: EdDSA, DLEQ / PVSS, shuffle, ring signatures, ECIES ------------------------------------------
    def ed25519_verify(self, pks: bytes, msgs, sigs: bytes) -> bytes:
        """n x eddsa.VerifyWithChecks: pks [n][32], msgs list of bytes, sigs [n][64] R || s -> one status byte each
        (0 = valid, else the first failing check, B2K_ED_* of include/b2kyber.h)"""
        n = len(msgs)
        assert len(pks) == 32 * n and len(sigs) == 64 * n
        blob, offs = self._pack_msgs(msgs)
        return self._call("b2k_ed25519_verify", n, pks, blob, offs, sigs, out=n)

    def ed25519_verify_dev(self, n: int, d_pks: int, d_msgs: int, d_offsets: int, d_sigs: int, d_status: int):
        """the same on device pointers ([n][32], message bytes, [n+1] uint32 offsets, [n][64], [n] status); enqueue only"""
        self._call("b2k_ed25519_verify_dev", n, d_pks, d_msgs, d_offsets, d_sigs, d_status)

    SCHNORR_POINT_BYTES = {"bls12381_g1": 48, "bls12381_g2": 96}

    def schnorr_verify(self, group: str, pks: bytes, msgs, sigs: bytes) -> bytes:
        """n x schnorr.VerifyWithChecks over BLS12-381 keys on G1 or G2 (group "bls12381_g1" / "bls12381_g2"): pks [n][48 or 96],
        msgs list of bytes, sigs [n][80 or 128] R || s -> one status byte each (B2K_SCHNORR_* of include/b2kyber.h)"""
        pl = self.SCHNORR_POINT_BYTES[group]
        n = len(msgs)
        assert len(pks) == pl * n and len(sigs) == (pl + 32) * n
        blob, offs = self._pack_msgs(msgs)
        return self._call(f"b2k_{group}_schnorr_verify", n, pks, blob, offs, sigs, out=n)

    def schnorr_verify_dev(self, group: str, n: int, d_pks: int, d_msgs: int, d_offsets: int, d_sigs: int, d_status: int):
        """the same on device pointers ([n][48 or 96], message bytes, [n+1] uint32 offsets, [n][80 or 128], [n] status);
        enqueue only"""
        if group not in self.SCHNORR_POINT_BYTES:
            raise ValueError(f"unknown group {group!r}")
        self._call(f"b2k_{group}_schnorr_verify_dev", n, d_pks, d_msgs, d_offsets, d_sigs, d_status)

    def ed25519_dleq_verify(self, g: bytes, h: bytes, xg: bytes, xh: bytes, proofs: bytes) -> bytes:
        """n x dleq.Proof.Verify(G, H, xG, xH): points [n][32], proofs [n][128] C || R || VG || VH -> one status byte each
        (B2K_DLEQ_*: 0 OK, 2 INVALID, 3 POINT)"""
        n = len(g) // 32
        assert len(g) == len(h) == len(xg) == len(xh) == 32 * n and len(proofs) == 128 * n
        return self._call("b2k_ed25519_dleq_verify", n, g, h, xg, xh, proofs, out=n)

    def ed25519_dleq_verify_dev(self, n: int, d_g: int, d_h: int, d_xg: int, d_xh: int, d_proofs: int, d_status: int):
        """the same on device pointers; enqueue only"""
        self._call("b2k_ed25519_dleq_verify_dev", n, d_g, d_h, d_xg, d_xh, d_proofs, d_status)

    def ed25519_pvss_verify_enc_shares(self, h: bytes, commits: bytes, t: int, x: bytes, sh: bytes, v: bytes, proofs: bytes) -> bytes:
        """pvss.VerifyEncShareBatch for m deals: h [m][32], commits [m][t][32], x, sh, v [m][n][32], proofs [m][n][128]
        -> m*n status bytes (B2K_DLEQ_*)"""
        m = len(h) // 32
        n = len(x) // (32 * m)
        assert len(h) == 32 * m and len(commits) == 32 * m * t
        assert len(x) == len(sh) == len(v) == 32 * m * n and len(proofs) == 128 * m * n
        return self._call("b2k_ed25519_pvss_verify_enc_shares", m, t, n, h, commits, x, sh, v, proofs, out=m * n)

    def ed25519_pvss_verify_dec_shares(self, g: bytes, x: bytes, enc_v: bytes, dec_v: bytes, proofs: bytes) -> bytes:
        """pvss.VerifyDecShareBatch: g [32], x, enc_v, dec_v [n][32], proofs [n][128] -> n status bytes (B2K_DLEQ_*)"""
        n = len(x) // 32
        assert len(g) == 32 and len(x) == len(enc_v) == len(dec_v) == 32 * n and len(proofs) == 128 * n
        return self._call("b2k_ed25519_pvss_verify_dec_shares", n, g, x, enc_v, dec_v, proofs, out=n)

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
        return self._call("b2k_ed25519_shuffle_verify", m, k, g, h, x, y, xbar, ybar, proofs, bytes(proto), len(proto), out=m)

    def ed25519_shuffle_sequence_verifiable(self, nq: int, x: bytes, y: bytes, xbar: bytes, ybar: bytes, e: bytes):
        """shuffle.GetSequenceVerifiable: x, y, xbar, ybar [nq][k][32], e [nq][32] little-endian (raw) -> (xUp, yUp, xDown,
        yDown), each [k][32] canonical encodings"""
        k = len(x) // (32 * nq)
        assert k > 0 and len(x) == len(y) == len(xbar) == len(ybar) == 32 * nq * k and len(e) == 32 * nq
        outs = [bytearray(32 * k) for _ in range(4)]
        self._call("b2k_ed25519_shuffle_sequence_verifiable", nq, k, x, y, xbar, ybar, e, *outs)
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
        self._call("b2k_ed25519_anon_verify", n, bytes(ring) or None, int(linkable), sc or None, len(sc), m, blob, offs,
                   b"".join(sigs), status or None, tags or None)
        return bytes(status), bytes(tags)

    def ed25519_ecies_decrypt(self, priv: bytes, ctxts, length: int):
        """n x ecies.Decrypt(edwards25519, priv, ctxts[i], sha256.New); every ciphertext is 32 + length bytes (length =
        body + tag, >= 16) -> ([n] messages of length - 16 bytes, zero unless OK; n status bytes (B2K_ECIES_*: 0 OK, 1 POINT,
        2 AUTH))"""
        n = len(ctxts)
        assert len(priv) == 32 and all(len(c) == 32 + length for c in ctxts)
        msg, status = bytearray(max(n * (length - 16), 1)), bytearray(n)
        self._call("b2k_ed25519_ecies_decrypt", bytes(priv), n, length, b"".join(ctxts), msg, status)
        w = length - 16
        return [bytes(msg[w * i:w * i + w]) for i in range(n)], bytes(status)

    def ed25519_ecies_encrypt(self, pubs, rs, msgs):
        """n x ecies.Encrypt(edwards25519, pubs[i], msgs[i], sha256.New) with the ephemeral scalars rs[i] (32 bytes LE); all
        messages of one length -> ([n] ciphertexts R || C || tag, zero unless OK; n status bytes (0 OK, 1 POINT))"""
        n = len(msgs)
        length = len(msgs[0]) if n else 0
        assert len(pubs) == n and len(rs) == n and all(len(m) == length for m in msgs)
        out, status = bytearray(max(n * (length + 48), 1)), bytearray(n)
        self._call("b2k_ed25519_ecies_encrypt", n, b"".join(pubs), b"".join(rs), length, b"".join(msgs), out, status)
        w = length + 48
        return [bytes(out[w * i:w * i + w]) for i in range(n)], bytes(status)

    def bls12381_ecies_decrypt(self, group: int, priv: bytes, ctxts, length: int):
        """n x ecies.Decrypt(BLS12-381 G1 or G2, priv, ctxts[i], sha256.New), group 1 or 2; priv 32 bytes big-endian below r;
        every ciphertext is 48 (G1) or 96 (G2) + length bytes (length = body + tag, >= 16) -> ([n] messages of length - 16
        bytes, zero unless OK; n status bytes (B2K_ECIES_*: 0 OK, 1 POINT, 2 AUTH))"""
        pl = self.POINT_BYTES[f"bls12381_g{group}"][1]
        n = len(ctxts)
        assert len(priv) == 32 and all(len(c) == pl + length for c in ctxts)
        msg, status = bytearray(max(n * (length - 16), 1)), bytearray(n)
        self._call(f"b2k_bls12381_g{group}_ecies_decrypt", bytes(priv), n, length, b"".join(ctxts), msg, status)
        w = length - 16
        return [bytes(msg[w * i:w * i + w]) for i in range(n)], bytes(status)

    def bls12381_ecies_encrypt(self, group: int, pubs, rs, msgs):
        """n x ecies.Encrypt(BLS12-381 G1 or G2, pubs[i] compressed, msgs[i], sha256.New) with the ephemeral scalars rs[i]
        (32 bytes big-endian below r); all messages of one length -> ([n] ciphertexts R || C || tag, zero unless OK; n status
        bytes (0 OK, 1 POINT))"""
        pl = self.POINT_BYTES[f"bls12381_g{group}"][1]
        n = len(msgs)
        length = len(msgs[0]) if n else 0
        assert len(pubs) == n and len(rs) == n and all(len(m) == length for m in msgs)
        out, status = bytearray(max(n * (pl + length + 16), 1)), bytearray(n)
        self._call(f"b2k_bls12381_g{group}_ecies_encrypt", n, b"".join(pubs), b"".join(rs), length, b"".join(msgs), out, status)
        w = pl + length + 16
        return [bytes(out[w * i:w * i + w]) for i in range(n)], bytes(status)


class Comm:
    """One rank of the sharded MSM (include/b2kyber.h: b2k_comm_*): owns the rank's exchange slab on the engine's device.

    Wiring, one process per GPU:   c = Comm(eng, world, rank); blobs = all_gather(c.export()); c.connect(b"".join(blobs))
    one process, several engines:  comms = [Comm(e, n, r) ...]; Comm.connect_local(comms)
    """

    def __init__(self, eng: Engine, nranks: int, rank: int):
        self.eng, self.nranks, self.rank = eng, nranks, rank
        h = C.c_void_p()
        eng._call("b2k_comm_create", nranks, rank, C.byref(h))
        self.h = h

    def export(self) -> bytes:
        return self.eng._call("b2k_comm_export", out=COMM_BLOB_BYTES, h=self.h)

    def connect(self, blobs: bytes):
        assert len(blobs) == self.nranks * COMM_BLOB_BYTES
        self.eng._call("b2k_comm_connect", blobs, h=self.h)

    @staticmethod
    def connect_local(comms):
        comms[0].eng._call("b2k_comm_connect_local", len(comms), h=(C.c_void_p * len(comms))(*[c.h for c in comms]))

    def use_nccl(self, unique_id: bytes):
        self.eng._call("b2k_comm_use_nccl", unique_id, h=self.h)

    @staticmethod
    def nccl_unique_id(lib=None) -> bytes:
        buf = C.create_string_buffer(128)
        if (lib or load_library()).b2k_nccl_unique_id(buf) != 0:
            raise B2KError(-1, "b2k_nccl_unique_id failed (libnccl.so.2 not loadable)")
        return buf.raw

    def last_plan(self):
        a = (C.c_int * 4)()
        self.eng._call("b2k_comm_last_plan", a, h=self.h)
        return {"c": a[0], "W": a[1], "buckets_per_window": a[2], "bucket_bytes": a[3]}

    def msm_sharded_dev(self, n: int, d_scalars: int, d_points: int, d_out: int, shape: int = 0):
        """this rank's n resident pairs -> 48-byte sum over all ranks at d_out (enqueue only)"""
        self.eng._call("b2k_bls12381_g1_msm_sharded_dev", n, d_scalars, d_points, d_out, shape, h=self.h)

    def msm_sharded_async(self, n: int, h_scalars: int, h_points: int, h_out: int):
        """host pointers (page-locked); collect with eng.wait()"""
        self.eng._call("b2k_bls12381_g1_msm_sharded_async", n, h_scalars, h_points, h_out, h=self.h)

    @staticmethod
    def msm_multi_gpu(comms, scalars: bytes, points: bytes) -> bytes:
        """one process, len(comms) GPUs: the whole sharded MSM from host buffers (b2k_bls12381_g1_msm_multi_gpu)"""
        arr = (C.c_void_p * len(comms))(*[c.h for c in comms])
        return comms[0].eng._call("b2k_bls12381_g1_msm_multi_gpu", len(comms), len(scalars) // 32, scalars, points, out=48, h=arr)

    def close(self):
        if getattr(self, "h", None):
            self.eng.lib.b2k_comm_destroy(self.h)
            self.h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass
