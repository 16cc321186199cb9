"""CPU tests of the ctypes binding (kyber_b200/capi.py): its signatures are read from include/b2kyber.h, and its methods pass
the sizes, NULL pointers and bytes the C ABI expects -- checked against a stub library, generated from the same header, that
records every call."""
import ast
import ctypes as C
import re
import subprocess

import pytest

from kyber_b200 import capi


def test_every_header_prototype_gets_a_signature():
    sigs = capi.header_signatures()
    with open(capi.HEADER_PATH) as f:
        src = re.sub(r"/\*.*?\*/", " ", f.read(), flags=re.S)
    protos = re.findall(r"\b(b2k_[a-z0-9_]+)\s*\(", src)
    assert len(protos) == len(set(protos)) == len(sigs) and set(protos) == set(sigs)
    vp, sz = C.c_void_p, C.c_size_t
    assert sigs["b2k_version"] == (C.c_char_p, [])
    assert sigs["b2k_last_error"] == (C.c_char_p, [vp])
    assert sigs["b2k_destroy"][0] is None
    assert sigs["b2k_launch_count"][0] is C.c_uint64
    assert sigs["b2k_set_msm_reduce"] == (C.c_int, [vp, C.c_int, C.c_int, C.c_int])
    assert sigs["b2k_bls12381_hash_to_g1"] == (C.c_int, [vp, sz, vp, vp, vp, C.c_uint32, vp])
    assert sigs["b2k_bdn_coefficients"] == (C.c_int, [sz, vp, sz, C.c_int, vp])


@pytest.mark.parametrize("decl", ["int b2k_x(b2k_ctx* ctx, float scale);", "double b2k_x(b2k_ctx* ctx);",
                                  "int b2k_x(b2k_ctx* ctx, size_t);"])
def test_a_type_without_mapping_raises(tmp_path, decl):
    hdr = tmp_path / "h.h"
    hdr.write_text("/* a comment (with b2k_y(void);) */\nint b2k_ok(const uint8_t* in /*[n][64]*/,\n           size_t n);\n" + decl)
    with pytest.raises(ValueError, match="b2k_x"):
        capi.header_signatures(str(hdr))


def test_binding_declares_no_signature_of_its_own():
    with open(capi.__file__) as f:
        src = f.read()
    tree = ast.parse(src)
    everywhere = [n for n in ast.walk(tree) if isinstance(n, ast.Attribute) and n.attr in ("argtypes", "restype")]
    loader = next(n for n in ast.walk(tree) if isinstance(n, ast.FunctionDef) and n.name == "load_library")
    inside = [n for n in ast.walk(loader) if isinstance(n, ast.Attribute) and n.attr in ("argtypes", "restype")]
    assert len(everywhere) == len(inside) > 0
    stems = {id(v) for n in ast.walk(tree) if isinstance(n, ast.JoinedStr) for v in n.values}      # f"b2k_{curve}_..." parts
    named = {n.attr for n in ast.walk(tree) if isinstance(n, ast.Attribute)} | {
        n.value for n in ast.walk(tree) if isinstance(n, ast.Constant) and isinstance(n.value, str) and id(n) not in stems}
    named = {s for s in named if re.fullmatch(r"b2k_\w+", s)}
    assert named and named <= set(capi.header_signatures())


# ---- stub library ----------------------------------------------------------------------------------------------------------
_CTYPE = {C.c_int: "int", C.c_size_t: "size_t", C.c_uint32: "uint32_t", C.c_uint64: "uint64_t", C.c_void_p: "void*",
          C.c_char_p: "const char*", None: "void"}
_HOOK = C.CFUNCTYPE(C.c_longlong, C.c_char_p, C.c_int, C.POINTER(C.c_uint64))
_KEEP = []          # the hook outlives the test: an Engine's __del__ may still call the stub
CTX, COMM = 0xC7000, 0xC0000

# bytes behind each pointer argument (by position) of the calls whose bytes the tests compare; the last one is the output,
# which the stub fills with 0xA5 after reading it
READS = {
    "b2k_bls12381_g1_mul_batch": lambda a: {2: 32 * a[1], 3: 96 * a[1], 4: 48 * a[1]},
    "b2k_bls12381_g1_msm": lambda a: {2: 32 * a[1], 3: 96 * a[1], 4: 48},
    "b2k_bls12381_pairing_check": lambda a: {2: 96 * a[1], 3: 192 * a[1], 4: 96 * a[1], 5: 192 * a[1], 6: a[1]},
}


def _stub_source(sigs) -> str:
    lines = ["#include <stddef.h>", "#include <stdint.h>", "typedef long long (*hook_t)(const char*, int, const uint64_t*);",
             "static hook_t hook;", 'extern "C" void stub_set_hook(hook_t h) { hook = h; }']
    for name, (res, args) in sigs.items():
        params = ", ".join(f"{_CTYPE[a]} a{i}" for i, a in enumerate(args)) or "void"
        vals = ", ".join(f"(uint64_t)(uintptr_t)a{i}" if a is C.c_void_p else f"(uint64_t)a{i}" for i, a in enumerate(args)) or "0"
        call = f'hook("{name}", {len(args)}, v)'
        body = {None: f"{call};", C.c_char_p: f'{call}; return "stub";'}.get(res, f"return ({_CTYPE[res]}){call};")
        lines.append(f'extern "C" {_CTYPE[res]} {name}({params}) {{ const uint64_t v[] = {{{vals}}}; {body} }}')
    return "\n".join(lines) + "\n"


@pytest.fixture
def calls(tmp_path, monkeypatch):
    """(name, args) of every call into the stub: integers as passed; pointers as None (NULL), their bytes (READS), the stub's
    context / communicator handle, or True"""
    sigs = capi.header_signatures()
    src, so = tmp_path / "stub.cpp", str(tmp_path / "libstub.so")
    src.write_text(_stub_source(sigs))
    subprocess.run(["g++", "-shared", "-fPIC", "-O0", str(src), "-o", so], check=True)
    log = []

    def record(name, argc, v):
        name, a = name.decode(), [v[i] for i in range(argc)]
        if name in ("b2k_create", "b2k_comm_create"):
            C.c_void_p.from_address(a[-1]).value = CTX if name == "b2k_create" else COMM
        reads = READS.get(name, lambda a: {})(a)
        log.append((name, [(None if not x else C.string_at(x, reads[i]) if i in reads else x if x in (CTX, COMM) else True)
                           if t is C.c_void_p else x for i, (x, t) in enumerate(zip(a, sigs[name][1]))]))
        if reads:
            C.memset(a[max(reads)], 0xA5, reads[max(reads)])
        return 0

    _KEEP.append(_HOOK(record))
    monkeypatch.setattr(capi, "LIB_PATH", so)
    capi.load_library.cache_clear()
    capi.load_library().stub_set_hook(_KEEP[-1])
    yield log
    capi.load_library.cache_clear()


def _last(log, name):
    return next(args for n, args in reversed(log) if n == name)


def test_library_is_loaded_once_and_shared(calls):
    a, b = capi.Engine(), capi.Engine()
    assert a.lib is b.lib is capi.load_library()
    assert capi.Engine.bdn_coefficients(bytes(96), 96) == bytes(32)          # the stub writes nothing
    assert _last(calls, "b2k_bdn_coefficients") == [1, True, 96, 0, True]
    assert _last(calls, "b2k_create")[0] == 0 and a.h.value == CTX
    a.close(), b.close()


def test_null_pointers(calls):
    eng = capi.Engine()
    pt, m = bytes(range(32)), b"msg"
    # shuffle: g / h None = the base point; an empty proto is still a pointer
    eng.ed25519_shuffle_verify(2, pt * 2, pt * 2, pt * 2, pt * 2, bytes(32 * 27))
    assert _last(calls, "b2k_ed25519_shuffle_verify")[3:5] == [None, None]
    assert _last(calls, "b2k_ed25519_shuffle_verify")[5:] == [True] * 5 + [True, 0, True]
    eng.ed25519_shuffle_verify(2, pt * 2, pt * 2, pt * 2, pt * 2, bytes(32 * 27), b"p", g=pt, h=pt)
    assert _last(calls, "b2k_ed25519_shuffle_verify")[3:5] == [True, True]
    # commit_batch: base None (or empty) = the generator
    for base, want in ((None, None), (b"", None), (bytes(96), True)):
        assert eng.commit_batch("bls12381_g1", pt, base) == bytes(96)
        assert _last(calls, "b2k_bls12381_g1_commit_batch") == [CTX, 1, True, want, True]
    # bn256 HashG1: an empty dst is NULL; empty messages are still a pointer
    eng.bn256_hash_g1([m])
    assert _last(calls, "b2k_bn256_hash_g1") == [CTX, 1, True, True, None, 0, True]
    eng.bn256_hash_g1([b""], b"d")
    assert _last(calls, "b2k_bn256_hash_g1") == [CTX, 1, True, True, True, 1, True]
    eng.bls12381_hash_to_g1([b"", b""], b"D")
    assert _last(calls, "b2k_bls12381_hash_to_g1") == [CTX, 2, True, True, True, 1, True]
    # IBE encrypt: dst None = the default DST; an empty identity or dst is still a pointer
    eng.bls12381_ibe_encrypt(1, bytes(48), b"", [m], [b"sig"])
    assert _last(calls, "b2k_bls12381_ibe_encrypt_cca_g1")[2:7] == [True, 0, None, 0, 1]
    eng.bls12381_ibe_encrypt(1, bytes(48), b"id", [m], [b"sig"], dst=b"")
    assert _last(calls, "b2k_bls12381_ibe_encrypt_cca_g1")[2:7] == [True, 2, True, 0, 1]
    # ring signatures: an empty ring or scope is NULL; empty messages are still a pointer
    eng.ed25519_anon_verify(b"", [b""], [bytes(32)])
    assert _last(calls, "b2k_ed25519_anon_verify") == [CTX, 0, None, 0, None, 0, 1, True, True, True, True, True]
    eng.ed25519_anon_verify(b"", [b""], [bytes(64)], scope=b"")
    assert _last(calls, "b2k_ed25519_anon_verify")[1:6] == [0, None, 1, None, 0]
    eng.ed25519_anon_verify(pt, [m], [bytes(96)], scope=b"s")
    assert _last(calls, "b2k_ed25519_anon_verify")[1:6] == [1, True, 1, True, 1]
    # ECIES of empty messages: every buffer is still a pointer
    assert eng.ed25519_ecies_encrypt([pt], [pt], [b""]) == ([bytes(48)], b"\x00")
    assert _last(calls, "b2k_ed25519_ecies_encrypt") == [CTX, 1, True, True, 0, True, True, True]
    # a communicator's calls go to its own handle
    comm = capi.Comm(eng, 2, 0)
    comm.connect(bytes(2 * capi.COMM_BLOB_BYTES))
    assert _last(calls, "b2k_comm_create") == [CTX, 2, 0, True] and _last(calls, "b2k_comm_connect") == [COMM, True]
    comm.close(), eng.close()


def test_sizes_and_bytes(calls):
    eng = capi.Engine()
    s, p = bytes(range(64)), bytes(i % 251 for i in range(192))
    assert eng.bls12381_g1_mul_batch(s, p) == b"\xa5" * 96
    assert _last(calls, "b2k_bls12381_g1_mul_batch") == [CTX, 2, s, p, bytes(96)]
    assert eng.bls12381_g1_msm(bytearray(s), memoryview(bytearray(p))) == b"\xa5" * 48
    assert _last(calls, "b2k_bls12381_g1_msm") == [CTX, 2, s, p, bytes(48)]
    a1, a2, b1, b2 = bytes([1]) * 192, bytes([2]) * 384, bytes([3]) * 192, bytes([4]) * 384
    assert eng.bls12381_pairing_check(a1, a2, b1, b2) == b"\xa5\xa5"
    assert _last(calls, "b2k_bls12381_pairing_check") == [CTX, 2, a1, a2, b1, b2, bytes(2)]
    with pytest.raises(AssertionError):
        eng.bls12381_g1_msm(s, p[:-1])
    # raw calls on the bound library take the pointer half of _buf's (pointer, keepalive) pairs
    out = bytearray(48)
    bufs = [capi._buf(x) for x in (s, p, out)]
    assert eng.lib.b2k_bls12381_g1_msm(eng.h, 2, *[b[0] for b in bufs]) == 0 and out == b"\xa5" * 48
    assert _last(calls, "b2k_bls12381_g1_msm") == [CTX, 2, s, p, bytes(48)]
    eng.close()
