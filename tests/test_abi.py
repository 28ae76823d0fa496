"""CPU checks of the C-ABI boundary: the shared library loads and exports every
symbol include/ga_b200.h declares; host-only entry points behave; the product
package never imports the oracle."""
import ctypes as C
import os
import re

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _header():
    """include/ga_b200.h without comments and preprocessor lines."""
    src = open(os.path.join(ROOT, "include", "ga_b200.h")).read()
    src = re.sub(r"/\*.*?\*/", "", src, flags=re.S)
    return re.sub(r"^\s*#.*$", "", src, flags=re.M)


def _declared_functions():
    """{name: (return type, [parameter declarations])} of every function the header declares."""
    return {name: (" ".join(ret.split()), [p.strip() for p in params.split(",") if p.strip() not in ("", "void")])
            for ret, name, params in re.findall(r"([^;{}]*?)\b(ga_\w+)\s*\(([^)]*)\)\s*;", _header())}


def _declared_fields(struct):
    """[field declarations] of `typedef struct <struct> {...}` in the header, one per field ('void *q, *k' -> two)."""
    body = re.search(r"typedef struct %s \{(.*?)\} %s;" % (struct, struct), _header(), flags=re.S).group(1)
    fields = []
    for decl in filter(str.strip, body.split(";")):
        first, *more = decl.split(",")
        base = re.match(r"\s*((?:const\s+)?\w+)", first).group(1)
        fields += [" ".join(first.split())] + ["%s %s" % (base, m.strip()) for m in more]
    return fields


def _ctype_matches(decl, ct):
    """decl: a named C declaration of the header ('const float *bias', 'int64_t n'); ct: the ctypes type for it.
    A pointer may be c_void_p or a POINTER to the pointee's type."""
    from gaussiananything_b200 import _lib
    base, stars = re.fullmatch(r"\s*(?:const\s+)?(\w+)\s*(\**)\s*\w+\s*", decl).groups()
    scalar = {"int": C.c_int, "int32_t": C.c_int32, "int64_t": C.c_int64, "size_t": C.c_size_t, "float": C.c_float}
    want = scalar[base] if base in scalar else getattr(_lib, base, None)
    if stars:
        return ct is C.c_void_p or (want is not None and ct is C.POINTER(want))
    return ct is want


def test_library_exports_every_declared_symbol():
    from gaussiananything_b200 import _lib
    L = _lib.lib()
    names = _declared_functions()
    assert len(names) >= 7
    for n in names:
        assert hasattr(L, n), "libga_b200.so does not export %s" % n
    assert b"sm_90a" in L.ga_b200_version()


def test_ctypes_table_matches_header():
    """_lib.lib() declares restype and argtypes for every function of the header, parameter by parameter as the
    header states them, the ctypes structures have the header's fields in the header's order, and the EPI_* mode
    constants are the header's GA_EPI_*.  ctypes does not check a call against the C prototype: a wrong width, a
    missing argument or a wrong mode would pass a wrong value silently."""
    from gaussiananything_b200 import _lib
    L = _lib.lib()
    decls = _declared_functions()
    assert sorted(_lib.ABI) == sorted(decls), set(_lib.ABI) ^ set(decls)
    rets = {"int": C.c_int, "size_t": C.c_size_t, "const char *": C.c_char_p}
    for name, (ret, params) in decls.items():
        fn = getattr(L, name)
        assert fn.restype is rets[ret], (name, ret, fn.restype)
        assert fn.argtypes is not None and len(fn.argtypes) == len(params), (name, params, fn.argtypes)
        for decl, ct in zip(params, fn.argtypes):
            assert _ctype_matches(decl, ct), (name, decl, ct)
    for cls in (_lib.GaRasterLayout, _lib.GaGemmEpilogue, _lib.GaVaeEncHead):
        fields = _declared_fields(cls.__name__)
        assert [n for n, _ in cls._fields_] == [re.search(r"(\w+)\s*$", f).group(1) for f in fields], cls.__name__
        for f, (n, ct) in zip(fields, cls._fields_):
            assert _ctype_matches(f, ct), (cls.__name__, f, ct)
    header = open(os.path.join(ROOT, "include", "ga_b200.h")).read()
    modes = {"EPI_" + n: int(v) for n, v in re.findall(r"^#define GA_EPI_(\w+)\s+(\d+)", header, flags=re.M)}
    assert len(modes) == 6 and modes == {n: getattr(_lib, n) for n in dir(_lib) if n.startswith("EPI_")}, modes


def test_layout_ex_is_host_only_and_monotonic():
    from gaussiananything_b200 import _lib
    L = _lib.lib()
    a, b = _lib.GaRasterLayout(), _lib.GaRasterLayout()
    assert L.ga_raster_layout_ex(1, 1000, 2, 64, 64, 5000, 0, C.byref(a)) == 0
    assert L.ga_raster_layout_ex(1, 1000, 2, 64, 64, 10000, 0, C.byref(b)) == 0
    assert b.total_bytes > a.total_bytes > 0
    offs = [a.status, a.rec, a.depth, a.rect, a.tile_count, a.tile_start, a.keys, a.ids, a.final_T, a.n_contrib]
    assert offs == sorted(offs) and all(o % 256 == 0 for o in offs)
    # error behaviour: bad sizes are rejected, not crashed on
    assert L.ga_raster_layout_ex(0, 10, 1, 64, 64, 10, 0, C.byref(a)) == -1
    assert L.ga_raster_layout_ex(1, 10, 1, 5000, 64, 10, 0, C.byref(a)) == -3
    assert L.ga_raster_backward_scratch_bytes(1, 1000, 2) >= 1000 * 2 * 18 * 4


def test_tile_replicas_read_from_the_layout():
    """raster.workspace_views finds the big-tile list after the tile counters, whose replica count it reads from the
    layout; the layout grows by exactly that many words per tile plus one."""
    from gaussiananything_b200 import raster
    R = raster.tile_replicas()
    assert R >= 1
    a, b = raster.layout(1, 1, 1, 128, 128, 1), raster.layout(1, 1, 4, 128, 128, 1)      # 64 and 256 tiles
    assert b.tile_start - b.tile_count == 256 * (R + 1) * 4 and a.tile_start - a.tile_count == 64 * (R + 1) * 4


def test_forward_ex_rejects_null_small_workspace_and_one_status_pointer():
    """Argument checks that return before any CUDA call, so the dummy pointers below are never dereferenced."""
    from gaussiananything_b200 import _lib
    L = _lib.lib()

    def fwd(ptr, status_host, status_event):
        return L.ga_raster_forward_ex(ptr, 1, 10, 1, ptr, ptr, ptr, 32, 32, 1.0, ptr, ptr, ptr, ptr, 0, 10, 0,
                                      status_host, status_event, None)
    assert fwd(None, None, None) == -1
    assert fwd(256, None, None) == -2                    # a 0-byte workspace is smaller than the layout
    # the status read-back takes both the pinned buffer and the event, or neither
    assert fwd(256, 256, None) == -1 and fwd(256, None, 256) == -1


def test_gemm_validate_rules():
    """ga_gemm_validate is host-only: fake, never dereferenced addresses.  Each rule of the header, one at a time,
    from an accepted call of every mode."""
    from gaussiananything_b200 import _lib
    L = _lib.lib()
    A, W, OUT = 0x100000, 0x200000, 0x300000
    base = dict(M=300, N=512, K=256, lda=264, ldw=256, bn=128)

    def rc(mode, bn=None, M=None, N=None, K=None, lda=None, ldw=None, A_=A, W_=W, **fields):
        f = dict({0: dict(out=OUT, ld_out=512), 1: dict(out=OUT, ld_out=512), 2: dict(out=OUT, ld_out=515),
                  3: dict(out=OUT, ld_out=512), 5: dict(out=OUT, ld_out=256),
                  4: dict(q=OUT, k=OUT + 0x10000, vt=OUT + 0x20000, heads=4, first_part=1, rows_per_batch=150,
                          tok_pitch=256)}.get(mode, dict(out=OUT, ld_out=512)), **fields)
        e = _lib.GaGemmEpilogue(mode=mode, eps=1e-5, **f)
        g = lambda v, k: base[k] if v is None else v
        return L.ga_gemm_validate(A_, g(lda, "lda"), W_, g(ldw, "ldw"), g(M, "M"), g(N, "N"), g(K, "K"), C.byref(e),
                                  g(bn, "bn"))

    for mode in range(6):
        assert rc(mode) == 0, mode
        for bn in (64, 192, 256):
            assert rc(mode, bn=bn) == (-1 if mode == 4 and bn != 256 else 0), (mode, bn)
    assert rc(3, gate=0x400000, gate_ld=512, rows_per_batch=1) == 0
    assert L.ga_gemm_validate(A, 264, W, 256, 300, 512, 256, None, 128) == -1           # epi NULL
    bad = [
        dict(A_=0), dict(W_=0), dict(M=0), dict(N=0), dict(K=0), dict(bn=96), dict(bn=0),
        dict(A_=A + 8), dict(W_=W + 2),                                              # TMA bases: 16 bytes
        dict(lda=260), dict(ldw=252), dict(lda=248), dict(K=272),                    # pitch % 8, pitch >= K
        dict(out=0), dict(ld_out=511),
        dict(out=OUT + 8), dict(out=OUT + 4),                                         # fp32: 16-byte out
        dict(gate=0x400000, gate_ld=512, rows_per_batch=0), dict(gate=0x400000, gate_ld=511, rows_per_batch=1),
    ]
    for kw in bad[:15]:
        for mode in (0, 1, 2, 3, 5):
            if "ld_out" in kw and mode == 5:
                continue
            assert rc(mode, **kw) == -1, (mode, kw)
    for mode in (2, 3):
        assert rc(mode, out=OUT + 8) == -1 and rc(mode, out=OUT + 4) == -1
    for mode in (0, 1):
        assert rc(mode, out=OUT + 8) == 0 and rc(mode, out=OUT + 4) == -1 and rc(mode, out=OUT + 2) == -1
    assert rc(5, out=OUT + 4) == 0 and rc(5, out=OUT + 2) == -1
    assert rc(5, ld_out=255) == -1 and rc(5, N=511, ld_out=256) == -1              # GEGLU: ld_out >= N / 2, N even
    for kw in bad[17:]:
        assert rc(3, **kw) == -1, kw
    assert rc(3, gate=0, gate_ld=0, rows_per_batch=0) == 0                          # no gate: neither is read
    assert rc(6) == -1 and rc(-1) == -1
    # HEADS: N = 512 = 2 parts of 4 heads x 64, starting at k
    assert rc(4, bn=256) == 0 and rc(4, first_part=0) == 0
    heads_bad = [dict(heads=0), dict(heads=3), dict(first_part=2), dict(first_part=-1), dict(heads=2),
                 dict(k=0), dict(vt=0), dict(k=OUT + 8), dict(vt=OUT + 0x20008),
                 dict(rows_per_batch=0), dict(tok_pitch=149)]
    for kw in heads_bad:
        assert rc(4, **kw) == -1, kw
    assert rc(4, N=448) == -1                                                        # not whole heads
    assert rc(4, N=768, first_part=0) == 0 and rc(4, N=768, first_part=1) == -1    # a 4th part
    assert rc(4, N=1024, first_part=0) == -1
    assert rc(4, q=0) == 0 and rc(4, q=0, first_part=0) == -1                       # q only when part 0 is reached
    assert rc(4, N=256, first_part=0, k=0, vt=0) == 0                              # q only
    assert rc(4, N=256, first_part=0, q=0) == -1


def test_attention_validate_rules():
    from gaussiananything_b200 import _lib
    L = _lib.lib()
    Q, K, V, O = 0x100000, 0x200000, 0x300000, 0x400000

    def rc(causal=0, **kw):
        a = dict(Q=Q, K=K, V=V, O=O, B=2, H=16, Nq=768, Nk=1369, pq=768, pk=1408)
        a.update(kw)
        if causal and "Nk" not in kw:
            a.update(Nk=a["Nq"], pk=_ru(a["Nq"]))
        return L.ga_attention_validate(a["Q"], a["K"], a["V"], a["O"], a["B"], a["H"], a["Nq"], a["Nk"], a["pq"],
                                       a["pk"], causal)

    _ru = lambda n: (n + 127) // 128 * 128
    assert rc() == 0 and rc(causal=1) == 0 and rc(Nq=17, pq=17) == 0 and rc(O=O + 4) == 0
    for kw in (dict(Q=0), dict(K=0), dict(V=0), dict(O=0), dict(B=0), dict(H=0), dict(Nq=0), dict(Nk=0),
               dict(pq=767), dict(pk=1280), dict(pk=1409), dict(Q=Q + 8), dict(K=K + 8), dict(V=V + 2),
               dict(O=O + 2)):
        assert rc(**kw) == -1, kw
    assert rc(causal=1, Nk=767, pk=768) == -1 and rc(causal=0, Nk=767, pk=768) == 0
    assert rc(B=1, H=65535) == 0 and rc(B=2, H=32768) == -3 and rc(B=65536, H=1) == -3


def test_product_never_touches_the_oracle():
    pkg = os.path.join(ROOT, "gaussiananything_b200")
    for dp, _, fs in os.walk(pkg):
        for f in fs:
            if f.endswith((".py", ".cu", ".cuh", ".h")):
                s = open(os.path.join(dp, f)).read()
                assert "import oracle" not in s and "from oracle" not in s, f
                assert "surfel_oracle.so" not in s and "libsurfel_oracle" not in s, f


def test_cpu_tensors_fail_loudly():
    import torch
    from gaussiananything_b200 import raster
    with pytest.raises(RuntimeError):
        raster.forward_raw(torch.zeros(1, 4, 13), torch.eye(4).reshape(1, 1, 4, 4),
                           torch.eye(4).reshape(1, 1, 4, 4), torch.ones(3), 32, 32)


def test_install_shims_registers_reference_module_names():
    import sys
    import gaussiananything_b200 as ga
    saved = {k: sys.modules.get(k) for k in ("diff_surfel_rasterization", "transport", "transport.transport")}
    try:
        ga.install_shims()
        import diff_surfel_rasterization as dsr          # the name nsr/gs_surfel.py:15 imports
        import transport as tr                           # the name flow_matching_trainer.py imports
        assert hasattr(dsr, "GaussianRasterizationSettings") and hasattr(dsr, "GaussianRasterizer")
        assert hasattr(tr, "create_transport") and hasattr(tr, "Sampler")
        fields = dsr.GaussianRasterizationSettings._fields
        assert fields == ("image_height", "image_width", "tanfovx", "tanfovy", "bg", "scale_modifier", "viewmatrix",
                          "projmatrix", "sh_degree", "campos", "prefiltered", "debug")
    finally:
        for k, v in saved.items():
            if v is None:
                sys.modules.pop(k, None)
            else:
                sys.modules[k] = v


def test_missing_library_fails_loudly_in_every_binding():
    """No CPU fallback anywhere on the product path: with the shared library absent the rasteriser, the DiT binding and
    the VAE decoder all raise (checked in a child process so this process keeps its loaded library)."""
    import subprocess
    import sys
    code = (
        "import torch\n"
        "from gaussiananything_b200 import _lib, raster, dit, vae_decoder\n"
        "n = 0\n"
        "for f in (_lib.lib, dit._bind, lambda: vae_decoder.SurfelDecoder({}, 12, 12),\n"
        "          lambda: raster.layout(1, 10, 1, 32, 32, 100)):\n"
        "    try:\n"
        "        f()\n"
        "    except RuntimeError as e:\n"
        "        assert 'no CPU fallback' in str(e) or 'missing' in str(e), e\n"
        "        n += 1\n"
        "print('raised', n)\n")
    env = dict(os.environ, GA_B200_LIB="/nonexistent/libga_b200.so")
    out = subprocess.run([sys.executable, "-c", code], cwd=ROOT, env=env, capture_output=True, text=True, timeout=300)
    assert out.returncode == 0, out.stderr[-2000:]
    assert "raised 4" in out.stdout, out.stdout + out.stderr[-1000:]


def test_decoder_refuses_cpu_devices():
    """(The DiT modules' CPU refusal is in tests/test_oracle_dit.py::test_dit_module_has_reference_state_dict_layout.)"""
    from gaussiananything_b200.vae_decoder import SurfelDecoder
    with pytest.raises(RuntimeError, match="no CPU fallback"):
        SurfelDecoder({}, 12, 12, device="cpu")
