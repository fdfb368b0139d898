"""The C-ABI library loads on a CPU-only box and exports every symbol include/gnark_b200.h
declares; product code fails loudly (no CPU fallback) when no device is present."""
import os
import re

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def declared_symbols():
    src = open(os.path.join(ROOT, "include", "gnark_b200.h")).read()
    src = re.sub(r"/\*.*?\*/", "", src, flags=re.S)
    return sorted(set(re.findall(r"\b(b200_[a-z0-9_]+)\s*\(", src)))


def test_exports(b200lib):
    syms = declared_symbols()
    assert len(syms) >= 30
    for s in syms:
        assert hasattr(b200lib, s), f"{s} declared in include/gnark_b200.h but not exported"
    from gnark_b200 import lib
    assert set(lib.EXPORTS) == set(syms)
    assert b"sm_90a" in b200lib.b200_version()


def test_no_cpu_fallback(b200lib):
    import torch
    if torch.cuda.is_available():
        pytest.skip("device present")
    from gnark_b200 import lib
    with pytest.raises(lib.B200Error):
        lib.init([0])
    with pytest.raises(lib.B200Error):
        lib.Table(lib.BN254, 1, np.zeros((4, 8), dtype=np.uint64), precomp=False)
    with pytest.raises(lib.B200Error):
        lib.Domain(lib.BN254, 4)


def test_product_does_not_import_oracle():
    """oracle/ is test infrastructure: no product source may import, include or link it."""
    pkg = os.path.join(ROOT, "gnark_b200")
    pat = re.compile(r"^\s*(from\s+oracle|import\s+oracle|#\s*include\s+[\"<][^\">]*oracle)", re.M)
    for dirpath, _, files in os.walk(pkg):
        for f in files:
            if f.endswith((".py", ".cu", ".cuh", ".h", ".cpp")) or f == "Makefile":
                txt = open(os.path.join(dirpath, f), errors="ignore").read()
                assert not pat.search(txt), f
                assert "liboracle" not in txt, f


def test_host_point_helpers(b200lib):
    """b200_point_add_jac / b200_point_to_affine are pure CPU (used to combine shards)."""
    import random
    from gnark_b200 import lib
    from oracle import ec, ff
    from oracle.params import CURVES
    rng = random.Random(2)
    for c in CURVES.values():
        for group in (1, 2):
            F = ff.base_field(c, group)
            from util import pick_base
            _, base = pick_base(c, group, rng)
            p = ec.scalar_mul(F, 1234567, base)
            q = ec.scalar_mul(F, 7654321, base)
            J = lambda pt: np.concatenate([ec.pack_points(c, group, [pt]).reshape(-1),
                                           ff.pack_elements(F.coords(F.one), c.p, c.fp_limbs).reshape(-1)])
            acc = J(p)
            lib.point_add_jac(c.curve_id, group, acc, J(q))
            aff = lib.point_to_affine(c.curve_id, group, acc)
            assert ec.unpack_points(c, group, aff)[0] == ec.affine_add(F, p, q)
            acc = J(p)
            lib.point_add_jac(c.curve_id, group, acc, J(p))           # doubling path
            assert ec.unpack_points(c, group, lib.point_to_affine(c.curve_id, group, acc))[0] == ec.affine_add(F, p, p)


def test_file_staging_of_dump_slices(hostemu, tmp_path):
    """file_stage.h - the host half of b200_table_upload_file (point slices of gnark's ProvingKey dump go from the file
    to the device through two staging slots): every byte of the range exactly once and in place, ranges that are not a
    multiple of the slot, a range inside a larger file, a file that is too short, a missing file."""
    import ctypes
    import numpy as np
    rs = np.random.RandomState(3)
    data = rs.randint(0, 256, size=100_003, dtype=np.uint8)
    f = tmp_path / "dump.bin"
    f.write_bytes(data.tobytes())
    path = str(f).encode()
    hostemu.emu_stage_file.argtypes = [ctypes.c_char_p, ctypes.c_uint64, ctypes.c_size_t, ctypes.c_size_t, ctypes.c_void_p]
    for off, nbytes, slot in ((0, 100_003, 4096), (17, 64 * 1000, 64 * 7), (99_000, 1003, 1 << 20), (5, 0, 128), (0, 4096, 4096)):
        out = np.zeros(max(nbytes, 1), dtype=np.uint8)
        assert hostemu.emu_stage_file(path, off, nbytes, slot, out.ctypes.data) == 0
        assert np.array_equal(out[:nbytes], data[off:off + nbytes]), (off, nbytes, slot)
    out = np.zeros(2000, dtype=np.uint8)
    assert hostemu.emu_stage_file(path, 99_000, 2000, 512, out.ctypes.data) == -2         # range exceeds the file
    assert hostemu.emu_stage_file(str(tmp_path / "missing").encode(), 0, 16, 16, out.ctypes.data) == -1


def test_pedersen_fold_host(b200lib):
    """b200_pedersen_fold (ProofOfKnowledge.Fold, backend/groth16/bn254/prove.go:127) is pure CPU: sum_i c^i * pok_i
    against the big-int oracle, for 0, 1 and several proofs of knowledge, a challenge of 0 and a pok at infinity"""
    import random
    from gnark_b200 import lib
    from oracle import ec, ff
    from oracle.params import CURVES
    rng = random.Random(12)
    for c in (CURVES["bn254"], CURVES["bls12-381"], CURVES["bw6-761"]):
        F = ff.Fp(c.p)
        for count, chal in ((0, 5), (1, rng.randrange(c.r)), (4, rng.randrange(c.r)), (3, 0), (3, 1)):
            pts = [ec.scalar_mul(F, rng.randrange(1, c.r), c.g1) for _ in range(count)]
            if count == 4:
                pts[2] = None                                               # a pok at infinity: (0, 0) in gnark's layout
            want = None
            for i, P in enumerate(pts):
                want = ec.affine_add(F, want, ec.scalar_mul(F, pow(chal, i, c.r), P))
            packed = ec.pack_points(c, 1, pts) if count else np.zeros(0, dtype=np.uint64)
            got = lib.pedersen_fold(c.curve_id, packed, ff.pack_elements([chal], c.r, c.fr_limbs))
            assert ec.unpack_points(c, 1, got)[0] == want, (c.name, count, chal)
