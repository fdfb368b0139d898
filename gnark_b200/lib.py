"""ctypes binding of libgnark_b200.so (include/gnark_b200.h).

This is the Python twin of the cgo shim shown in INTEGRATION.md.  It loads the
in-tree CUDA library ONLY: there is no CPU fallback, and nothing here imports
``oracle/``.  A missing library or a missing CUDA device raises.
"""

import ctypes
import os

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_HERE, "lib", "libgnark_b200.so")

BN254, BLS12_381, BLS12_377, BW6_761 = 0, 1, 2, 3
DIF, DIT = 0, 1
TABLE_PRECOMP = 1
TABLE_SRC_ON_DEVICE = 2
POINTS_RAW, POINTS_COMPRESSED = 1, 2
VEC_MUL, VEC_ADD, VEC_SUB = 0, 1, 2

CURVE_IDS = {"bn254": BN254, "bls12-381": BLS12_381, "bls12-377": BLS12_377, "bw6-761": BW6_761}
# (fr limbs64, fp limbs64, g2 extension degree)
CURVE_SHAPES = {BN254: (4, 4, 2), BLS12_381: (4, 6, 2), BLS12_377: (4, 6, 2), BW6_761: (6, 12, 1)}

EXPORTS = [
    "b200_version", "b200_last_error", "b200_device_count", "b200_init", "b200_shutdown", "b200_set_stream",
    "b200_sync", "b200_alloc", "b200_free", "b200_h2d", "b200_d2h", "b200_host_alloc", "b200_host_free",
    "b200_table_upload", "b200_table_upload_file", "b200_table_free", "b200_table_info", "b200_msm", "b200_msm_g1", "b200_msm_g2",
    "b200_msm_async", "b200_msm_pipelined", "b200_msm_join", "b200_msm_profile", "b200_ntt_domain_new", "b200_ntt_domain_free", "b200_ntt", "b200_ntt_async",
    "b200_groth16_compute_h", "b200_vec_op", "b200_vec_bit_reverse", "b200_vec_scale_powers",
    "b200_vec_batch_invert", "b200_plonk_constraints_coset", "b200_plonk_divide_by_zh",
    "b200_vec_axpy", "b200_vec_scan", "b200_plonk_build_z", "b200_poly_eval", "b200_poly_div_by_linear",
    "b200_point_add_jac", "b200_point_to_affine", "b200_groth16_pk_load", "b200_groth16_pk_free", "b200_groth16_prove", "b200_groth16_msms",
    "b200_groth16_assemble", "b200_fixed_base_batch", "b200_msm_submit",
    "b200_plonk_pk_load", "b200_plonk_pk_free", "b200_plonk_prove", "b200_plonk_begin", "b200_plonk_commit_z",
    "b200_plonk_quotient", "b200_plonk_linearise", "b200_plonk_batch_open", "b200_plonk_end", "b200_plonk_bsb22_coset",
    "b200_comm_unique_id", "b200_comm_init", "b200_comm_init_all", "b200_comm_destroy", "b200_comm_info",
    "b200_points_allreduce", "b200_msm_allreduce", "b200_msm_submit_dev", "b200_plonk_last_stage_ms", "b200_points_fold",
    "b200_plonk_set_qk", "b200_plonk_set_quotient_randomizers", "b200_table_upload_encoded", "b200_msm_gather", "b200_pedersen_key_load", "b200_pedersen_key_free", "b200_pedersen_commit", "b200_pedersen_fold",
    "b200_points_ntt", "b200_msm_indexed", "b200_msm_batch", "b200_ntt_batch", "b200_groth16_prove_batch",
    "b200_poly_eval_batch", "b200_kzg_open_batch", "b200_kzg_fold_open", "b200_points_scale", "b200_points_decode",
]
COMM_ID_BYTES = 128


class B200Error(RuntimeError):
    pass


class PlonkPkDesc(ctypes.Structure):
    _fields_ = ([("log2n", ctypes.c_uint32)]
                + [(k, ctypes.c_void_p) for k in ("ql", "qr", "qm", "qo", "qk", "perm", "srs_canonical")]
                + [("n_qcp", ctypes.c_uint32), ("qcp", ctypes.POINTER(ctypes.c_void_p))])


class PlonkChallenges(ctypes.Structure):
    _fields_ = ([(k, ctypes.c_void_p) for k in ("gamma", "beta", "alpha", "zeta", "v", "bl", "br", "bo", "bz")]
                + [("pi2", ctypes.POINTER(ctypes.c_void_p)), ("out_bsb22", ctypes.c_void_p), ("qk", ctypes.c_void_p),
                   ("hr", ctypes.c_void_p)])


class Groth16PkDesc(ctypes.Structure):
    _fields_ = [
        ("curve", ctypes.c_int32),
        ("domain_size", ctypes.c_uint64),
        ("domain_gen", ctypes.c_void_p),
        ("coset_gen", ctypes.c_void_p),
        ("g1_alpha", ctypes.c_void_p),
        ("g1_beta", ctypes.c_void_p),
        ("g1_delta", ctypes.c_void_p),
        ("g2_beta", ctypes.c_void_p),
        ("g2_delta", ctypes.c_void_p),
        ("g1_a", ctypes.c_void_p), ("n_a", ctypes.c_size_t),
        ("g1_b", ctypes.c_void_p), ("n_b", ctypes.c_size_t),
        ("g1_z", ctypes.c_void_p), ("n_z", ctypes.c_size_t),
        ("g1_k", ctypes.c_void_p), ("n_k", ctypes.c_size_t),
        ("g2_b", ctypes.c_void_p), ("n_b2", ctypes.c_size_t),
        ("infinity_a", ctypes.c_void_p),
        ("infinity_b", ctypes.c_void_p),
        ("nb_wires", ctypes.c_size_t),
        ("nb_public", ctypes.c_size_t),
        ("flags", ctypes.c_int32),
        ("shard_rank", ctypes.c_int32),
        ("shard_world", ctypes.c_int32),
        ("k_removed", ctypes.c_void_p),
        ("n_k_removed", ctypes.c_size_t),
        ("dump_path", ctypes.c_char_p),
        ("dump_off_a", ctypes.c_uint64), ("dump_off_b", ctypes.c_uint64), ("dump_off_z", ctypes.c_uint64),
        ("dump_off_k", ctypes.c_uint64), ("dump_off_b2", ctypes.c_uint64),
    ]


_lib = None


def load(path: str = None):
    """Load the shared library (no CUDA call is made here)."""
    global _lib
    if _lib is not None and path is None:
        return _lib
    # GB200_LIB: load another build of the same library (e.g. libgnark_b200_opt.so, `make -C gnark_b200/csrc opt`:
    # dedicated Montgomery squaring + lazily reduced Fp2 product) for A/B runs on hardware
    p = path or os.environ.get("GB200_LIB") or LIB_PATH
    if not os.path.exists(p):
        raise B200Error(
            f"{p} not found: build it with `python -c 'import __graft_entry__ as g; g.build()'` "
            "(there is no CPU fallback)")
    lib = ctypes.CDLL(p)
    lib.b200_version.restype = ctypes.c_char_p
    lib.b200_last_error.restype = ctypes.c_char_p
    variant = p != LIB_PATH      # an A/B build loaded through GB200_LIB may predate the newest entry points
    missing = [name for name in EXPORTS if not hasattr(lib, name)]
    if missing and not variant:
        raise B200Error(f"{p} lacks {missing}: stale build, rebuild it (make -C gnark_b200/csrc)")
    for name in EXPORTS:
        if name in missing:
            continue
        fn = getattr(lib, name)
        if name not in ("b200_version", "b200_last_error"):
            fn.restype = ctypes.c_int32
    vp, sz, i32, u32 = ctypes.c_void_p, ctypes.c_size_t, ctypes.c_int32, ctypes.c_uint32
    lib.b200_device_count.argtypes = [ctypes.POINTER(i32)]
    lib.b200_init.argtypes = [i32, ctypes.POINTER(i32)]
    lib.b200_set_stream.argtypes = [i32, vp]
    lib.b200_sync.argtypes = [i32]
    lib.b200_alloc.argtypes = [i32, sz, ctypes.POINTER(vp)]
    lib.b200_free.argtypes = [i32, vp]
    lib.b200_h2d.argtypes = [i32, vp, vp, sz]
    lib.b200_d2h.argtypes = [i32, vp, vp, sz]
    lib.b200_host_alloc.argtypes = [sz, ctypes.POINTER(vp)]
    lib.b200_host_free.argtypes = [vp]
    lib.b200_table_upload.argtypes = [i32, i32, i32, vp, sz, i32, ctypes.POINTER(vp)]
    lib.b200_table_upload_file.argtypes = [i32, i32, i32, ctypes.c_char_p, ctypes.c_uint64, sz, i32, ctypes.POINTER(vp)]
    lib.b200_table_free.argtypes = [vp]
    lib.b200_table_info.argtypes = [vp, ctypes.POINTER(sz), ctypes.POINTER(i32), ctypes.POINTER(i32),
                                    ctypes.POINTER(i32), ctypes.POINTER(sz)]
    for n in ("b200_msm", "b200_msm_g1", "b200_msm_g2"):
        getattr(lib, n).argtypes = [vp, sz, sz, vp, i32, vp]
    lib.b200_msm_async.argtypes = [vp, sz, sz, vp, vp]
    lib.b200_msm_pipelined.argtypes = [vp, sz, sz, vp, vp]
    lib.b200_msm_join.argtypes = [i32]
    lib.b200_msm_submit.argtypes = [vp, sz, sz, vp, vp]
    if "b200_comm_init" not in missing:
        lib.b200_comm_unique_id.argtypes = [vp]
        lib.b200_comm_init.argtypes = [i32, i32, i32, vp]
        lib.b200_comm_init_all.argtypes = [i32, ctypes.POINTER(i32)]
        lib.b200_comm_destroy.argtypes = [i32]
        lib.b200_comm_info.argtypes = [i32, ctypes.POINTER(i32), ctypes.POINTER(i32)]
        lib.b200_points_allreduce.argtypes = [i32, i32, i32, vp, sz, vp]
        lib.b200_msm_allreduce.argtypes = [vp, sz, sz, vp, i32, vp]
        lib.b200_msm_submit_dev.argtypes = [vp, sz, sz, vp, vp]
    if "b200_msm_gather" not in missing:
        lib.b200_msm_gather.argtypes = [vp, sz, vp, sz, i32, vp, sz, i32, vp]
        lib.b200_pedersen_key_load.argtypes = [i32, i32, vp, vp, sz, ctypes.POINTER(vp)]
        lib.b200_pedersen_key_free.argtypes = [vp]
        lib.b200_pedersen_commit.argtypes = [vp, vp, sz, i32, vp, vp]
        lib.b200_pedersen_fold.argtypes = [i32, vp, sz, vp, vp]
    if "b200_msm_indexed" not in missing:
        lib.b200_msm_indexed.argtypes = [vp, vp, sz, i32, vp, i32, vp]
    if "b200_msm_batch" not in missing:
        lib.b200_msm_batch.argtypes = [vp, sz, sz, sz, vp, i32, vp]
    if "b200_kzg_open_batch" not in missing:
        lib.b200_poly_eval_batch.argtypes = [i32, i32, vp, sz, sz, i32, vp, vp]
        lib.b200_kzg_open_batch.argtypes = [vp, vp, sz, sz, i32, vp, vp, vp]
        lib.b200_kzg_fold_open.argtypes = [vp, vp, sz, sz, i32, vp, vp, vp]
    if "b200_table_upload_encoded" not in missing:
        lib.b200_table_upload_encoded.argtypes = [i32, i32, i32, vp, sz, i32, i32, ctypes.POINTER(vp)]
    if "b200_plonk_set_qk" not in missing:
        lib.b200_plonk_set_qk.argtypes = [vp, vp]
    if "b200_plonk_set_quotient_randomizers" not in missing:
        lib.b200_plonk_set_quotient_randomizers.argtypes = [vp, vp]
    if "b200_points_fold" not in missing:
        lib.b200_points_fold.argtypes = [i32, i32, i32, vp, u32, u32, vp]
    if "b200_plonk_last_stage_ms" not in missing:
        lib.b200_plonk_last_stage_ms.argtypes = [vp, ctypes.POINTER(ctypes.c_double)]
    lib.b200_plonk_pk_load.argtypes = [i32, i32, ctypes.POINTER(PlonkPkDesc), ctypes.POINTER(vp)]
    lib.b200_plonk_pk_free.argtypes = [vp]
    lib.b200_plonk_prove.argtypes = [vp, vp, vp, vp, ctypes.POINTER(PlonkChallenges), vp, vp]
    lib.b200_plonk_begin.argtypes = [vp, vp, vp, vp, vp, vp, vp, ctypes.POINTER(vp), vp, ctypes.POINTER(vp), vp]
    lib.b200_plonk_commit_z.argtypes = [vp, vp, vp, vp, vp]
    lib.b200_plonk_quotient.argtypes = [vp, vp, vp]
    lib.b200_plonk_linearise.argtypes = [vp, vp, vp, vp]
    lib.b200_plonk_batch_open.argtypes = [vp, vp, vp]
    lib.b200_plonk_end.argtypes = [vp]
    lib.b200_plonk_bsb22_coset.argtypes = [vp, vp, vp, u32, u32, vp]
    lib.b200_fixed_base_batch.argtypes = [i32, i32, i32, vp, vp, i32, sz, vp, i32]
    lib.b200_msm_profile.argtypes = [vp, sz, sz, vp, vp, ctypes.POINTER(ctypes.c_float)]
    lib.b200_ntt_domain_new.argtypes = [i32, i32, u32, vp, vp, ctypes.POINTER(vp)]
    lib.b200_ntt_domain_free.argtypes = [vp]
    lib.b200_ntt.argtypes = [vp, vp, i32, i32, i32, i32]
    lib.b200_ntt_async.argtypes = [vp, vp, i32, i32, i32]
    if "b200_ntt_batch" not in missing:
        lib.b200_ntt_batch.argtypes = [vp, vp, sz, i32, i32, i32, i32]
    if "b200_points_ntt" not in missing:
        lib.b200_points_ntt.argtypes = [vp, i32, vp, i32, i32]
    if "b200_points_scale" not in missing:
        lib.b200_points_scale.argtypes = [i32, i32, i32, vp, sz, i32, vp, vp]
        lib.b200_points_decode.argtypes = [i32, i32, i32, vp, sz, i32, vp, i32]
    lib.b200_groth16_compute_h.argtypes = [vp, vp, vp, vp, sz, i32, vp, i32]
    lib.b200_vec_op.argtypes = [i32, i32, i32, vp, vp, vp, sz]
    lib.b200_vec_bit_reverse.argtypes = [i32, i32, vp, u32]
    lib.b200_vec_scale_powers.argtypes = [i32, i32, vp, sz, vp, vp]
    lib.b200_vec_batch_invert.argtypes = [i32, i32, vp, sz]
    lib.b200_plonk_constraints_coset.argtypes = [vp, vp, vp, vp]
    lib.b200_plonk_divide_by_zh.argtypes = [vp, u32, vp]
    lib.b200_vec_axpy.argtypes = [i32, i32, vp, vp, vp, sz]
    lib.b200_vec_scan.argtypes = [i32, i32, i32, vp, sz, i32]
    lib.b200_plonk_build_z.argtypes = [vp, vp, vp, vp, vp, vp, vp, vp]
    lib.b200_poly_eval.argtypes = [i32, i32, vp, sz, vp, vp]
    lib.b200_poly_div_by_linear.argtypes = [i32, i32, vp, sz, vp, vp]
    lib.b200_point_add_jac.argtypes = [i32, i32, vp, vp]
    lib.b200_point_to_affine.argtypes = [i32, i32, vp, vp]
    lib.b200_groth16_pk_load.argtypes = [i32, ctypes.POINTER(Groth16PkDesc), ctypes.POINTER(vp)]
    lib.b200_groth16_pk_free.argtypes = [vp]
    lib.b200_groth16_prove.argtypes = [vp, vp, vp, vp, vp, sz, vp, vp, vp, vp, vp, vp]
    lib.b200_groth16_msms.argtypes = [vp, vp, vp, vp, vp, sz, vp]
    lib.b200_groth16_assemble.argtypes = [vp, vp, vp, vp, vp, vp, vp]
    if "b200_groth16_prove_batch" not in missing:
        pp = ctypes.POINTER(vp)
        lib.b200_groth16_prove_batch.argtypes = [vp, sz, pp, pp, pp, pp, sz, vp, vp, vp, vp, vp, vp]
    if path is None:
        _lib = lib
    return lib


def check(rc: int):
    if rc != 0:
        raise B200Error(load().b200_last_error().decode())


def ptr(a) -> ctypes.c_void_p:
    """Host pointer of a numpy array / device pointer of a torch CUDA tensor / raw int."""
    if a is None:
        return ctypes.c_void_p(0)
    if isinstance(a, np.ndarray):
        assert a.flags["C_CONTIGUOUS"]
        return ctypes.c_void_p(a.ctypes.data)
    if hasattr(a, "data_ptr"):
        return ctypes.c_void_p(a.data_ptr())
    return ctypes.c_void_p(int(a))


def device_count() -> int:
    n = ctypes.c_int32(0)
    check(load().b200_device_count(ctypes.byref(n)))
    return n.value


def init(dev_ids=None):
    lib = load()
    if not dev_ids:
        check(lib.b200_init(0, None))
    else:
        arr = (ctypes.c_int32 * len(dev_ids))(*dev_ids)
        check(lib.b200_init(len(dev_ids), arr))


def comm_unique_id() -> np.ndarray:
    """128 opaque bytes (an NCCL unique id) created on rank 0; ship them to every rank, then comm_init."""
    out = np.zeros(COMM_ID_BYTES, dtype=np.uint8)
    check(load().b200_comm_unique_id(ptr(out)))
    return out


def comm_init(dev: int, world: int, rank: int, unique_id=None):
    """the library's own communicator for `dev` (one process per GPU); world == 1 clears it"""
    check(load().b200_comm_init(dev, world, rank, ptr(unique_id)))


def comm_init_torch(dev: int, pg=None):
    """one process per GPU under torch.distributed: rank 0's id is broadcast over the existing process group"""
    import torch
    import torch.distributed as dist
    world, rank = dist.get_world_size(pg), dist.get_rank(pg)
    if world == 1:
        comm_init(dev, 1, 0)
        return
    ident = comm_unique_id() if rank == 0 else np.zeros(COMM_ID_BYTES, dtype=np.uint8)
    t = torch.from_numpy(ident)
    if dist.get_backend(pg) == "nccl":
        t = t.cuda(dev)
    dist.broadcast(t, src=dist.get_global_rank(pg, 0) if pg is not None else 0, group=pg)
    comm_init(dev, world, rank, t.cpu().numpy())


def comm_init_all(dev_ids):
    arr = (ctypes.c_int32 * len(dev_ids))(*dev_ids)
    check(load().b200_comm_init_all(len(dev_ids), arr))


def comm_destroy(dev: int):
    check(load().b200_comm_destroy(dev))


def comm_info(dev: int):
    w, r = ctypes.c_int32(1), ctypes.c_int32(0)
    check(load().b200_comm_info(dev, ctypes.byref(w), ctypes.byref(r)))
    return w.value, r.value


def points_allreduce(dev: int, curve: int, group: int, d_partials, count: int, d_totals=None):
    """d_totals[k] = sum over ranks of d_partials[k] (device Jacobian points); in place when d_totals is None"""
    check(load().b200_points_allreduce(dev, curve, group, ptr(d_partials), count,
                                       ptr(d_totals if d_totals is not None else d_partials)))


def points_fold(dev: int, curve: int, group: int, d_gathered, world: int, count: int, d_totals):
    """d_totals[k] = sum_r d_gathered[r][k] on the device (the reduction half of points_allreduce)"""
    check(load().b200_points_fold(dev, curve, group, ptr(d_gathered), world, count, ptr(d_totals)))


def set_stream(dev: int, cuda_stream: int):
    check(load().b200_set_stream(dev, ctypes.c_void_p(cuda_stream)))


def sync(dev: int = 0):
    check(load().b200_sync(dev))


class Table:
    """Device-resident MSM base table (the reference's pinned G1Device / G2Device slices,
    backend/accelerated/icicle/groth16/bn254/provingkey.go)."""

    def __init__(self, curve: int, group: int, points, dev: int = 0, precomp: bool = True, n: int = None,
                 on_device: bool = False):
        self.curve, self.group, self.dev = curve, group, dev
        frl, fpl, deg = CURVE_SHAPES[curve]
        self.fr_limbs = frl
        self.coord_limbs = fpl * (deg if group == 2 else 1)
        if n is None:
            n = points.size // (2 * self.coord_limbs)
        self.n = n
        flags = (TABLE_PRECOMP if precomp else 0) | (TABLE_SRC_ON_DEVICE if on_device else 0)
        h = ctypes.c_void_p(0)
        check(load().b200_table_upload(dev, curve, group, ptr(points), n, flags, ctypes.byref(h)))
        self.handle = h

    @classmethod
    def from_file(cls, curve: int, group: int, path: str, byte_offset: int, n: int, dev: int = 0, precomp: bool = True):
        """n affine points read straight from a file region (a point slice of gnark's ProvingKey dump) into HBM."""
        t = cls.__new__(cls)
        t.curve, t.group, t.dev = curve, group, dev
        frl, fpl, deg = CURVE_SHAPES[curve]
        t.fr_limbs = frl
        t.coord_limbs = fpl * (deg if group == 2 else 1)
        t.n = n
        h = ctypes.c_void_p(0)
        check(load().b200_table_upload_file(dev, curve, group, os.fsencode(path), byte_offset, n,
                                            TABLE_PRECOMP if precomp else 0, ctypes.byref(h)))
        t.handle = h
        return t

    @classmethod
    def from_encoded(cls, curve: int, group: int, data: bytes, n: int, encoding: int, dev: int = 0, precomp: bool = True):
        """n points in gnark-crypto's serialised encoding (POINTS_RAW / POINTS_COMPRESSED), decoded on the device"""
        t = cls.__new__(cls)
        t.curve, t.group, t.dev = curve, group, dev
        frl, fpl, deg = CURVE_SHAPES[curve]
        t.fr_limbs = frl
        t.coord_limbs = fpl * (deg if group == 2 else 1)
        t.n = n
        buf = np.frombuffer(data, dtype=np.uint8).copy() if n else np.zeros(1, dtype=np.uint8)
        h = ctypes.c_void_p(0)
        check(load().b200_table_upload_encoded(dev, curve, group, ptr(buf), n, encoding, TABLE_PRECOMP if precomp else 0,
                                               ctypes.byref(h)))
        t.handle = h
        return t

    def info(self):
        n, c, w, p, b = ctypes.c_size_t(), ctypes.c_int32(), ctypes.c_int32(), ctypes.c_int32(), ctypes.c_size_t()
        check(load().b200_table_info(self.handle, ctypes.byref(n), ctypes.byref(c), ctypes.byref(w), ctypes.byref(p),
                                     ctypes.byref(b)))
        return {"n": n.value, "window_bits": c.value, "n_windows": w.value, "precomp": p.value,
                "device_bytes": b.value}

    def msm(self, scalars, off: int = 0, n: int = None, on_device: bool = False) -> np.ndarray:
        """sum scalars[i] * bases[off+i] -> Jacobian {X,Y,Z} (gnark layout, uint64 limbs)."""
        if n is None:
            n = (scalars.size if isinstance(scalars, np.ndarray) else scalars.numel()) // self.fr_limbs
        out = np.zeros(3 * self.coord_limbs, dtype=np.uint64)
        fn = load().b200_msm_g1 if self.group == 1 else load().b200_msm_g2
        check(fn(self.handle, off, n, ptr(scalars), 1 if on_device else 0, ptr(out)))
        return out

    def msm_allreduce(self, scalars, off: int = 0, n: int = None, on_device: bool = False) -> np.ndarray:
        """this rank's shard of a point-range-sharded MSM + the combine over the library's communicator: the full sum
        on every rank (b200_msm when there is no communicator)"""
        if n is None:
            n = (scalars.size if isinstance(scalars, np.ndarray) else scalars.numel()) // self.fr_limbs
        out = np.zeros(3 * self.coord_limbs, dtype=np.uint64)
        check(load().b200_msm_allreduce(self.handle, off, n, ptr(scalars), 1 if on_device else 0, ptr(out)))
        return out

    def msm_gather(self, idx, scalars, off: int = 0) -> np.ndarray:
        """sum_j scalars[idx[j]] * bases[off + j] (wire filtering on the device); idx: uint32 host array or int32/uint32
        device tensor, scalars: the full wire vector (host array or device tensor)"""
        idx_dev, sc_dev = hasattr(idx, "data_ptr"), hasattr(scalars, "data_ptr")
        n_idx = idx.numel() if idx_dev else idx.size
        n_sc = (scalars.numel() if sc_dev else scalars.size) // self.fr_limbs
        if not idx_dev:
            idx = np.ascontiguousarray(idx, dtype=np.uint32)
        out = np.zeros(3 * self.coord_limbs, dtype=np.uint64)
        check(load().b200_msm_gather(self.handle, off, ptr(idx), n_idx, 1 if idx_dev else 0, ptr(scalars), n_sc,
                                     1 if sc_dev else 0, ptr(out)))
        return out

    def msm_indexed(self, idx, scalars) -> np.ndarray:
        """sum_j scalars[j] * bases[idx[j]] -> Jacobian (gnark layout): the bases picked by index (any order, repeats
        allowed, each below the table's point count), e.g. kzg.Commit of a sparse Lagrange-form vector.  idx: uint32 host
        array or int32/uint32 device tensor; scalars: (len(idx), fr_limbs) host array or device tensor"""
        idx_dev, sc_dev = hasattr(idx, "data_ptr"), hasattr(scalars, "data_ptr")
        n = idx.numel() if idx_dev else np.asarray(idx).size
        if not idx_dev:
            idx = np.ascontiguousarray(idx, dtype=np.uint32)
        if not sc_dev:
            scalars = np.ascontiguousarray(scalars, dtype=np.uint64)
        n_sc = (scalars.numel() if sc_dev else scalars.size) // self.fr_limbs
        if n_sc != n:
            raise ValueError(f"msm_indexed: {n} indices and {n_sc} scalars")
        out = np.zeros(3 * self.coord_limbs, dtype=np.uint64)
        check(load().b200_msm_indexed(self.handle, ptr(idx), n, 1 if idx_dev else 0, ptr(scalars), 1 if sc_dev else 0,
                                      ptr(out)))
        return out

    def msm_batch(self, scalars, off: int = 0, n: int = None) -> np.ndarray:
        """out[b] = sum_i scalars[b, i] * bases[off + i] for every row b: several MSMs over one base range in one call
        (one pipeline for the whole batch).  scalars: (batch, n, fr_limbs) host array or contiguous device tensor,
        item-major; n defaults to the row length.  Returns (batch, 3 * coord_limbs) Jacobian points (gnark layout)."""
        sc_dev = hasattr(scalars, "data_ptr")
        if sc_dev:
            if not scalars.is_contiguous():
                raise ValueError("msm_batch: the device scalars must be contiguous")
            total = scalars.numel()
        else:
            scalars = np.ascontiguousarray(scalars, dtype=np.uint64)
            total = scalars.size
        batch = int(scalars.shape[0])
        if n is None:
            n = total // (batch * self.fr_limbs) if batch else 0
        if total != batch * n * self.fr_limbs:
            raise ValueError(f"msm_batch: {total} scalar words for {batch} rows of {n} scalars")
        out = np.zeros((batch, 3 * self.coord_limbs), dtype=np.uint64)
        check(load().b200_msm_batch(self.handle, off, n, batch, ptr(scalars), 1 if sc_dev else 0, ptr(out)))
        return out

    def kzg_open_batch(self, polys, points, on_device: bool = False):
        """kzg.Open of every row on this G1 SRS: polys (batch, n, fr_limbs) host array or contiguous device tensor
        (on_device), points (batch, fr_limbs) Montgomery, one per row.  Returns (values (batch, fr_limbs) = p_b(z_b),
        proofs (batch, 3 * coord_limbs) Jacobian commitments of (p_b - p_b(z_b)) / (X - z_b) over srs[0, n - 1))."""
        polys, batch, n = _poly_rows(polys, self.fr_limbs, on_device)
        points = _fr_rows(points, batch, self.fr_limbs, "kzg_open_batch: points")
        values = np.zeros((batch, self.fr_limbs), dtype=np.uint64)
        proofs = np.zeros((batch, 3 * self.coord_limbs), dtype=np.uint64)
        check(load().b200_kzg_open_batch(self.handle, ptr(polys), n, batch, 1 if on_device else 0, ptr(points),
                                         ptr(values), ptr(proofs)))
        return values, proofs

    def kzg_fold_open(self, polys, z, gamma, on_device: bool = False) -> np.ndarray:
        """kzg.BatchOpenSinglePoint's H: the Jacobian commitment of (f - f(z)) / (X - z), f = sum_b gamma^b polys[b];
        polys as for kzg_open_batch, z and gamma one fr.Element each (Montgomery)."""
        polys, batch, n = _poly_rows(polys, self.fr_limbs, on_device)
        z = _fr_rows(z, 1, self.fr_limbs, "kzg_fold_open: z")
        gamma = _fr_rows(gamma, 1, self.fr_limbs, "kzg_fold_open: gamma")
        out = np.zeros(3 * self.coord_limbs, dtype=np.uint64)
        check(load().b200_kzg_fold_open(self.handle, ptr(polys), n, batch, 1 if on_device else 0, ptr(z), ptr(gamma),
                                        ptr(out)))
        return out

    def msm_async(self, d_scalars, d_out, off: int = 0, n: int = None):
        check(load().b200_msm_async(self.handle, off, n, ptr(d_scalars), ptr(d_out)))

    def msm_pipelined(self, d_scalars, d_out, off: int = 0, n: int = None):
        """stream-ordered, tail overlapped with the next call; results valid after join()."""
        check(load().b200_msm_pipelined(self.handle, off, n, ptr(d_scalars), ptr(d_out)))

    def msm_submit(self, h_scalars, h_out, off: int = 0, n: int = None):
        """asynchronous MSM from PINNED host buffers (torch pinned tensors / b200_host_alloc memory); the result
        lands in h_out after sync(dev).  Consecutive submissions overlap upload, compute, tail and download."""
        if n is None:
            n = h_scalars.numel() // self.fr_limbs
        check(load().b200_msm_submit(self.handle, off, n, ptr(h_scalars), ptr(h_out)))

    def msm_submit_dev(self, h_scalars, d_out, off: int = 0, n: int = None):
        """msm_submit with the result left on the device (d_out: 3 * coord_limbs int64 of device memory)"""
        if n is None:
            n = h_scalars.numel() // self.fr_limbs
        check(load().b200_msm_submit_dev(self.handle, off, n, ptr(h_scalars), ptr(d_out)))

    def join(self):
        check(load().b200_msm_join(self.dev))

    MSM_STAGES = ("decompose", "sort", "offsets_scan", "accumulate", "combine", "reduce_chunks", "set_sum_finish")

    def msm_profile(self, d_scalars, d_out, off: int = 0, n: int = None) -> dict:
        ms = (ctypes.c_float * 7)()
        check(load().b200_msm_profile(self.handle, off, n, ptr(d_scalars), ptr(d_out), ms))
        return dict(zip(self.MSM_STAGES, [float(x) for x in ms]))

    def free(self):
        if self.handle:
            check(load().b200_table_free(self.handle))
            self.handle = None

    def __del__(self):
        try:
            self.free()
        except Exception:
            pass


class Domain:
    """Device-resident fft.Domain."""

    def __init__(self, curve: int, log2n: int, dev: int = 0, generator=None, coset_gen=None):
        self.curve, self.log2n, self.dev = curve, log2n, dev
        self.n = 1 << log2n
        self.fr_limbs = CURVE_SHAPES[curve][0]
        h = ctypes.c_void_p(0)
        check(load().b200_ntt_domain_new(dev, curve, log2n, ptr(generator), ptr(coset_gen), ctypes.byref(h)))
        self.handle = h

    def ntt(self, data, inverse=False, decimation=DIF, on_coset=False, on_device=False):
        check(load().b200_ntt(self.handle, ptr(data), 1 if on_device else 0, 1 if inverse else 0, decimation,
                              1 if on_coset else 0))
        return data

    def ntt_batch(self, data, inverse=False, decimation=DIF, on_coset=False, on_device=False):
        """In place on `batch` vectors of this domain's size in one call (item-major: batch * n * fr_limbs words, a
        host array or a contiguous device tensor), each transformed as ntt() would."""
        total = data.numel() if on_device else data.size
        per = self.n * self.fr_limbs
        if total % per:
            raise ValueError(f"ntt_batch: {total} words is not a whole number of {self.n}-element vectors")
        check(load().b200_ntt_batch(self.handle, ptr(data), total // per, 1 if on_device else 0, 1 if inverse else 0,
                                    decimation, 1 if on_coset else 0))
        return data

    def ntt_async(self, d_data, inverse=False, decimation=DIF, on_coset=False):
        check(load().b200_ntt_async(self.handle, ptr(d_data), 1 if inverse else 0, decimation, 1 if on_coset else 0))

    def points_ntt(self, points, group=1, inverse=True):
        """Group-element NTT of 2^log2n affine points of this domain's curve (kzg.ToLagrangeG1 for inverse=True:
        monomial SRS [tau^k]G -> Lagrange basis [L_i(tau)]G; inverse=False goes back), natural order in and out.
        A numpy array is transformed in a copy that is returned; a device tensor in place (and returned)."""
        on_dev = hasattr(points, "data_ptr")
        if not on_dev:
            points = np.array(points, dtype=np.uint64, order="C", copy=True)
        check(load().b200_points_ntt(self.handle, group, ptr(points), 1 if on_dev else 0, 1 if inverse else 0))
        return points

    def compute_h(self, a, b, c, length=None, on_device=False, out=None, out_on_device=False):
        if length is None:
            length = a.size // self.fr_limbs
        if out is None:
            out = np.zeros((self.n, self.fr_limbs), dtype=np.uint64)
        check(load().b200_groth16_compute_h(self.handle, ptr(a), ptr(b), ptr(c), length, 1 if on_device else 0,
                                            ptr(out), 1 if out_on_device else 0))
        return out

    def free(self):
        if self.handle:
            check(load().b200_ntt_domain_free(self.handle))
            self.handle = None

    def __del__(self):
        try:
            self.free()
        except Exception:
            pass


def fixed_base_batch(curve: int, group: int, base_affine: np.ndarray, scalars, n: int = None, dev: int = 0,
                     out=None) -> np.ndarray:
    """[k_i * base] as affine points (curve.BatchScalarMultiplicationG1/G2).  scalars / out: host numpy arrays or
    device tensors (anything with data_ptr()); returns out."""
    frl, fpl, deg = CURVE_SHAPES[curve]
    cl = fpl * (deg if group == 2 else 1)
    on_dev = hasattr(scalars, "data_ptr")
    if n is None:
        n = (scalars.numel() if on_dev else scalars.size) // frl
    if out is None:
        out = np.zeros((n, 2 * cl), dtype=np.uint64)
    check(load().b200_fixed_base_batch(dev, curve, group, ptr(base_affine), ptr(scalars), 1 if on_dev else 0, n,
                                       ptr(out), 1 if hasattr(out, "data_ptr") else 0))
    return out


def points_scale(curve: int, group: int, points, c, t=None, n: int = None, dev: int = 0):
    """points[i] <- (c * t^i) * points[i] in place (t None: t = 1), the point vectors of a Groth16 MPC contribution
    (mpcsetup phase1.go SrsCommons.update, phase2.go Phase2.update).  points: affine points in gnark layout, a host numpy
    array or a device tensor (anything with data_ptr()); c, t: one fr.Element each (Montgomery limbs).  Returns points."""
    frl, fpl, deg = CURVE_SHAPES[curve]
    cl = fpl * (deg if group == 2 else 1)
    on_dev = hasattr(points, "data_ptr")
    if n is None:
        n = (points.numel() if on_dev else points.size) // (2 * cl)
    c = np.ascontiguousarray(c, dtype=np.uint64)
    t = None if t is None else np.ascontiguousarray(t, dtype=np.uint64)
    check(load().b200_points_scale(dev, curve, group, ptr(points), n, 1 if on_dev else 0, ptr(c), ptr(t)))
    return points


def points_decode(curve: int, group: int, data, n: int, encoding: int, dev: int = 0, out=None):
    """n points in gnark-crypto's serialised encoding (POINTS_RAW / POINTS_COMPRESSED, fixed size per point) -> affine
    points in gnark layout, decoded on the device.  out: a host numpy array (default) or a device tensor; returns out."""
    frl, fpl, deg = CURVE_SHAPES[curve]
    cl = fpl * (deg if group == 2 else 1)
    if out is None:
        out = np.zeros((n, 2 * cl), dtype=np.uint64)
    buf = np.frombuffer(bytes(data), dtype=np.uint8).copy() if n else np.zeros(1, dtype=np.uint8)
    check(load().b200_points_decode(dev, curve, group, ptr(buf), n, encoding, ptr(out), 1 if hasattr(out, "data_ptr") else 0))
    return out


class PlonkKey:
    """device-resident PLONK proving key behind b200_plonk_pk_load / b200_plonk_prove (plonk_host.cu)"""

    def __init__(self, curve: int, log2n: int, ql, qr, qm, qo, qk, perm, srs_canonical, dev: int = 0, qcp=()):
        self.curve, self.log2n, self.dev = curve, log2n, dev
        self.n_qcp = len(qcp)
        frl, fpl, _ = CURVE_SHAPES[curve]
        self.fr_limbs, self.fp_limbs = frl, fpl
        keep = [np.ascontiguousarray(a, dtype=np.uint64) for a in (ql, qr, qm, qo, qk)]
        perm = np.ascontiguousarray(perm, dtype=np.int64)
        srs = np.ascontiguousarray(srs_canonical, dtype=np.uint64)
        d = PlonkPkDesc()
        d.log2n = log2n
        for k, a in zip(("ql", "qr", "qm", "qo", "qk"), keep):
            setattr(d, k, ptr(a).value)
        d.perm, d.srs_canonical = ptr(perm).value, ptr(srs).value
        qk_ = [np.ascontiguousarray(a, dtype=np.uint64) for a in qcp]
        qarr = (ctypes.c_void_p * max(1, len(qk_)))(*[ptr(a).value for a in qk_])
        d.n_qcp, d.qcp = len(qk_), ctypes.cast(qarr, ctypes.POINTER(ctypes.c_void_p))
        h = ctypes.c_void_p(0)
        check(load().b200_plonk_pk_load(dev, curve, ctypes.byref(d), ctypes.byref(h)))
        self.handle = h

    def prove(self, l, r, o, gamma, beta, alpha, zeta, v, bl, br, bo, bz, pi2=(), qk=None, hr=None):
        """all scalars: uint64 limb arrays (Montgomery); bl/br/bo: (2, limbs), bz: (3, limbs); pi2: one committed
        polynomial per BSB22 gate of the key; hr: (2, limbs) quotient-shard randomisers = StatisticalZK.  Returns (points (10, 3*fp_limbs) Jacobian, values (7 + n_qcp,
        fr_limbs)[, bsb22 digests (n_qcp, 3*fp_limbs)])."""
        args = [np.ascontiguousarray(a, dtype=np.uint64) for a in (l, r, o, gamma, beta, alpha, zeta, v, bl, br, bo, bz)]
        ch = PlonkChallenges()
        for k, a in zip(("gamma", "beta", "alpha", "zeta", "v", "bl", "br", "bo", "bz"), args[3:]):
            setattr(ch, k, ptr(a).value)
        if qk is not None:       # this proof's complete Qk (public inputs folded in), Lagrange / regular
            qk = np.ascontiguousarray(qk, dtype=np.uint64)
            ch.qk = ptr(qk).value
        if hr is not None:
            hr = np.ascontiguousarray(hr, dtype=np.uint64)
            ch.hr = ptr(hr).value
        pts = np.zeros((10, 3 * self.fp_limbs), dtype=np.uint64)
        vals = np.zeros((7 + self.n_qcp, self.fr_limbs), dtype=np.uint64)
        pk_ = [np.ascontiguousarray(a, dtype=np.uint64) for a in pi2]
        parr = (ctypes.c_void_p * max(1, len(pk_)))(*[ptr(a).value for a in pk_])
        bsb = np.zeros((max(1, self.n_qcp), 3 * self.fp_limbs), dtype=np.uint64)
        if self.n_qcp:
            if len(pk_) != self.n_qcp:
                raise ValueError("one committed polynomial per BSB22 gate of the key is required")
            ch.pi2, ch.out_bsb22 = ctypes.cast(parr, ctypes.POINTER(ctypes.c_void_p)), ptr(bsb).value
        check(load().b200_plonk_prove(self.handle, ptr(args[0]), ptr(args[1]), ptr(args[2]), ctypes.byref(ch), ptr(pts),
                                      ptr(vals)))
        return (pts, vals, bsb[:self.n_qcp]) if self.n_qcp else (pts, vals)

    STAGES = ("begin_lro", "commit_z", "quotient", "linearise", "batch_open")

    def last_stage_ms(self) -> dict:
        """wall-clock ms of the five stages of the last prove() on this key"""
        ms = (ctypes.c_double * 5)()
        check(load().b200_plonk_last_stage_ms(self.handle, ms))
        return dict(zip(self.STAGES, [float(x) for x in ms]))

    def free(self):
        if self.handle:
            check(load().b200_plonk_pk_free(self.handle))
            self.handle = None

    def __del__(self):
        try:
            self.free()
        except Exception:
            pass


class PedersenKey:
    """device-resident pedersen.ProvingKey{Basis, BasisExpSigma} of one Groth16 commitment (ProvingKey.CommitmentKeys[i])"""

    def __init__(self, curve: int, basis, basis_exp_sigma, dev: int = 0):
        self.curve, self.dev = curve, dev
        self.fr_limbs, self.fp_limbs, _ = CURVE_SHAPES[curve]
        basis = np.ascontiguousarray(basis, dtype=np.uint64)
        sig = np.ascontiguousarray(basis_exp_sigma, dtype=np.uint64)
        self.n = basis.size // (2 * self.fp_limbs)
        if sig.size != basis.size:
            raise ValueError("Basis and BasisExpSigma differ in length")
        h = ctypes.c_void_p(0)
        check(load().b200_pedersen_key_load(dev, curve, ptr(basis), ptr(sig), self.n, ctypes.byref(h)))
        self.handle = h

    def commit(self, values, want_commitment=True, want_pok=True):
        """(commitment, pok) as G1Affine limb arrays (None for the one not asked for): Commit (prove.go:84) and
        ProveKnowledge (prove.go:114) over one upload of the values"""
        on_dev = hasattr(values, "data_ptr")
        n = (values.numel() if on_dev else values.size) // self.fr_limbs
        cm = np.zeros(2 * self.fp_limbs, dtype=np.uint64) if want_commitment else None
        pok = np.zeros(2 * self.fp_limbs, dtype=np.uint64) if want_pok else None
        check(load().b200_pedersen_commit(self.handle, ptr(values), n, 1 if on_dev else 0, ptr(cm), ptr(pok)))
        return cm, pok

    def free(self):
        if self.handle:
            check(load().b200_pedersen_key_free(self.handle))
            self.handle = None

    def __del__(self):
        try:
            self.free()
        except Exception:
            pass


def pedersen_fold(curve: int, poks: np.ndarray, challenge: np.ndarray) -> np.ndarray:
    """ProofOfKnowledge.Fold (prove.go:127): sum_i challenge^i * poks[i]; host CPU"""
    fpl = CURVE_SHAPES[curve][1]
    poks = np.ascontiguousarray(poks, dtype=np.uint64)
    out = np.zeros(2 * fpl, dtype=np.uint64)
    check(load().b200_pedersen_fold(curve, ptr(poks), poks.size // (2 * fpl), ptr(challenge), ptr(out)))
    return out


def point_add_jac(curve: int, group: int, acc: np.ndarray, q: np.ndarray) -> np.ndarray:
    """acc += q on Jacobian points in gnark layout (host CPU; no device needed)."""
    check(load().b200_point_add_jac(curve, group, ptr(acc), ptr(q)))
    return acc


def point_to_affine(curve: int, group: int, p: np.ndarray) -> np.ndarray:
    out = np.zeros(p.size // 3 * 2, dtype=np.uint64)
    check(load().b200_point_to_affine(curve, group, ptr(p), ptr(out)))
    return out


# ---- vector ops / PLONK building blocks ----------------------------------------------------------
def vec_op(dev, curve, op, d_out, d_a, d_b, n):
    check(load().b200_vec_op(dev, curve, op, ptr(d_out), ptr(d_a), ptr(d_b), n))


def vec_bit_reverse(dev, curve, d_data, log2n):
    check(load().b200_vec_bit_reverse(dev, curve, ptr(d_data), log2n))


def vec_scale_powers(dev, curve, d_data, n, s_mont, g_mont):
    check(load().b200_vec_scale_powers(dev, curve, ptr(d_data), n, ptr(s_mont), ptr(g_mont)))


def vec_batch_invert(dev, curve, d_data, n):
    check(load().b200_vec_batch_invert(dev, curve, ptr(d_data), n))


class PlonkCosetArgs(ctypes.Structure):
    _fields_ = ([(k, ctypes.c_void_p) for k in ("l", "r", "o", "z", "s1", "s2", "s3", "ql", "qr", "qm", "qo", "qk",
                                                "alpha", "beta", "gamma", "bl", "br", "bo", "bz")]
                + [(k, ctypes.c_int32) for k in ("nbl", "nbr", "nbo", "nbz")]
                + [("coset_index", ctypes.c_uint32), ("rho", ctypes.c_uint32), ("out", ctypes.c_void_p)])


def plonk_constraints_coset(domain0: "Domain", big_coset_gen, big_gen, polys: dict, alpha, beta, gamma, blind: dict,
                            coset_index: int, rho: int, d_out):
    """polys: name -> device tensor (n fr.Elements on the current coset); blind: name -> host array or None."""
    a = PlonkCosetArgs()
    keep = []
    for k in ("l", "r", "o", "z", "s1", "s2", "s3", "ql", "qr", "qm", "qo", "qk"):
        setattr(a, k, ptr(polys[k]).value)
    for k, v in (("alpha", alpha), ("beta", beta), ("gamma", gamma)):
        setattr(a, k, ptr(v).value)
    frl = domain0.fr_limbs
    for k in ("l", "r", "o", "z"):
        b = blind.get(k)
        if b is None or b.size == 0:
            setattr(a, "b" + k, None)
            setattr(a, "nb" + k, 0)
        else:
            keep.append(b)
            setattr(a, "b" + k, ptr(b).value)
            setattr(a, "nb" + k, b.size // frl)
    a.coset_index, a.rho, a.out = coset_index, rho, ptr(d_out).value
    check(load().b200_plonk_constraints_coset(domain0.handle, ptr(big_coset_gen), ptr(big_gen), ctypes.byref(a)))


def plonk_bsb22_coset(domain0: "Domain", d_qcp, d_pi2, coset_index: int, rho: int, d_out):
    """BSB22 commitment gate: out[slot of point j] += qcp[j] * pi2[j] on one coset"""
    check(load().b200_plonk_bsb22_coset(domain0.handle, ptr(d_qcp), ptr(d_pi2), coset_index, rho, ptr(d_out)))


def plonk_divide_by_zh(domain1: "Domain", domain0_log2n: int, d_data):
    check(load().b200_plonk_divide_by_zh(domain1.handle, domain0_log2n, ptr(d_data)))


SCAN_PRODUCT, SCAN_SUM = 0, 1


def vec_scan(dev, curve, op, d_data, n, exclusive=False):
    check(load().b200_vec_scan(dev, curve, op, ptr(d_data), n, 1 if exclusive else 0))


def plonk_build_z(domain0: "Domain", d_l, d_r, d_o, d_perm, beta, gamma, d_z):
    check(load().b200_plonk_build_z(domain0.handle, ptr(d_l), ptr(d_r), ptr(d_o), ptr(d_perm), ptr(beta), ptr(gamma),
                                    ptr(d_z)))


def poly_eval(dev, curve, d_coeffs, n, x) -> np.ndarray:
    out = np.zeros(CURVE_SHAPES[curve][0], dtype=np.uint64)
    check(load().b200_poly_eval(dev, curve, ptr(d_coeffs), n, ptr(x), ptr(out)))
    return out


def _poly_rows(polys, fr_limbs, on_device):
    """(polys, batch, n) of a (batch, n, fr_limbs) host array or contiguous device tensor"""
    if on_device:
        if not polys.is_contiguous():
            raise ValueError("the device polynomials must be contiguous")
    else:
        polys = np.ascontiguousarray(polys, dtype=np.uint64)
    if len(polys.shape) != 3 or int(polys.shape[2]) != fr_limbs:
        raise ValueError(f"polynomials must be shaped (batch, n, {fr_limbs}), not {tuple(polys.shape)}")
    return polys, int(polys.shape[0]), int(polys.shape[1])


def _fr_rows(a, rows, fr_limbs, what):
    a = np.ascontiguousarray(a, dtype=np.uint64)
    if a.size != rows * fr_limbs:
        raise ValueError(f"{what}: {a.size} words for {rows} fr.Elements")
    return a


def poly_eval_batch(dev, curve, polys, points, on_device: bool = False) -> np.ndarray:
    """values[b] = polys[b](points[b]) for every row: polys (batch, n, fr_limbs) host array or contiguous device tensor
    (on_device), points (batch, fr_limbs) Montgomery on the host.  Returns (batch, fr_limbs)."""
    frl = CURVE_SHAPES[curve][0]
    polys, batch, n = _poly_rows(polys, frl, on_device)
    points = _fr_rows(points, batch, frl, "poly_eval_batch: points")
    out = np.zeros((batch, frl), dtype=np.uint64)
    check(load().b200_poly_eval_batch(dev, curve, ptr(polys), n, batch, 1 if on_device else 0, ptr(points), ptr(out)))
    return out


def poly_div_by_linear(dev, curve, d_coeffs, n, z) -> np.ndarray:
    """in place quotient; returns the claimed value p(z)"""
    out = np.zeros(CURVE_SHAPES[curve][0], dtype=np.uint64)
    check(load().b200_poly_div_by_linear(dev, curve, ptr(d_coeffs), n, ptr(z), ptr(out)))
    return out


def vec_axpy(dev, curve, d_y, a_mont, d_x, n):
    """y += a * x on device vectors"""
    check(load().b200_vec_axpy(dev, curve, ptr(d_y), ptr(a_mont), ptr(d_x), n))
