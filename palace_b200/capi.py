"""ctypes binding of the C ABI in include/b2p.h (libb2p.so, hand-written sm_90a kernels).

This is the only way Python reaches the product: there is no Python/NumPy/torch implementation of
any operator behind it and no CPU fallback. Loading fails loudly when the library has not been
built (``python -c 'import __graft_entry__ as g; g.build()'``) and every entry point fails when no
sm_90 GPU (H100) is present. torch is used by the callers only to own device memory and streams.
"""
from __future__ import annotations

import ctypes as C
import os

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_HERE, "libb2p.so")

CURLCURL, ND_MASS, CURLCURL_MASS, H1_DIFFUSION, ND_WEAKCURL, ND_MIXEDCURL = 0, 1, 2, 3, 4, 5
# Raviart-Thomas mass on hexahedra: p is the ND-equivalent order (RT_{p-1}), Gc is not read (may be None)
RT_MASS = 6

_lib = None


class B2PError(RuntimeError):
    pass


class OpDesc(C.Structure):
    _fields_ = [
        ("kind", C.c_int), ("p", C.c_int), ("ne", C.c_int), ("lsize", C.c_int64),
        ("idx", C.c_void_p), ("orient", C.c_void_p), ("dof_map", C.c_void_p),
        ("Bo", C.c_void_p), ("Bc", C.c_void_p), ("Gc", C.c_void_p),
        ("coeff_ctx", C.c_void_p), ("coeff_ctx_bytes", C.c_size_t), ("assemble_qdata", C.c_int),
    ]


def lib():
    global _lib
    if _lib is None:
        if not os.path.exists(LIB_PATH):
            raise B2PError(f"{LIB_PATH} not built: run __graft_entry__.build() (nvcc, sm_90a). No CPU fallback exists.")
        _lib = C.CDLL(LIB_PATH)
        _lib.b2p_last_error.restype = C.c_char_p
        _lib.b2p_last_error.argtypes = [C.c_void_p]
        _lib.b2p_op_lsize.restype = C.c_int64
        _lib.b2p_op_algorithmic_bytes.restype = C.c_int64
        for name in ("b2p_op_lsize", "b2p_op_algorithmic_bytes", "b2p_op_destroy", "b2p_geom_destroy", "b2p_ctx_destroy"):
            getattr(_lib, name).argtypes = [C.c_void_p]
        _lib.b2p_op_destroy.restype = None
        _lib.b2p_geom_destroy.restype = None
        _lib.b2p_ctx_destroy.restype = None
    return _lib


def _chk(rc, ctx=None):
    if rc != 0:
        msg = lib().b2p_last_error(ctx)
        raise B2PError(f"b2p error {rc}: {msg.decode() if msg else '?'}")


def _np(a, dtype):
    return np.ascontiguousarray(a, dtype=dtype)


def _ptr(a):
    return None if a is None else a.ctypes.data_as(C.c_void_p)


def _vp(x):
    """Device pointer of a torch tensor / int / None."""
    if x is None:
        return None
    if hasattr(x, "data_ptr"):
        return C.c_void_p(x.data_ptr())
    return C.c_void_p(int(x))


def _stream(stream):
    if stream is None:
        import torch

        return C.c_void_p(torch.cuda.current_stream().cuda_stream)
    return C.c_void_p(int(stream))


class Ctx:
    def __init__(self, device=0, nccl_uid=None, rank=0, nranks=1):
        h = C.c_void_p()
        if nranks > 1:
            buf = (C.c_char * 128).from_buffer_copy(bytes(nccl_uid))
            _chk(lib().b2p_ctx_create_dist(int(device), buf, int(rank), int(nranks), C.byref(h)))
        else:
            _chk(lib().b2p_ctx_create(int(device), C.byref(h)))
        self.h = h
        self.rank, self.nranks = rank, nranks

    @staticmethod
    def nccl_unique_id() -> bytes:
        buf = (C.c_char * 128)()
        _chk(lib().b2p_nccl_unique_id(buf))
        return bytes(buf)

    def close(self):
        if self.h:
            lib().b2p_ctx_destroy(self.h)
            self.h = None


class LaunchInfo(C.Structure):
    _fields_ = [
        ("kernel", C.c_char * 48), ("max_grid", C.c_int), ("grid", C.c_int), ("workers", C.c_int), ("elems_per_batch", C.c_int),
        ("batches", C.c_int64), ("seq", C.c_int64), ("geom", C.c_char * 8),
    ]


def last_launch(ctx: Ctx) -> dict:
    """The last persistent element kernel launched on ``ctx`` (b2p_ctx_last_launch): kernel name and form, max_grid (SM count x
    CTAs per SM), grid, workers per CTA, elems_per_batch, batches, seq (launches recorded so far) and geom, the geometry source
    ("qdata": stored per-point q-data, "nodes": evaluated from the vertices of a trilinear mesh)."""
    r = LaunchInfo()
    _chk(lib().b2p_ctx_last_launch(ctx.h, C.byref(r)), ctx.h)
    return {name: (getattr(r, name).decode() if name in ("kernel", "geom") else int(getattr(r, name))) for name, _ in LaunchInfo._fields_}


class DenseOpDesc(C.Structure):
    _fields_ = [
        ("kind", C.c_int), ("P", C.c_int), ("Q", C.c_int), ("ne", C.c_int), ("lsize", C.c_int64), ("idx", C.c_void_p),
        ("orient", C.c_void_p), ("curl_orient", C.c_void_p), ("interp", C.c_void_p), ("deriv", C.c_void_p),
        ("coeff_ctx", C.c_void_p), ("coeff_ctx_bytes", C.c_size_t),
    ]


class Geom:
    def __init__(self, ctx: Ctx, h):
        self.ctx, self.h = ctx, h

    @classmethod
    def general(cls, ctx, qdata):
        """Prebuilt q-data [ne][11][Q] for any element type (dense-basis operators)."""
        qdata = _np(qdata, np.float64)
        h = C.c_void_p()
        _chk(lib().b2p_geom_create_qdata_general(ctx.h, int(qdata.shape[0]), int(qdata.shape[2]), _ptr(qdata), C.byref(h)), ctx.h)
        g = cls(ctx, h)
        g.ne, g.q1d = qdata.shape[0], 0
        return g

    @classmethod
    def hex(cls, ctx, xe, attr, mesh_order, q1d, nodeB, nodeG, qw1d):
        xe = _np(xe, np.float64)
        attr = _np(attr, np.int32)
        nodeB, nodeG, qw1d = _np(nodeB, np.float64), _np(nodeG, np.float64), _np(qw1d, np.float64)
        h = C.c_void_p()
        _chk(lib().b2p_geom_create_hex(ctx.h, int(xe.shape[0]), int(mesh_order), int(q1d), _ptr(xe), _ptr(nodeB), _ptr(nodeG),
                                       _ptr(qw1d), _ptr(attr), C.byref(h)), ctx.h)
        g = cls(ctx, h)
        g.ne, g.q1d = xe.shape[0], q1d
        return g

    @classmethod
    def from_qdata(cls, ctx, qdata, q1d):
        qdata = _np(qdata, np.float64)
        h = C.c_void_p()
        _chk(lib().b2p_geom_create_qdata(ctx.h, int(qdata.shape[0]), int(q1d), _ptr(qdata), C.byref(h)), ctx.h)
        g = cls(ctx, h)
        g.ne, g.q1d = qdata.shape[0], q1d
        return g

    def qdata(self):
        out = np.empty((self.ne, 11, self.q1d ** 3))
        _chk(lib().b2p_geom_get_qdata(self.h, _ptr(out)), self.ctx.h)
        return out

    def close(self):
        if self.h:
            lib().b2p_geom_destroy(self.h)
            self.h = None


def _desc(kind, p, lsize, idx, orient, dof_map, Bo, Bc, Gc, coeff, assemble):
    keep = []
    d = OpDesc()
    d.kind, d.p = int(kind), int(p)
    idx = _np(idx, np.int32)
    d.ne, d.lsize = idx.shape[0], int(lsize)
    keep.append(idx)
    d.idx = _ptr(idx)
    for name, arr, dt in (("orient", orient, np.int8), ("dof_map", dof_map, np.int32), ("Bo", Bo, np.float64),
                          ("Bc", Bc, np.float64), ("Gc", Gc, np.float64)):
        if arr is not None:
            a = _np(arr, dt)
            keep.append(a)
            setattr(d, name, _ptr(a))
    if coeff is not None:
        c = _np(coeff, np.float64)
        keep.append(c)
        d.coeff_ctx = _ptr(c)
        d.coeff_ctx_bytes = c.nbytes
    d.assemble_qdata = int(bool(assemble))
    return d, keep


class Op:
    """One local partially assembled operator (a ceed::Operator sub-operator)."""

    def __init__(self, ctx, h, lsize):
        self.ctx, self.h, self.lsize = ctx, h, lsize

    @classmethod
    def create(cls, ctx, geom, kind, p, lsize, idx, orient, dof_map, Bo, Bc, Gc, coeff, assemble=False):
        d, keep = _desc(kind, p, lsize, idx, orient, dof_map, Bo, Bc, Gc, coeff, assemble)
        h = C.c_void_p()
        _chk(lib().b2p_op_create(ctx.h, geom.h, C.byref(d), C.byref(h)), ctx.h)
        return cls(ctx, h, lsize)

    @classmethod
    def create_dense(cls, ctx, geom, kind, lsize, idx, orient, interp, deriv, coeff, curl_orient=None, fine=None):
        """Dense-basis operator from FULL DofToQuad tables (native dof order)."""
        keep = []
        d = DenseOpDesc()
        idx = _np(idx, np.int32)
        d.kind, d.ne, d.P, d.lsize = int(kind), idx.shape[0], idx.shape[1], int(lsize)
        tab = deriv if deriv is not None else interp
        d.Q = int(np.asarray(tab).shape[1])
        for name, arr, dt in (("idx", idx, np.int32), ("orient", orient, np.int8), ("curl_orient", curl_orient, np.int8),
                              ("interp", interp, np.float64), ("deriv", deriv, np.float64)):
            if arr is not None:
                a = _np(arr, dt)
                keep.append(a)
                setattr(d, name, _ptr(a))
        h = C.c_void_p()
        if fine is not None:
            _chk(lib().b2p_op_coarsen_dense(fine.h, C.byref(d), C.byref(h)), ctx.h)
            return cls(ctx, h, lsize)
        c = _np(coeff, np.float64)
        d.coeff_ctx, d.coeff_ctx_bytes = _ptr(c), c.nbytes
        _chk(lib().b2p_op_create_dense(ctx.h, geom.h, C.byref(d), C.byref(h)), ctx.h)
        return cls(ctx, h, lsize)

    def coarsen_dense(self, lsize, idx, orient, interp, deriv, curl_orient=None):
        """Coarse level of a dense-basis operator: geometry, kind and coefficient of self, tables and restriction of the coarse
        space (tabulated at the same quadrature points)."""
        return Op.create_dense(self.ctx, None, 0, lsize, idx, orient, interp, deriv, None, curl_orient=curl_orient, fine=self)

    @classmethod
    def create_sum(cls, ctx, ops, coefs):
        """One operator for sum_t coefs[t] * ops[t] (ND terms on one geometry / space): one launch per apply."""
        n = len(ops)
        arr = (C.c_void_p * n)(*[o.h for o in ops])
        cf = _np(coefs, np.float64)
        h = C.c_void_p()
        _chk(lib().b2p_op_create_sum(ctx.h, n, arr, _ptr(cf), C.byref(h)), ctx.h)
        return cls(ctx, h, ops[0].lsize)

    def coarsen(self, p, lsize, idx, orient, dof_map, Bo, Bc, Gc):
        d, keep = _desc(0, p, lsize, idx, orient, dof_map, Bo, Bc, Gc, None, False)
        h = C.c_void_p()
        _chk(lib().b2p_op_coarsen(self.h, C.byref(d), C.byref(h)), self.ctx.h)
        return Op(self.ctx, h, lsize)

    def apply(self, x, y, stream=None):
        _chk(lib().b2p_op_apply(self.h, _vp(x), _vp(y), _stream(stream)), self.ctx.h)

    def apply_add(self, x, y, stream=None):
        _chk(lib().b2p_op_apply_add(self.h, _vp(x), _vp(y), _stream(stream)), self.ctx.h)

    def apply_add_ex(self, alpha, x, y, masked=False, simple_kernel=False, halfwarp_kernel=False, round1_kernel=False, cta_kernel=False,
                     transpose=False, stream=None):
        flags = ((1 if masked else 0) | (2 if simple_kernel else 0) | (4 if halfwarp_kernel else 0) | (8 if round1_kernel else 0)
                 | (16 if cta_kernel else 0) | (32 if transpose else 0))
        _chk(lib().b2p_op_apply_add_ex(self.h, C.c_double(alpha), _vp(x), _vp(y), flags, _stream(stream)), self.ctx.h)

    def apply_add_pair(self, alpha, x0, x1, y0, y1, masked=False, stream=None):
        _chk(lib().b2p_op_apply_add_pair(self.h, C.c_double(alpha), _vp(x0), _vp(x1), _vp(y0), _vp(y1), 1 if masked else 0,
                                         _stream(stream)), self.ctx.h)

    def apply_add_split(self, alpha, x, xg, y, yg, n_owned, e_begin, e_count, masked=False, halfwarp_kernel=False, round1_kernel=False,
                        cta_kernel=False, stream=None):
        _chk(lib().b2p_op_apply_add_split(self.h, C.c_double(alpha), _vp(x), _vp(xg), _vp(y), _vp(yg), C.c_int64(n_owned), int(e_begin),
                                          int(e_count), (1 if masked else 0) | (4 if halfwarp_kernel else 0) | (8 if round1_kernel else 0) | (16 if cta_kernel else 0),
                                          _stream(stream)), self.ctx.h)

    def set_essential(self, ess_ldofs):
        e = _np(ess_ldofs, np.int32)
        _chk(lib().b2p_op_set_essential(self.h, _ptr(e), C.c_int64(e.size)), self.ctx.h)

    def diag_add(self, d, stream=None):
        _chk(lib().b2p_op_diag_add(self.h, _vp(d), _stream(stream)), self.ctx.h)

    def set_coeff(self, coeff):
        c = _np(coeff, np.float64)
        _chk(lib().b2p_op_set_coeff(self.h, _ptr(c), C.c_size_t(c.nbytes)), self.ctx.h)

    def algorithmic_bytes(self):
        return int(lib().b2p_op_algorithmic_bytes(self.h))

    def close(self):
        if self.h:
            lib().b2p_op_destroy(self.h)
            self.h = None


# ------------------------------------------------------------------------------------------------
# Interpolators, halo exchange, true-dof operators and solvers (linear algebra layer of include/b2p.h)
# ------------------------------------------------------------------------------------------------


class InterpComp(C.Structure):
    _fields_ = [("in_off", C.c_int), ("in_n", C.c_int * 3), ("out_off", C.c_int), ("out_n", C.c_int * 3), ("A", C.c_void_p * 3)]


class InterpDesc(C.Structure):
    _fields_ = [
        ("ne", C.c_int), ("in_P", C.c_int), ("in_lsize", C.c_int64), ("in_idx", C.c_void_p), ("in_orient", C.c_void_p),
        ("in_dof_map", C.c_void_p), ("out_P", C.c_int), ("out_lsize", C.c_int64), ("out_idx", C.c_void_p),
        ("out_orient", C.c_void_p), ("out_dof_map", C.c_void_p), ("ncomp", C.c_int), ("comps", InterpComp * 3),
    ]


class DenseInterpDesc(C.Structure):
    _fields_ = [
        ("ne", C.c_int), ("in_P", C.c_int), ("out_P", C.c_int), ("in_lsize", C.c_int64), ("out_lsize", C.c_int64),
        ("in_idx", C.c_void_p), ("in_orient", C.c_void_p), ("in_curl_orient", C.c_void_p), ("out_idx", C.c_void_p),
        ("out_orient", C.c_void_p), ("out_curl_orient", C.c_void_p), ("mat", C.c_void_p),
    ]


class CurlInterpDesc(C.Structure):
    _fields_ = [
        ("ne", C.c_int), ("p", C.c_int), ("nd_lsize", C.c_int64), ("nd_idx", C.c_void_p), ("nd_orient", C.c_void_p),
        ("nd_dof_map", C.c_void_p), ("rt_lsize", C.c_int64), ("rt_idx", C.c_void_p), ("rt_orient", C.c_void_p),
        ("rt_dof_map", C.c_void_p), ("D", C.c_void_p),
    ]


class Interp:
    """Element-local tensor interpolator between two hex spaces (p-prolongation, discrete gradient, discrete curl)."""

    def __init__(self, ctx, in_space, out_space, comps):
        """in_space/out_space: dicts(P, lsize, idx, orient, dof_map); comps: list of
        dict(in_off, in_n, out_off, out_n, A=[Ax, Ay, Az])."""
        keep = []
        d = InterpDesc()
        for pre, sp in (("in", in_space), ("out", out_space)):
            idx = _np(sp["idx"], np.int32)
            keep.append(idx)
            setattr(d, pre + "_P", int(sp["P"]))
            setattr(d, pre + "_lsize", int(sp["lsize"]))
            setattr(d, pre + "_idx", _ptr(idx))
            if sp.get("orient") is not None:
                o = _np(sp["orient"], np.int8)
                keep.append(o)
                setattr(d, pre + "_orient", _ptr(o))
            if sp.get("dof_map") is not None:
                m = _np(sp["dof_map"], np.int32)
                keep.append(m)
                setattr(d, pre + "_dof_map", _ptr(m))
        d.ne = _np(in_space["idx"], np.int32).shape[0]
        d.ncomp = len(comps)
        for c, cc in enumerate(comps):
            d.comps[c].in_off, d.comps[c].out_off = int(cc["in_off"]), int(cc["out_off"])
            for a in range(3):
                d.comps[c].in_n[a], d.comps[c].out_n[a] = int(cc["in_n"][a]), int(cc["out_n"][a])
                A = _np(cc["A"][a], np.float64)
                assert A.shape == (cc["out_n"][a], cc["in_n"][a])
                keep.append(A)
                d.comps[c].A[a] = A.ctypes.data
        h = C.c_void_p()
        _chk(lib().b2p_interp_create(ctx.h, C.byref(d), C.byref(h)), ctx.h)
        self.ctx, self.h = ctx, h
        self.in_lsize, self.out_lsize = int(in_space["lsize"]), int(out_space["lsize"])

    @classmethod
    def dense(cls, ctx, mat, in_idx, in_lsize, out_idx, out_lsize, in_orient=None, in_curl_orient=None, out_orient=None,
              out_curl_orient=None):
        """Element-dense interpolator (any element type): one [out_P][in_P] matrix, native dof order."""
        d = DenseInterpDesc()
        keep = []
        mat = _np(mat, np.float64)
        in_idx, out_idx = _np(in_idx, np.int32), _np(out_idx, np.int32)
        assert mat.shape == (out_idx.shape[1], in_idx.shape[1]) and in_idx.shape[0] == out_idx.shape[0]
        d.ne, d.in_P, d.out_P = in_idx.shape[0], in_idx.shape[1], out_idx.shape[1]
        d.in_lsize, d.out_lsize = int(in_lsize), int(out_lsize)
        d.in_idx, d.out_idx, d.mat = _ptr(in_idx), _ptr(out_idx), _ptr(mat)
        for name, arr in (("in_orient", in_orient), ("in_curl_orient", in_curl_orient), ("out_orient", out_orient),
                          ("out_curl_orient", out_curl_orient)):
            if arr is not None:
                a = _np(arr, np.int8)
                keep.append(a)
                setattr(d, name, _ptr(a))
        h = C.c_void_p()
        _chk(lib().b2p_interp_create_dense(ctx.h, C.byref(d), C.byref(h)), ctx.h)
        self = cls.__new__(cls)
        self.ctx, self.h = ctx, h
        self.in_lsize, self.out_lsize = int(in_lsize), int(out_lsize)
        return self

    @classmethod
    def curl_hex(cls, ctx, nd_space, rt_space, p):
        """Discrete curl ND_p -> RT_{p-1} on hexahedra (sum-factorised, b2p_interp_create_curl_hex): Mult gives B = curl E on the
        RT dofs. nd_space / rt_space: dicts of host.assemble.space_dict."""
        from .host import assemble as asm

        p = int(p)
        d = CurlInterpDesc()
        keep = []
        ne = np.shape(nd_space["idx"])[0]
        for pre, sp, P in (("nd", nd_space, 3 * p * (p + 1) ** 2), ("rt", rt_space, 3 * p * p * (p + 1))):
            idx = _np(sp["idx"], np.int32)
            if idx.shape != (ne, P):
                raise ValueError(f"curl_hex: {pre} idx has shape {idx.shape}, expected ({ne}, {P}) for p={p}")
            keep.append(idx)
            setattr(d, pre + "_lsize", int(sp["lsize"]))
            setattr(d, pre + "_idx", _ptr(idx))
            for key, dtype, shape in (("orient", np.int8, (ne, P)), ("dof_map", np.int32, (P,))):
                if sp.get(key) is not None:
                    a = _np(sp[key], dtype)
                    if a.shape != shape:
                        raise ValueError(f"curl_hex: {pre} {key} has shape {a.shape}, expected {shape}")
                    keep.append(a)
                    setattr(d, f"{pre}_{key}", _ptr(a))
        D = _np(asm.curl_table(p), np.float64)
        d.ne, d.p, d.D = ne, p, _ptr(D)
        h = C.c_void_p()
        _chk(lib().b2p_interp_create_curl_hex(ctx.h, C.byref(d), C.byref(h)), ctx.h)
        self = cls.__new__(cls)
        self.ctx, self.h = ctx, h
        self.in_lsize, self.out_lsize = int(nd_space["lsize"]), int(rt_space["lsize"])
        return self

    def apply_add(self, x, y, transpose=False, alpha=1.0, stream=None):
        _chk(lib().b2p_interp_apply_add(self.h, int(transpose), C.c_double(alpha), _vp(x), _vp(y), _stream(stream)), self.ctx.h)


class Halo:
    def __init__(self, ctx, n_true, n_ghost, nbr_ranks, send_counts, send_idx, recv_counts):
        nbr = _np(nbr_ranks, np.int32)
        sc, rc = _np(send_counts, np.int64), _np(recv_counts, np.int64)
        si = _np(send_idx, np.int32)
        h = C.c_void_p()
        _chk(lib().b2p_halo_create(ctx.h, C.c_int64(n_true), C.c_int64(n_ghost), int(nbr.size), _ptr(nbr), _ptr(sc), _ptr(si), _ptr(rc),
                                   C.byref(h)), ctx.h)
        self.ctx, self.h = ctx, h

    def enable_p2p(self, all_gather):
        """Switch ParOperator::Mult's exchange to peer-memory stores. ``all_gather(bytes) -> list[bytes]``
        gathers one blob per rank (e.g. torch.distributed.all_gather_object)."""
        n = C.c_size_t()
        _chk(lib().b2p_halo_p2p_export(self.h, None, C.byref(n)), self.ctx.h)
        buf = (C.c_char * n.value)()
        _chk(lib().b2p_halo_p2p_export(self.h, buf, C.byref(n)), self.ctx.h)
        blobs = all_gather(bytes(buf))
        allb = b"".join(blobs)
        arr = (C.c_char * len(allb)).from_buffer_copy(allb)
        _chk(lib().b2p_halo_p2p_import(self.h, arr, C.c_size_t(n.value), len(blobs)), self.ctx.h)

    def forward(self, lvec):
        _chk(lib().b2p_halo_forward(self.h, _vp(lvec)), self.ctx.h)

    def reverse(self, lvec):
        _chk(lib().b2p_halo_reverse(self.h, _vp(lvec)), self.ctx.h)


class Csr:
    """Fully assembled device CSR matrix of a sum of local operators (coarse levels; BilinearForm::FullAssemble)."""

    def __init__(self, ctx, op: Op):
        self.ctx = ctx
        h = C.c_void_p()
        _chk(lib().b2p_csr_create(ctx.h, op.h, C.byref(h)), ctx.h)
        self.h = h
        lib().b2p_csr_rows.restype = C.c_int64
        lib().b2p_csr_nnz.restype = C.c_int64
        self.n, self.nnz = int(lib().b2p_csr_rows(h)), int(lib().b2p_csr_nnz(h))

    def assemble(self, ops, coefs=None, stream=None):
        n = len(ops)
        arr = (C.c_void_p * n)(*[o.h for o in ops])
        cf = _np(coefs if coefs is not None else np.ones(n), np.float64)
        _chk(lib().b2p_csr_assemble(self.h, n, arr, _ptr(cf), _stream(stream)), self.ctx.h)

    def eliminate(self, ess_dofs, diag_policy=1, stream=None):
        ess = _np(ess_dofs, np.int32)
        _chk(lib().b2p_csr_eliminate(self.h, _ptr(ess), C.c_int64(ess.size), int(diag_policy), _stream(stream)), self.ctx.h)

    def mult(self, x, y, stream=None):
        _chk(lib().b2p_csr_mult(self.h, _vp(x), _vp(y), _stream(stream)), self.ctx.h)

    def diag(self, d, stream=None):
        _chk(lib().b2p_csr_diag(self.h, _vp(d), _stream(stream)), self.ctx.h)

    def to_scipy(self, stream=None):
        import scipy.sparse as sp

        rowptr, col, val = np.empty(self.n + 1, np.int32), np.empty(self.nnz, np.int32), np.empty(self.nnz)
        _chk(lib().b2p_csr_get_host(self.h, _ptr(rowptr), _ptr(col), _ptr(val), _stream(stream)), self.ctx.h)
        return sp.csr_matrix((val, col, rowptr), shape=(self.n, self.n))

    def close(self):
        if self.h:
            lib().b2p_csr_destroy.restype = None
            lib().b2p_csr_destroy(self.h)
            self.h = None


def _device_view(ptr, n, ctype):
    """1-D tensor viewing n elements of library-owned device memory (no copy)."""
    import torch

    dtype = np.dtype(ctype)
    if torch.cuda.device_count() > 0:
        class _Cai:  # __cuda_array_interface__ lets torch wrap a raw device pointer
            pass

        o = _Cai()
        o.__cuda_array_interface__ = {"shape": (int(n),), "typestr": dtype.str, "data": (int(ptr or 0), False), "version": 2}
        return torch.as_tensor(o, device="cuda")
    # no CUDA device: the library is the host-thread emulation build, whose device memory is host memory
    return torch.from_numpy(np.ctypeslib.as_array(C.cast(ptr, C.POINTER(ctype)), shape=(int(n),)))


def set_stream(ctx, stream=None):
    _chk(lib().b2p_ctx_set_stream(ctx.h, _stream(stream)), ctx.h)


def vec_dot(ctx, x, y):
    out = C.c_double()
    _chk(lib().b2p_vec_dot(ctx.h, C.c_int64(x.numel()), _vp(x), _vp(y), C.byref(out)), ctx.h)
    return out.value


def vec_sum(ctx, x):
    out = C.c_double()
    _chk(lib().b2p_vec_sum(ctx.h, C.c_int64(x.numel()), _vp(x), C.byref(out)), ctx.h)
    return out.value


def vec_axpby(ctx, a, x, b, y):
    _chk(lib().b2p_vec_axpby(ctx.h, C.c_int64(x.numel()), C.c_double(a), _vp(x), C.c_double(b), _vp(y)), ctx.h)


def vec_axpbypcz(ctx, a, x, b, y, g, z):
    _chk(lib().b2p_vec_axpbypcz(ctx.h, C.c_int64(x.numel()), C.c_double(a), _vp(x), C.c_double(b), _vp(y), C.c_double(g), _vp(z)), ctx.h)


def vec_orthogonalize(ctx, kind, V, w):
    """Gram-Schmidt of w against the list V (0 MGS, 1 CGS, 2 CGS2); returns H (numpy)."""
    m = len(V)
    ptrs = (C.c_void_p * m)(*[v.data_ptr() for v in V])
    H = np.zeros(m)
    _chk(lib().b2p_vec_orthogonalize(ctx.h, int(kind), C.c_int64(w.numel()), m, ptrs, _vp(w), _ptr(H)), ctx.h)
    return H


class Operator:
    """True-dof operator handle (ParOperator / interpolator)."""

    def __init__(self, ctx, h):
        self.ctx, self.h = ctx, h

    @classmethod
    def par(cls, ctx, tsize, lsize, ops, coefs=None, ess_tdofs=None, diag_policy=1, halo=None):
        n = len(ops)
        arr = (C.c_void_p * n)(*[o.h for o in ops])
        cf = _np(coefs if coefs is not None else np.ones(n), np.float64)
        ess = _np(ess_tdofs if ess_tdofs is not None else np.zeros(0), np.int32)
        h = C.c_void_p()
        _chk(lib().b2p_operator_par(ctx.h, C.c_int64(tsize), C.c_int64(lsize), n, arr, _ptr(cf), _ptr(ess), C.c_int64(ess.size),
                                    int(diag_policy), halo.h if halo else None, C.byref(h)), ctx.h)
        o = cls(ctx, h)
        o._keep = list(ops)
        return o

    @classmethod
    def from_csr(cls, ctx, csr):
        """The assembled matrix behind the operator interface (coarse-level solvers); csr must outlive it."""
        h = C.c_void_p()
        _chk(lib().b2p_operator_csr(ctx.h, csr.h, C.byref(h)), ctx.h)
        o = cls(ctx, h)
        o._csr = csr
        return o

    def is_fused(self):
        return int(lib().b2p_operator_par_is_fused(self.h)) == 1

    def set_coefficients(self, coefs):
        cf = _np(coefs, np.float64)
        _chk(lib().b2p_operator_par_set_coefficients(self.h, int(cf.size), _ptr(cf)), self.ctx.h)

    def set_interior(self, ne_interior):
        _chk(lib().b2p_operator_par_set_interior(self.h, int(ne_interior)), self.ctx.h)

    @classmethod
    def interp(cls, ctx, it: Interp, in_halo=None, in_tsize=0, out_halo=None, out_tsize=0):
        h = C.c_void_p()
        _chk(lib().b2p_operator_interp(ctx.h, it.h, in_halo.h if in_halo else None, C.c_int64(in_tsize),
                                       out_halo.h if out_halo else None, C.c_int64(out_tsize), C.byref(h)), ctx.h)
        o = cls(ctx, h)
        o._keep = [it]
        return o

    def mult(self, x, y):
        _chk(lib().b2p_operator_mult(self.h, _vp(x), _vp(y)), self.ctx.h)

    def mult_transpose(self, x, y):
        _chk(lib().b2p_operator_mult_transpose(self.h, _vp(x), _vp(y)), self.ctx.h)

    def add_mult(self, x, y, a=1.0):
        _chk(lib().b2p_operator_add_mult(self.h, _vp(x), _vp(y), C.c_double(a)), self.ctx.h)

    def assemble_diagonal(self, d):
        _chk(lib().b2p_operator_assemble_diagonal(self.h, _vp(d)), self.ctx.h)

    @property
    def height(self):
        lib().b2p_operator_height.restype = C.c_int64
        return int(lib().b2p_operator_height(self.h))


class SpMat:
    """Device CSR matrix with its transpose (b2p_spmat): the prolongation of a non-conforming space."""

    def __init__(self, ctx, A):
        import scipy.sparse as sp

        A = sp.csr_matrix(A)
        A.sort_indices()
        self.ctx, self.shape = ctx, A.shape
        rp, cl, vl = _np(A.indptr, np.int32), _np(A.indices, np.int32), _np(A.data, np.float64)
        self.h = C.c_void_p()
        _chk(lib().b2p_spmat_create(ctx.h, C.c_int64(A.shape[0]), C.c_int64(A.shape[1]), _ptr(rp), _ptr(cl), _ptr(vl), C.byref(self.h)),
             ctx.h)

    def mult(self, x, y, transpose=False):
        _chk(lib().b2p_spmat_mult(self.h, 1 if transpose else 0, _vp(x), _vp(y)), self.ctx.h)

    def __del__(self):
        try:
            lib().b2p_spmat_destroy(self.h)
        except Exception:
            pass


def operator_rap(ctx, A_local, P: SpMat, ess_tdofs=None, diag_policy=1):
    """ParOperator with a general prolongation: P^T A_local P with essential true dofs (b2p_operator_rap)."""
    ess = _np(ess_tdofs if ess_tdofs is not None else np.zeros(0), np.int32)
    h = C.c_void_p()
    _chk(lib().b2p_operator_rap(ctx.h, A_local.h, P.h, _ptr(ess), C.c_int64(ess.size), int(diag_policy), C.byref(h)), ctx.h)
    o = Operator(ctx, h)
    o._keep = [A_local, P]
    return o


def operator_triple(ctx, L, A_mid, R):
    """y = L A_mid R x with sparse L / R (SpMat or None): b2p_operator_triple."""
    h = C.c_void_p()
    _chk(lib().b2p_operator_triple(ctx.h, L.h if L is not None else None, A_mid.h, R.h if R is not None else None, C.byref(h)), ctx.h)
    o = Operator(ctx, h)
    o._keep = [L, A_mid, R]
    return o


CG, GMRES, FGMRES = 0, 1, 2
MGS, CGS, CGS2 = 0, 1, 2
PC_RIGHT, PC_LEFT = 0, 1


class Solver:
    def __init__(self, ctx, h):
        self.ctx, self.h = ctx, h
        self._keep = []

    @classmethod
    def jacobi(cls, ctx, omega=1.0, sf_max=1.0):
        h = C.c_void_p()
        _chk(lib().b2p_solver_jacobi(ctx.h, C.c_double(omega), C.c_double(sf_max), C.byref(h)), ctx.h)
        return cls(ctx, h)

    @classmethod
    def chebyshev(cls, ctx, smooth_it=1, order=4, sf_max=1.0, sf_min=0.0, fourth_kind=True):
        h = C.c_void_p()
        _chk(lib().b2p_solver_chebyshev(ctx.h, smooth_it, order, C.c_double(sf_max), C.c_double(sf_min), int(fourth_kind), C.byref(h)), ctx.h)
        return cls(ctx, h)

    @classmethod
    def distrelax(cls, ctx, G: Operator, smooth_it=1, cheby_smooth_it=1, cheby_order=4, sf_max=1.0, sf_min=0.0, fourth_kind=True):
        h = C.c_void_p()
        _chk(lib().b2p_solver_distrelax(ctx.h, G.h, smooth_it, cheby_smooth_it, cheby_order, C.c_double(sf_max), C.c_double(sf_min),
                                        int(fourth_kind), C.byref(h)), ctx.h)
        s = cls(ctx, h)
        s._keep.append(G)
        return s

    def distrelax_set_operators(self, A: Operator, A_G: Operator):
        self._keep += [A, A_G]
        _chk(lib().b2p_solver_distrelax_set_operators(self.h, A.h, A_G.h), self.ctx.h)

    @classmethod
    def gmg(cls, ctx, coarse, P, G=None, cycle_it=1, smooth_it=1, cheby_order=4, sf_max=1.0, sf_min=0.0, fourth_kind=True):
        n_levels = len(P) + 1
        Parr = (C.c_void_p * max(1, len(P)))(*[p.h for p in P])
        Garr = None
        if G is not None:
            Garr = (C.c_void_p * n_levels)(*[(g.h if g is not None else None) for g in G])
        h = C.c_void_p()
        _chk(lib().b2p_solver_gmg(ctx.h, coarse.h, n_levels, Parr, Garr, cycle_it, smooth_it, cheby_order, C.c_double(sf_max),
                                  C.c_double(sf_min), int(fourth_kind), C.byref(h)), ctx.h)
        s = cls(ctx, h)
        s._keep += [coarse, list(P), G]
        s.n_levels = n_levels
        return s

    def gmg_set_operators(self, A, A_aux=None):
        n = len(A)
        Aarr = (C.c_void_p * n)(*[a.h for a in A])
        Garr = None
        if A_aux is not None:
            Garr = (C.c_void_p * n)(*[(a.h if a is not None else None) for a in A_aux])
        self._keep += [list(A), A_aux]
        _chk(lib().b2p_solver_gmg_set_operators(self.h, Aarr, Garr), self.ctx.h)

    @classmethod
    def krylov(cls, ctx, kind, rel_tol=1e-6, abs_tol=0.0, max_it=100, max_dim=-1, orthog=MGS, pc_side=PC_RIGHT):
        h = C.c_void_p()
        _chk(lib().b2p_solver_krylov(ctx.h, int(kind), C.byref(h)), ctx.h)
        s = cls(ctx, h)
        _chk(lib().b2p_solver_krylov_config(h, C.c_double(rel_tol), C.c_double(abs_tol), int(max_it), int(max_dim), int(orthog),
                                            int(pc_side)), ctx.h)
        return s

    @classmethod
    def assembled(cls, ctx, inner, inner_pc=None):
        """Coarse solver on the device-assembled matrix of the ParOperator given to set_operator (MfemWrapperSolver)."""
        h = C.c_void_p()
        _chk(lib().b2p_solver_assembled(ctx.h, inner.h, inner_pc.h if inner_pc is not None else None, C.byref(h)), ctx.h)
        s = cls(ctx, h)
        s._keep += [inner, inner_pc]
        return s

    def assembled_nnz(self):
        lib().b2p_solver_assembled_nnz.restype = C.c_int64
        return int(lib().b2p_solver_assembled_nnz(self.h))

    @classmethod
    def amg(cls, ctx, cycle_it=1, smooth_it=1):
        """Smoothed-aggregation AMG on an assembled matrix (set_operator: Operator.from_csr, or wrap it in Solver.assembled)."""
        h = C.c_void_p()
        _chk(lib().b2p_solver_amg(ctx.h, int(cycle_it), int(smooth_it), C.byref(h)), ctx.h)
        return cls(ctx, h)

    @classmethod
    def ams(cls, ctx, G, coords, cycle_it=1, smooth_it=1, singular=False):
        """AMS (cycle type 14) for the eliminated ND p = 1 matrix; G: scipy sparse discrete gradient [n_edges x n_vertices] (entries
        +-1), coords: [n_vertices, 3] vertex coordinates."""
        import scipy.sparse as sp

        G = sp.csr_matrix(G)
        G.sum_duplicates()
        G.sort_indices()
        rp, col, val = _np(G.indptr, np.int32), _np(G.indices, np.int32), _np(G.data, np.float64)
        X = _np(coords, np.float64).reshape(-1, 3)
        h = C.c_void_p()
        _chk(lib().b2p_solver_ams(ctx.h, int(cycle_it), int(smooth_it), int(bool(singular)), C.c_int64(G.shape[0]), C.c_int64(X.shape[0]),
                                  _ptr(rp), _ptr(col), _ptr(val), _ptr(X), C.byref(h)), ctx.h)
        return cls(ctx, h)

    def levels(self, hierarchy=0):
        """(rows, nnz) per level of an AMG / AMS hierarchy (AMS: 0 = G, 1-3 = Pi_x, Pi_y, Pi_z) of this solver, of the inner solver
        of Solver.assembled, or of either as a multigrid's coarse solver."""
        rows, nnz = (C.c_int64 * 16)(), (C.c_int64 * 16)()
        n = lib().b2p_solver_amg_levels(self.h, int(hierarchy), rows, nnz, 16)
        if n < 0:
            raise B2PError(f"b2p_solver_amg_levels: no hierarchy {hierarchy} on this solver")
        return list(rows[:n]), list(nnz[:n])

    def setup_ms(self):
        lib().b2p_solver_amg_setup_ms.restype = C.c_double
        return float(lib().b2p_solver_amg_setup_ms(self.h))

    def set_check_interval(self, check_every):
        _chk(lib().b2p_solver_krylov_set_check_interval(self.h, int(check_every)), self.ctx.h)

    def set_preconditioner(self, pc):
        self._keep.append(pc)
        _chk(lib().b2p_solver_set_preconditioner(self.h, pc.h if pc else None), self.ctx.h)

    def set_operator(self, A: Operator):
        self._keep.append(A)
        _chk(lib().b2p_solver_set_operator(self.h, A.h), self.ctx.h)

    def set_initial_guess(self, flag):
        _chk(lib().b2p_solver_set_initial_guess(self.h, int(flag)), self.ctx.h)

    def mult(self, x, y):
        _chk(lib().b2p_solver_mult(self.h, _vp(x), _vp(y)), self.ctx.h)

    def mult2(self, x, y, r):
        _chk(lib().b2p_solver_mult2(self.h, _vp(x), _vp(y), _vp(r)), self.ctx.h)

    def mult_transpose2(self, x, y, r):
        _chk(lib().b2p_solver_mult_transpose2(self.h, _vp(x), _vp(y), _vp(r)), self.ctx.h)

    def stats(self):
        its, conv = C.c_int(), C.c_int()
        r0, r1 = C.c_double(), C.c_double()
        _chk(lib().b2p_solver_stats(self.h, C.byref(its), C.byref(r0), C.byref(r1), C.byref(conv)), self.ctx.h)
        return dict(its=its.value, initial_res=r0.value, final_res=r1.value, converged=bool(conv.value))

    def lambda_max(self):
        out = C.c_double()
        _chk(lib().b2p_solver_lambda_max(self.h, C.byref(out)), self.ctx.h)
        return out.value


# ------------------------------------------------------------------------------------------------
# Complex operators / solvers on split (real, imag) vectors
# ------------------------------------------------------------------------------------------------


def vec_cdot(ctx, xr, xi, yr, yi):
    out = (C.c_double * 2)()
    _chk(lib().b2p_vec_cdot(ctx.h, C.c_int64(xr.numel()), _vp(xr), _vp(xi), _vp(yr), _vp(yi), out), ctx.h)
    return complex(out[0], out[1])


def vec_caxpy(ctx, a, xr, xi, yr, yi):
    a = complex(a)
    _chk(lib().b2p_vec_caxpy(ctx.h, C.c_int64(xr.numel()), C.c_double(a.real), C.c_double(a.imag), _vp(xr), _vp(xi), _vp(yr), _vp(yi)), ctx.h)


class ComplexOperator:
    def __init__(self, ctx, h):
        self.ctx, self.h = ctx, h

    @classmethod
    def par(cls, ctx, tsize, lsize, ops, coefs, ess_tdofs=None, diag_policy=1):
        n = len(ops)
        arr = (C.c_void_p * n)(*[o.h for o in ops])
        cr = _np([complex(c).real for c in coefs], np.float64)
        ci = _np([complex(c).imag for c in coefs], np.float64)
        ess = _np(ess_tdofs if ess_tdofs is not None else np.zeros(0), np.int32)
        h = C.c_void_p()
        _chk(lib().b2p_coperator_par(ctx.h, C.c_int64(tsize), C.c_int64(lsize), n, arr, _ptr(cr), _ptr(ci), _ptr(ess), C.c_int64(ess.size),
                                     int(diag_policy), C.byref(h)), ctx.h)
        o = cls(ctx, h)
        o._keep = list(ops)
        return o

    @classmethod
    def wrap(cls, ctx, Ar=None, Ai=None):
        """A = Ar + i Ai from two real true-dof operators (ComplexWrapperOperator): partitioned spaces, assembled matrices, ..."""
        h = C.c_void_p()
        _chk(lib().b2p_coperator_wrap(ctx.h, Ar.h if Ar is not None else None, Ai.h if Ai is not None else None, C.byref(h)), ctx.h)
        o = cls(ctx, h)
        o._keep = [Ar, Ai]
        return o

    def mult(self, xr, xi, yr, yi):
        _chk(lib().b2p_coperator_mult(self.h, _vp(xr), _vp(xi), _vp(yr), _vp(yi)), self.ctx.h)

    def set_coefficients(self, coefs):
        cr = _np([complex(c).real for c in coefs], np.float64)
        ci = _np([complex(c).imag for c in coefs], np.float64)
        _chk(lib().b2p_coperator_set_coefficients(self.h, int(cr.size), _ptr(cr), _ptr(ci)), self.ctx.h)

    def fused_applies(self):
        f = lib().b2p_coperator_fused_applies
        f.restype = C.c_long
        return int(f(self.h))

    def fused_path(self):
        """0 term by term, 1 two real sums, 2 one pass (nd4, p <= 3), 3 one pass (CTA-per-batch kernel)."""
        return int(lib().b2p_coperator_fused_path(self.h))

    def mult_hermitian_transpose(self, xr, xi, yr, yi):
        _chk(lib().b2p_coperator_mult_hermitian_transpose(self.h, _vp(xr), _vp(xi), _vp(yr), _vp(yi)), self.ctx.h)

    def add_mult(self, xr, xi, yr, yi, a):
        a = complex(a)
        _chk(lib().b2p_coperator_add_mult(self.h, _vp(xr), _vp(xi), _vp(yr), _vp(yi), C.c_double(a.real), C.c_double(a.imag)), self.ctx.h)

    def assemble_diagonal(self, dr, di):
        _chk(lib().b2p_coperator_assemble_diagonal(self.h, _vp(dr), _vp(di)), self.ctx.h)


class ComplexSolver:
    def __init__(self, ctx, h):
        self.ctx, self.h = ctx, h
        self._keep = []

    @classmethod
    def real_pc(cls, ctx, real_solver: Solver):
        h = C.c_void_p()
        _chk(lib().b2p_csolver_real_pc(ctx.h, real_solver.h, C.byref(h)), ctx.h)
        s = cls(ctx, h)
        s._keep.append(real_solver)
        return s

    @classmethod
    def assembled(cls, ctx, inner: Solver, inner_pc: Solver = None, complex_matrix=False):
        """Coarse solver on the device-assembled matrix of the complex operator given to set_operator
        (MfemWrapperSolver<ComplexOperator>): the real solver ``inner`` (taken over, with its preconditioner ``inner_pc``) runs
        on Ar + Ai for each part, or with ``complex_matrix`` once on the real 2n block [[Ar, Ai], [Ai, -Ar]]."""
        h = C.c_void_p()
        _chk(lib().b2p_csolver_assembled(ctx.h, inner.h, inner_pc.h if inner_pc is not None else None, int(bool(complex_matrix)),
                                         C.byref(h)), ctx.h)
        s = cls(ctx, h)
        s._keep += [inner, inner_pc]
        return s

    def assembled_nnz(self):
        """Entries of the real matrix the inner solver sees (this solver or the multigrid that took it over); -1 before set_operator."""
        f = lib().b2p_csolver_assembled_nnz
        f.restype = C.c_int64
        return int(f(self.h))

    def assembled_device_arrays(self):
        """(rowptr, col, val) of the real matrix the inner solver sees, as tensors viewing the solver's device memory (valid until
        its next set_operator): int32 rowptr[rows + 1], int32 col[nnz], float64 val[nnz]."""
        rows, nnz = C.c_int64(), C.c_int64()
        rp, cl, vl = C.c_void_p(), C.c_void_p(), C.c_void_p()
        _chk(lib().b2p_csolver_assembled_device_arrays(self.h, C.byref(rows), C.byref(nnz), C.byref(rp), C.byref(cl), C.byref(vl)),
             self.ctx.h)
        return (_device_view(rp.value, rows.value + 1, C.c_int32), _device_view(cl.value, nnz.value, C.c_int32),
                _device_view(vl.value, nnz.value, C.c_double))

    @classmethod
    def gmg(cls, ctx, coarse, P, G=None, cycle_it=1, smooth_it=1, cheby_order=4, sf_max=1.0):
        """Complex-valued p-multigrid (PCMatReal = false): real prolongations / gradients, complex level operators."""
        n_levels = len(P) + 1
        Parr = (C.c_void_p * max(1, len(P)))(*[p.h for p in P])
        Garr = None
        if G is not None:
            Garr = (C.c_void_p * n_levels)(*[(g.h if g is not None else None) for g in G])
        h = C.c_void_p()
        _chk(lib().b2p_csolver_gmg(ctx.h, coarse.h, n_levels, Parr, Garr, int(cycle_it), int(smooth_it), int(cheby_order),
                                   C.c_double(sf_max), C.byref(h)), ctx.h)
        s = cls(ctx, h)
        s._keep += [coarse, list(P), G]
        return s

    def gmg_set_operators(self, A, A_aux=None):
        n = len(A)
        Aarr = (C.c_void_p * n)(*[a.h for a in A])
        Garr = None
        if A_aux is not None:
            Garr = (C.c_void_p * n)(*[(a.h if a is not None else None) for a in A_aux])
        self._keep += [list(A), A_aux]
        _chk(lib().b2p_csolver_gmg_set_operators(self.h, Aarr, Garr), self.ctx.h)

    @classmethod
    def chebyshev(cls, ctx, smooth_it=1, order=4, sf_max=1.0):
        h = C.c_void_p()
        _chk(lib().b2p_csolver_chebyshev(ctx.h, int(smooth_it), int(order), C.c_double(sf_max), C.byref(h)), ctx.h)
        return cls(ctx, h)

    def lambda_max(self):
        out = C.c_double()
        _chk(lib().b2p_csolver_lambda_max(self.h, C.byref(out)), self.ctx.h)
        return out.value

    @classmethod
    def jacobi(cls, ctx, omega=1.0):
        h = C.c_void_p()
        _chk(lib().b2p_csolver_jacobi(ctx.h, C.c_double(omega), C.byref(h)), ctx.h)
        return cls(ctx, h)

    @classmethod
    def krylov(cls, ctx, kind, rel_tol=1e-6, abs_tol=0.0, max_it=100, max_dim=-1, orthog=MGS, pc_side=PC_RIGHT):
        h = C.c_void_p()
        _chk(lib().b2p_csolver_krylov(ctx.h, int(kind), C.byref(h)), ctx.h)
        _chk(lib().b2p_csolver_krylov_config(h, C.c_double(rel_tol), C.c_double(abs_tol), int(max_it), int(max_dim), int(orthog),
                                             int(pc_side)), ctx.h)
        return cls(ctx, h)

    def set_operator(self, A: ComplexOperator):
        self._keep.append(A)
        _chk(lib().b2p_csolver_set_operator(self.h, A.h), self.ctx.h)

    def set_preconditioner(self, pc):
        self._keep.append(pc)
        _chk(lib().b2p_csolver_set_preconditioner(self.h, pc.h if pc else None), self.ctx.h)

    def set_initial_guess(self, flag):
        _chk(lib().b2p_csolver_set_initial_guess(self.h, int(flag)), self.ctx.h)

    def mult(self, br, bi, xr, xi):
        _chk(lib().b2p_csolver_mult(self.h, _vp(br), _vp(bi), _vp(xr), _vp(xi)), self.ctx.h)

    def stats(self):
        its, conv = C.c_int(), C.c_int()
        r0, r1 = C.c_double(), C.c_double()
        _chk(lib().b2p_csolver_stats(self.h, C.byref(its), C.byref(r0), C.byref(r1), C.byref(conv)), self.ctx.h)
        return dict(its=its.value, initial_res=r0.value, final_res=r1.value, converged=bool(conv.value))


class KspConfig(C.Structure):
    """b2p_ksp_config (include/b2p.h): config::LinearSolverData as the composer reads it."""
    _fields_ = [("krylov_solver", C.c_int), ("tol", C.c_double), ("max_it", C.c_int), ("max_size", C.c_int), ("initial_guess", C.c_int),
                ("pc_side", C.c_int), ("gs_orthog", C.c_int), ("mg_cycle_it", C.c_int), ("mg_smooth_aux", C.c_int),
                ("mg_smooth_it", C.c_int), ("mg_smooth_order", C.c_int), ("mg_smooth_sf_max", C.c_double),
                ("mg_smooth_sf_min", C.c_double), ("mg_smooth_cheby_4th", C.c_int), ("coarse_type", C.c_int),
                ("coarse_tol", C.c_double), ("coarse_max_it", C.c_int)]


class Ksp:
    """BaseKspSolver (linalg/ksp.cpp): configuration -> Krylov solver + (multigrid) preconditioner, with the reference's
    NumTotalMult / NumTotalMultIts counters."""

    def __init__(self, ctx, order, P=(), G=None, coarse_solver=None, **overrides):
        self.ctx = ctx
        self.cfg = KspConfig()
        _chk(lib().b2p_ksp_config_default(C.byref(self.cfg), int(order)), ctx.h)
        for k, v in overrides.items():
            assert hasattr(self.cfg, k), k
            setattr(self.cfg, k, v)
        n_levels = len(P) + 1
        Parr = (C.c_void_p * max(1, len(P)))(*[p.h for p in P])
        Garr = None
        if G is not None:
            Garr = (C.c_void_p * n_levels)(*[(g.h if g is not None else None) for g in G])
        self.h = C.c_void_p()
        _chk(lib().b2p_ksp_create(ctx.h, C.byref(self.cfg), n_levels, Parr, Garr, coarse_solver.h if coarse_solver else None,
                                  C.byref(self.h)), ctx.h)
        self.n_levels = n_levels
        self._keep = [list(P), G, coarse_solver]

    def set_operators(self, op, pc_ops, aux_ops=None):
        A = (C.c_void_p * self.n_levels)(*[a.h for a in pc_ops])
        Ax = None
        if aux_ops is not None:
            Ax = (C.c_void_p * self.n_levels)(*[(a.h if a is not None else None) for a in aux_ops])
        _chk(lib().b2p_ksp_set_operators(self.h, op.h, A, Ax), self.ctx.h)
        self._keep += [op, list(pc_ops), aux_ops]

    def mult(self, x, y):
        _chk(lib().b2p_ksp_mult(self.h, _vp(x), _vp(y)), self.ctx.h)

    def stats(self):
        nm, nit, its, conv = C.c_int(), C.c_int(), C.c_int(), C.c_int()
        r0, r1 = C.c_double(), C.c_double()
        _chk(lib().b2p_ksp_stats(self.h, C.byref(nm), C.byref(nit), C.byref(its), C.byref(r0), C.byref(r1), C.byref(conv)), self.ctx.h)
        return {"num_total_mult": nm.value, "num_total_mult_its": nit.value, "its": its.value, "initial_res": r0.value,
                "final_res": r1.value, "converged": bool(conv.value)}

    def __del__(self):
        try:
            if self.h:
                lib().b2p_ksp_destroy(self.h)
                self.h = None
        except Exception:
            pass


class DivFree:
    """DivFreeSolver (linalg/divfree.cpp): y <- y + G psi with (G^T M_eps G) psi = -G^T M_eps y on the H1 hierarchy."""

    def __init__(self, ctx, nd_mass, grad, h1_ops, h1_P, h1_ess, h1_order, tol=1e-6, max_it=1000, coarse_type=1, coarse_tol=1e-3,
                 coarse_max_it=500, coarse_solver=None):
        self.ctx = ctx
        n_levels = len(h1_ops)
        assert len(h1_P) == n_levels - 1
        A = (C.c_void_p * n_levels)(*[a.h for a in h1_ops])
        Parr = (C.c_void_p * max(1, len(h1_P)))(*[p.h for p in h1_P])
        ess = np.ascontiguousarray(h1_ess, dtype=np.int32)
        self.h = C.c_void_p()
        _chk(lib().b2p_divfree_create(ctx.h, nd_mass.h, grad.h, n_levels, A, Parr, _ptr(ess), C.c_int64(ess.size), int(h1_order),
                                      C.c_double(tol), int(max_it), int(coarse_type), C.c_double(coarse_tol), int(coarse_max_it),
                                      coarse_solver.h if coarse_solver else None, C.byref(self.h)), ctx.h)
        self._keep = [nd_mass, grad, list(h1_ops), list(h1_P), coarse_solver]

    def mult(self, y):
        _chk(lib().b2p_divfree_mult(self.h, _vp(y)), self.ctx.h)

    def mult_complex(self, yr, yi):
        _chk(lib().b2p_divfree_mult_complex(self.h, _vp(yr), _vp(yi)), self.ctx.h)

    def stats(self):
        nm, nit, its, conv = C.c_int(), C.c_int(), C.c_int(), C.c_int()
        _chk(lib().b2p_divfree_stats(self.h, C.byref(nm), C.byref(nit), C.byref(its), C.byref(conv)), self.ctx.h)
        return {"num_mult": nm.value, "num_mult_its": nit.value, "its": its.value, "converged": bool(conv.value)}

    def __del__(self):
        try:
            if self.h:
                lib().b2p_divfree_destroy(self.h)
                self.h = None
        except Exception:
            pass


class VecFESpaceDesc(C.Structure):
    """b2p_vecfe_space_desc (include/b2p.h): a vector finite element space as libCEED sees a non-tensor basis."""
    _fields_ = [("P", C.c_int), ("map_type", C.c_int), ("interp", C.c_void_p), ("idx", C.c_void_p), ("orient", C.c_void_p),
                ("lsize", C.c_int64), ("curl_orient", C.c_void_p)]


MAP_HCURL, MAP_HDIV = 1, 2


def _vecfe_desc(sp, keep):
    interp = np.ascontiguousarray(sp["interp"], dtype=np.float64)
    idx = np.ascontiguousarray(sp["idx"], dtype=np.int32)
    ori = None if sp.get("orient") is None else np.ascontiguousarray(sp["orient"], dtype=np.int8)
    co = None if sp.get("curl_orient") is None else np.ascontiguousarray(sp["curl_orient"], dtype=np.int8)
    keep.extend([interp, idx, ori, co])
    return VecFESpaceDesc(int(sp["P"]), int(sp["map_type"]), interp.ctypes.data, idx.ctypes.data, None if ori is None else ori.ctypes.data,
                          int(sp["lsize"]), None if co is None else co.ctypes.data)


def vecfe_mass_operator(ctx, geom, space, coef=None):
    """b2p_operator_vecfe_mass: the mass operator of a table-described vector finite element space (e.g. Raviart-Thomas)."""
    keep = []
    d = _vecfe_desc(space, keep)
    n_attr, cptr = 0, None
    if coef is not None:
        c = np.ascontiguousarray(coef, dtype=np.float64).reshape(-1, 9)
        keep.append(c)
        n_attr, cptr = int(c.shape[0]), _ptr(c)
    h = C.c_void_p()
    _chk(lib().b2p_operator_vecfe_mass(ctx.h, geom.h, C.byref(d), n_attr, cptr, C.byref(h)), ctx.h)
    A = Operator(ctx, h)
    A._keep_vecfe = [geom, keep]
    return A


def flux_sqrt_scale(ctx, n, s, estimates):
    _chk(lib().b2p_flux_estimator_sqrt_scale(ctx.h, C.c_int64(n), C.c_double(s), _vp(estimates)), ctx.h)


class FluxEstimator:
    """CurlFluxErrorEstimator (linalg/errorestimator.cpp): flux projection M H = Flux B and the element-wise error integrals."""

    def __init__(self, ctx, geom, flux_space, smooth_space, coef_flux, coef_disc, coef_smooth, smooth_mass, tol=1e-6, max_it=500):
        self.ctx = ctx
        keep = []
        d1, d2 = _vecfe_desc(flux_space, keep), _vecfe_desc(smooth_space, keep)
        cf = np.ascontiguousarray(coef_flux, dtype=np.float64).reshape(-1, 9)
        cd = np.ascontiguousarray(coef_disc, dtype=np.float64).reshape(-1, 9)
        cs = np.ascontiguousarray(coef_smooth, dtype=np.float64).reshape(-1, 9)
        assert cf.shape == cd.shape == cs.shape
        self.h = C.c_void_p()
        _chk(lib().b2p_flux_estimator_create(ctx.h, geom.h, C.byref(d1), C.byref(d2), int(cf.shape[0]), _ptr(cf), _ptr(cd), _ptr(cs),
                                             smooth_mass.h, C.c_double(tol), int(max_it), C.byref(self.h)), ctx.h)
        self._keep = [geom, smooth_mass, keep]

    @classmethod
    def hex(cls, ctx, geom, flux_space, smooth_space, coef_flux, coef_disc, coef_smooth, smooth_mass, tol=1e-6, max_it=500):
        """b2p_flux_estimator_create_hex: the same estimator on hexahedra with sum-factorised spaces. flux_space / smooth_space are
        dicts of the fields Op.create takes (kind = ND_MASS or RT_MASS, one of each; p, lsize, idx, orient, dof_map, Bo, Bc;
        Gc, coeff and assemble optional)."""
        self = cls.__new__(cls)
        self.ctx = ctx
        keep = []

        def desc(sp):
            d, k = _desc(sp["kind"], sp["p"], sp["lsize"], sp["idx"], sp.get("orient"), sp.get("dof_map"), sp.get("Bo"), sp.get("Bc"),
                         sp.get("Gc"), sp.get("coeff"), sp.get("assemble", False))
            keep.append(k)
            return d

        d1, d2 = desc(flux_space), desc(smooth_space)
        cf = np.ascontiguousarray(coef_flux, dtype=np.float64).reshape(-1, 9)
        cd = np.ascontiguousarray(coef_disc, dtype=np.float64).reshape(-1, 9)
        cs = np.ascontiguousarray(coef_smooth, dtype=np.float64).reshape(-1, 9)
        assert cf.shape == cd.shape == cs.shape
        self.h = C.c_void_p()
        _chk(lib().b2p_flux_estimator_create_hex(ctx.h, geom.h, C.byref(d1), C.byref(d2), int(cf.shape[0]), _ptr(cf), _ptr(cd), _ptr(cs),
                                                 smooth_mass.h, C.c_double(tol), int(max_it), C.byref(self.h)), ctx.h)
        self._keep = [geom, smooth_mass, keep]
        return self

    def flux_mult(self, flux_dofs, rhs):
        """rhs = Flux flux_dofs: the right-hand side of the projection."""
        _chk(lib().b2p_flux_estimator_flux_mult(self.h, _vp(flux_dofs), _vp(rhs)), self.ctx.h)

    def project(self, flux_dofs, smooth_dofs):
        _chk(lib().b2p_flux_estimator_project(self.h, _vp(flux_dofs), _vp(smooth_dofs)), self.ctx.h)

    def integrate(self, flux_dofs, smooth_dofs, estimates):
        _chk(lib().b2p_flux_estimator_integrate(self.h, _vp(flux_dofs), _vp(smooth_dofs), _vp(estimates)), self.ctx.h)

    def indicator(self, flux_re, flux_im, Et, estimates):
        _chk(lib().b2p_flux_estimator_indicator(self.h, _vp(flux_re), _vp(flux_im) if flux_im is not None else None, C.c_double(Et),
                                                _vp(estimates)), self.ctx.h)

    def set_multigrid(self, ops, P, coarse_type=1, coarse_tol=1e-3, coarse_max_it=500, coarse_solver=None):
        """FluxProjector with "EstimatorMG": PCG preconditioned by the p-multigrid over ops (Operators, coarse -> fine, the last one
        the smooth-space mass operator given at construction) with the prolongations P (len(ops) - 1 Operators)."""
        n = len(ops)
        assert len(P) == n - 1
        A = (C.c_void_p * n)(*[a.h for a in ops])
        Parr = (C.c_void_p * max(1, len(P)))(*[p.h for p in P])
        _chk(lib().b2p_flux_estimator_set_multigrid(self.h, n, A, Parr, int(coarse_type), C.c_double(coarse_tol), int(coarse_max_it),
                                                    coarse_solver.h if coarse_solver else None), self.ctx.h)
        self._keep.append([list(ops), list(P), coarse_solver])

    def stats(self):
        nm, nit, its, conv = C.c_int(), C.c_int(), C.c_int(), C.c_int()
        _chk(lib().b2p_flux_estimator_stats(self.h, C.byref(nm), C.byref(nit), C.byref(its), C.byref(conv)), self.ctx.h)
        return {"num_mult": nm.value, "num_mult_its": nit.value, "its": its.value, "converged": bool(conv.value)}

    def __del__(self):
        try:
            if self.h:
                lib().b2p_flux_estimator_destroy(self.h)
                self.h = None
        except Exception:
            pass


class Eps:
    """The operator applications an outer eigen-solver asks for (ArpackEPSSolver::ApplyOp / ApplyOpB, linalg/arpack.cpp:631-674):
    host complex vectors in, host complex vectors out; operators, linear solve and work vectors stay on the device."""

    def __init__(self, ctx, n, K, M, op_inv, B=None, sinvert=True, gamma=1.0, delta=1.0):
        self.ctx, self.n = ctx, int(n)
        self.h = C.c_void_p()
        _chk(lib().b2p_eps_create(ctx.h, C.c_int64(self.n), K.h if K is not None else None, M.h if M is not None else None, op_inv.h,
                                  B.h if B is not None else None, int(bool(sinvert)), C.c_double(gamma), C.c_double(delta),
                                  C.byref(self.h)), ctx.h)
        self._keep = [K, M, op_inv, B]

    def _run(self, fn, x):
        x = np.ascontiguousarray(x, dtype=np.complex128)
        assert x.size == self.n
        y = np.empty(self.n, dtype=np.complex128)
        _chk(fn(self.h, x.ctypes.data_as(C.c_void_p), y.ctypes.data_as(C.c_void_p)), self.ctx.h)
        return y

    def apply_op(self, x):
        return self._run(lib().b2p_eps_apply_op, x)

    def apply_op_b(self, x):
        return self._run(lib().b2p_eps_apply_op_b, x)

    def __del__(self):
        try:
            if self.h:
                lib().b2p_eps_destroy(self.h)
                self.h = None
        except Exception:
            pass

