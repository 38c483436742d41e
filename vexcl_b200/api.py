"""Python mirror of the vex:: front end for the three hot paths, over the C ABI (ctypes).

Names, argument meaning and error behaviour follow the reference so that the parity tests
read like the reference's own tests (paths relative to /root/reference):

  Context            vexcl/devlist.hpp:273-391      (list of queues -> list of (device, stream))
  vector             vexcl/vector.hpp:220-935       (partitioned container, `=`, `+=`, ... with expressions)
  Reductor           vexcl/reductor.hpp:289-439
  SpMat              vexcl/spmat.hpp:56-386         (`y = A * x`, `y += 2 * (A * x)`, ...)
  partition          vexcl/vector.hpp:178-190

The C++ header front end in include/vexcl/ is the drop-in surface for C++ users; this module
exists so that tests and bench.py drive exactly the same C ABI from Python.  Everything that
computes goes through libvexb200.so; nothing here falls back to numpy.

Two process models share the code:
  * one process, several devices (the reference's model): Context([0, 1, ...]);
  * one process per device (torchrun): Context.distributed(rank, nranks, dev, ...): containers
    hold only the local slice, Reductor and SpMat combine over NCCL.
"""
from __future__ import annotations

import ctypes as C
from typing import Callable, Optional, Sequence

import numpy as np

from . import _lib as L

_NP2VEXB = {np.dtype(np.float64): L.F64, np.dtype(np.float32): L.F32, np.dtype(np.int32): L.I32,
            np.dtype(np.uint32): L.U32, np.dtype(np.int64): L.I64, np.dtype(np.uint64): L.U64}
_VEXB2NP = {v: k for k, v in _NP2VEXB.items()}
_SIZE = {L.F64: 8, L.F32: 4, L.I32: 4, L.U32: 4, L.I64: 8, L.U64: 8}


def _vdt(dtype) -> int:
    try:
        return _NP2VEXB[np.dtype(dtype)]
    except KeyError:
        raise TypeError(f"unsupported element type {dtype}") from None


def _is_float(t: int) -> bool:
    return t in (L.F64, L.F32)


def common_type(a: int, b: int) -> int:
    """Usual arithmetic conversions (what the device compiler applies to the reference's emitted C)."""
    if L.F64 in (a, b): return L.F64
    if L.F32 in (a, b): return L.F32
    if L.U64 in (a, b): return L.U64
    if L.I64 in (a, b): return L.I64
    if L.U32 in (a, b): return L.U32
    return L.I32


def partition(n: int, nparts: int, weights=None) -> np.ndarray:
    part = (C.c_size_t * (nparts + 1))()
    w = None
    if weights is not None:
        w = (C.c_double * nparts)(*[float(x) for x in weights])
    L.check(L.lib().vexb_partition(n, nparts, w, part))
    return np.array(list(part), dtype=np.int64)


# ------------------------------------------------------------------------------------------- Context
class Context:
    """A list of (device, stream) pairs, one per partition slot."""
    use_peer_reduce = True          # combine reductions through peer memory when a peer group exists

    def __init__(self, devices: Sequence[int] = (0,), use_nccl: Optional[bool] = None, weights=None, use_peer: bool = False,
                 peer_halo: Optional[bool] = None):
        """peer_halo: push SpMat halos through NVLink peer memory inside the product kernel (None: whenever the slots
        sit on distinct devices that can access each other; False: NCCL send/recv or copy-engine copies)."""
        lib = L.lib()
        L.check(lib.vexb_init())
        self.nparts = len(devices)
        self.local = list(range(self.nparts))
        self.devs = {k: int(d) for k, d in enumerate(devices)}
        self.streams = {}
        self.weights = weights
        for k in self.local:
            s = C.c_void_p()
            L.check(lib.vexb_stream_create(self.devs[k], C.byref(s)))
            self.streams[k] = s
        self.comms = None
        self.allgather = None
        distinct = len(set(devices)) == len(devices)
        if use_nccl is None:
            use_nccl = False
        if use_nccl and self.nparts > 1:
            if not distinct:
                raise ValueError("NCCL needs one distinct device per part")
            arr = (C.c_int * self.nparts)(*devices)
            out = (C.c_void_p * self.nparts)()
            L.check(lib.vexb_comm_create_all(self.nparts, arr, out))
            self.comms = {k: C.c_void_p(out[k]) for k in range(self.nparts)}
        self.peer_halo = (distinct and self.nparts > 1) if peer_halo is None else bool(peer_halo)
        self.peers = None
        if use_peer and self.nparts > 1:
            if not distinct:
                raise ValueError("peer groups need one distinct device per part")
            arr = (C.c_int * self.nparts)(*devices)
            out = (C.c_void_p * self.nparts)()
            L.check(lib.vexb_peer_create_all(self.nparts, arr, out))
            self.peers = {k: C.c_void_p(out[k]) for k in range(self.nparts)}
        self._ws = {}

    @classmethod
    def distributed(cls, rank: int, nranks: int, dev: int, unique_id: bytes,
                    allgather: Callable[[np.ndarray], list], use_peer: bool = True, peer_halo: Optional[bool] = None):
        """One process per device.  `unique_id`: the 128 bytes produced by rank 0's
        comm_unique_id() and broadcast by the launcher; `allgather(arr)` returns the list of every
        rank's int64 array (used once, at SpMat construction, to share ghost column lists)."""
        self = cls.__new__(cls)
        lib = L.lib()
        L.check(lib.vexb_init())
        self.nparts = nranks
        self.local = [rank]
        self.devs = {rank: dev}
        self.weights = None
        s = C.c_void_p()
        L.check(lib.vexb_stream_create(dev, C.byref(s)))
        self.streams = {rank: s}
        self.comms = None
        if nranks > 1:
            c = C.c_void_p()
            buf = C.create_string_buffer(unique_id, 128)
            L.check(lib.vexb_comm_create_rank(dev, nranks, rank, buf, C.byref(c)))
            self.comms = {rank: c}
        self.allgather = allgather
        self.peer_halo = (nranks > 1 and use_peer) if peer_halo is None else bool(peer_halo)
        self.peers = None
        if nranks > 1 and use_peer:
            # peer-memory group: exchange the CUDA IPC handles of the mailboxes through the launcher's all-gather
            # Every rank runs both collectives whatever happens locally, and the group is used only if ALL ranks
            # succeeded -- otherwise everybody falls back to ncclAllReduce (no rank may wait on a missing peer).
            p = C.c_void_p()
            h = C.create_string_buffer(64)
            ok = lib.vexb_peer_create(dev, rank, nranks, C.byref(p), h) == L.OK
            allh = allgather(np.frombuffer(h.raw, dtype=np.uint8).copy())
            if ok:
                cat = b"".join(np.asarray(a, dtype=np.uint8).tobytes() for a in allh)
                ok = lib.vexb_peer_connect(p, C.create_string_buffer(cat, 64 * nranks)) == L.OK
            everybody = allgather(np.array([1 if ok else 0], dtype=np.int64))
            if all(int(np.asarray(a)[0]) == 1 for a in everybody):
                self.peers = {rank: p}
            elif p.value:
                lib.vexb_peer_destroy(p)
        self._ws = {}
        return self

    @staticmethod
    def comm_unique_id() -> bytes:
        buf = C.create_string_buffer(128)
        L.check(L.lib().vexb_comm_unique_id(buf))
        return buf.raw

    @property
    def is_distributed(self) -> bool:
        return len(self.local) != self.nparts

    def size(self) -> int:
        return self.nparts

    def partition(self, n: int) -> np.ndarray:
        return partition(n, self.nparts, self.weights)

    def finish(self):
        for k in self.local:
            L.check(L.lib().vexb_stream_sync(self.devs[k], self.streams[k]))

    def use_stream(self, part: int, stream_ptr: int):
        """Run part `part` on an externally owned cudaStream_t (e.g. torch's current stream)."""
        self.streams = dict(self.streams)                     # a new table: cached argument arrays notice the change
        self.streams[part] = C.c_void_p(stream_ptr)

    def workspace(self, k: int, slices: int = 1):
        """(reduction workspace, result buffer) of slot k; `slices` > 1: room for that many combined reductions."""
        key = (k, slices) if slices > 1 else k
        if key not in self._ws:
            lib = L.lib()
            nb = C.c_size_t()
            L.check(lib.vexb_reduce_workspace_bytes(self.devs[k], C.byref(nb)))
            ws, res = C.c_void_p(), C.c_void_p()
            L.check(lib.vexb_malloc(self.devs[k], nb.value * slices, C.byref(ws)))
            L.check(lib.vexb_memset(self.devs[k], ws, 0, nb.value * slices, self.streams[k]))
            L.check(lib.vexb_malloc(self.devs[k], 128, C.byref(res)))
            self._ws[key] = (ws, res)
        return self._ws[key]

    def _arr(self, mapping):
        return (C.c_void_p * len(self.local))(*[mapping[k] for k in self.local])


# ------------------------------------------------------------------------------------------- expressions
class Node:
    """Expression tree node (the analogue of a Boost.Proto expression, operations.hpp:455-512)."""
    dtype: int = L.F64
    __array_ufunc__ = None          # numpy scalars defer to our reflected operators (np.float64(2) * v)

    def _bin(self, op, other, swap=False):
        o = wrap(other)
        return Binary(op, o, self) if swap else Binary(op, self, o)

    def __add__(self, o): return self._bin("ADD", o)
    def __radd__(self, o): return self._bin("ADD", o, True)
    def __sub__(self, o): return self._bin("SUB", o)
    def __rsub__(self, o): return self._bin("SUB", o, True)
    def __mul__(self, o):
        if isinstance(o, (SpMat, stencil)):
            return NotImplemented                      # x * A is not defined; x * s is stencil.__rmul__
        return self._bin("MUL", o)
    def __rmul__(self, o): return self._bin("MUL", o, True)
    def __truediv__(self, o): return self._bin("DIV", o)
    def __rtruediv__(self, o): return self._bin("DIV", o, True)
    def __mod__(self, o): return self._bin("MOD", o)
    def __and__(self, o): return self._bin("BAND", o)
    def __or__(self, o): return self._bin("BOR", o)
    def __xor__(self, o): return self._bin("BXOR", o)
    def __lshift__(self, o): return self._bin("SHL", o)
    def __rshift__(self, o): return self._bin("SHR", o)
    def __lt__(self, o): return self._bin("LT", o)
    def __gt__(self, o): return self._bin("GT", o)
    def __le__(self, o): return self._bin("LE", o)
    def __ge__(self, o): return self._bin("GE", o)
    def eq(self, o): return self._bin("EQ", o)
    def ne(self, o): return self._bin("NE", o)
    def logical_and(self, o): return self._bin("LAND", o)
    def logical_or(self, o): return self._bin("LOR", o)
    def logical_not(self): return Unary("LNOT", self)
    def __neg__(self): return Unary("NEG", self)
    def __pos__(self): return self


class Scalar(Node):
    def __init__(self, value, dtype=None):
        if dtype is None:
            if isinstance(value, (bool, np.bool_)):
                dtype, value = L.I32, int(value)
            elif isinstance(value, (int,)):
                dtype = L.I32 if -2**31 <= value < 2**31 else L.I64
            elif isinstance(value, float):
                dtype = L.F64
            elif isinstance(value, np.generic):
                dtype = _vdt(value.dtype)
            else:
                raise TypeError(f"cannot use {type(value)} as a scalar terminal")
        self.value, self.dtype = value, dtype


class ElementIndex(Node):
    """vex::element_index(offset) (element_index.hpp:40-111): the global element index."""
    dtype = L.U64

    def __init__(self, offset: int = 0):
        self.offset = offset


class Unary(Node):
    def __init__(self, op, a):
        self.op, self.a = op, a
        self.dtype = L.I32 if op == "LNOT" else a.dtype


class Func(Node):
    """Builtin function call (function.hpp:255-268).  Result type: common type of the arguments."""
    def __init__(self, op, *args):
        self.op, self.args = op, [wrap(a) for a in args]
        t = self.args[0].dtype
        for a in self.args[1:]:
            t = common_type(t, a.dtype)
        if op not in ("FABS", "FMIN", "FMAX") and not _is_float(t):
            t = L.F64                                 # C promotes integer arguments of math functions to double
        self.dtype = t


class Binary(Node):
    def __init__(self, op, a, b):
        self.op, self.a, self.b = op, a, b
        self.ctype = common_type(a.dtype, b.dtype)
        self.dtype = L.I32 if op in ("LT", "GT", "LE", "GE", "EQ", "NE", "LAND", "LOR") else self.ctype


class Select(Node):
    def __init__(self, cond, a, b):
        self.cond, self.a, self.b = wrap(cond), wrap(a), wrap(b)
        self.dtype = common_type(self.a.dtype, self.b.dtype)


def if_else(cond, a, b): return Select(cond, a, b)


class Call(Node):
    """Call of a user-defined device function (VEX_FUNCTION).  A raw_pointer goes to a parameter declared ptr(dtype)."""
    def __init__(self, fn: "UserFunction", args):
        self.fn, self.args = fn, [a if isinstance(a, Pointer) else wrap(a) for a in args]
        for a, t in zip(self.args, fn.arg_types):
            if isinstance(a, Pointer) and (a.offsets or t != L.PTR(a.dtype)):
                raise TypeError(f"{fn.name}: a raw_pointer without arithmetic goes to a parameter declared ptr() of its type")
            if not isinstance(a, Pointer) and t & 0x10:
                raise TypeError(f"{fn.name}: a ptr() parameter takes a raw_pointer")
        self.dtype = fn.ret


class ptr:
    """The type of a pointer parameter of a UserFunction: ptr(np.float64) is `double *`, ptr(np.float64, const=True)
    `const double *` (the same parameter to the library: the constness only goes into the prologue)."""
    def __init__(self, dtype, const: bool = False):
        self.dtype, self.const = _vdt(dtype), bool(const)


class UserFunction:
    """VEX_FUNCTION(ret, name, (type, arg)..., body) (vexcl/function.hpp:225): a device function given as C source.
    `args` is a list of (numpy dtype or ptr(dtype), name); inside `body` the arguments are available under their names
    (and, as in the reference's older form, as prm1, prm2, ...).  Expressions that call it run on the NVRTC side path.
    deps: UserFunctions the body calls by their names (VEX_FUNCTION_D); every program that calls this one holds them.
    preamble: file-scope text (helpers, macros) before the definition (VEX_FUNCTION_V1_WITH_PREAMBLE); helpers in it
    need no __device__."""

    def __init__(self, ret, name: str, args, body: str, deps=(), preamble: str = ""):
        self.ret = _vdt(ret)
        self.arg_types = [L.PTR(t.dtype) if isinstance(t, ptr) else _vdt(t) for t, _ in args]
        ctypes_names = {L.F64: "double", L.F32: "float", L.I32: "int", L.U32: "unsigned int", L.I64: "long long", L.U64: "unsigned long long"}
        prologue = "".join((f"{'const ' if t.const else ''}{ctypes_names[t.dtype]} *{nm} = prm{k + 1}; " if isinstance(t, ptr)
                            else f"const {ctypes_names[at]} {nm} = prm{k + 1}; ")
                           for k, (at, (t, nm)) in enumerate(zip(self.arg_types, args)))
        fid = C.c_int(-1)
        at = (C.c_int * max(len(args), 1))(*self.arg_types)
        dep_ids = [d.id if isinstance(d, UserFunction) else int(d) for d in deps]
        if dep_ids or preamble:
            da = (C.c_int * max(len(dep_ids), 1))(*dep_ids)
            L.check(L.lib().vexb_function_register_ex(name.encode(), self.ret, len(args), at, (prologue + body).encode(),
                                                      len(dep_ids), da, preamble.encode(), C.byref(fid)))
        else:
            L.check(L.lib().vexb_function_register(name.encode(), self.ret, len(args), at, (prologue + body).encode(), C.byref(fid)))
        self.id, self.name = fid.value, name

    def __call__(self, *args):
        if len(args) != len(self.arg_types):
            raise TypeError(f"{self.name} takes {len(self.arg_types)} arguments")
        return Call(self, args)


class Temp(Node):
    """vex::make_temp<tag, T>(expr) (vexcl/temporary.hpp): `expr` evaluated once per element, before the expression that
    uses it, into a local variable of `dtype` (expr's type by default) that every use reads.  Within one expression a tag
    is one temporary; the same tag over a different expression is refused."""
    def __init__(self, tag: int, expr, dtype=None):
        self.tag, self.a = int(tag), wrap(expr)
        self.dtype = self.a.dtype if dtype is None else _vdt(dtype)


def make_temp(tag: int, expr, dtype=None) -> Temp:
    """vex::make_temp<tag>(expr), or vex::make_temp<tag, dtype>(expr)."""
    return Temp(tag, expr, dtype)


class Pointer:
    """vex::raw_pointer(x) (vexcl/vector_pointer.hpp): the device address of x's element 0, for expressions that reach any
    element.  p[i], deref(p + i), (p + a)[b], i + p and p - i read one element (VEXB_OP_LOAD: every offset is widened to
    int64 on its own, as C does, then added; a read outside x gives 0, so a load under an if_else guard is safe); a
    UserFunction takes p itself for a ptr() parameter.  Nothing else is
    defined on a pointer.  x must have one slice, and every vector of an expression that holds p must live on p's
    device."""
    __array_ufunc__ = None

    def __init__(self, vec, offsets=()):
        self.vec, self.offsets, self.dtype = vec, tuple(offsets), vec.dtype      # offsets: (sign, node) in order

    def _offset(self, o, sign):
        if isinstance(o, Pointer):
            raise TypeError("two pointers do not combine")
        o = wrap(o)
        if _is_float(o.dtype):
            raise TypeError("pointer arithmetic takes an integral offset")
        return Pointer(self.vec, self.offsets + ((sign, o),))

    def __add__(self, o): return self._offset(o, +1)
    def __radd__(self, o): return self._offset(o, +1)
    def __sub__(self, o): return self._offset(o, -1)
    def __getitem__(self, i): return Load(self._offset(i, +1))

    def _refuse(self, *_):
        raise TypeError("a raw_pointer is only indexed, offset by an integer, dereferenced or passed to a user function")
    __rsub__ = __mul__ = __rmul__ = __truediv__ = __rtruediv__ = __mod__ = __neg__ = __lt__ = __gt__ = __le__ = __ge__ = _refuse
    __and__ = __or__ = __xor__ = __lshift__ = __rshift__ = _refuse


class Load(Node):
    """One element read through a pointer: *(p + offsets).  `args` holds the offset nodes (for the tree walkers)."""
    def __init__(self, p: Pointer):
        self.p, self.dtype = p, p.dtype
        self.args = [o for _, o in p.offsets]


def raw_pointer(x) -> Pointer:
    """vex::raw_pointer(x): refused, like the reference, for vectors of more than one slice."""
    if not isinstance(x, vector):
        raise TypeError("raw_pointer takes a vector")
    if x.ctx.nparts != 1:
        raise ValueError("raw_pointer is not supported for multi-device contexts")
    return Pointer(x)


def deref(p) -> Load:
    """*p: the element p points to."""
    if not isinstance(p, Pointer):
        raise TypeError("deref takes a raw_pointer or pointer arithmetic on one")
    return Load(p)


def _header_devices(ctx: Context):
    return sorted(set(ctx.devs[k] for k in ctx.local))


def push_program_header(ctx: Context, text: str):
    """vex::push_program_header(ctx, text) (backend/common.hpp:120-206): `text` goes at the very top of every kernel
    compiled from user text (expressions that call a UserFunction, stencil operators, user value types) on each device
    of ctx, once per distinct device.  It replaces the previous header until pop_program_header(ctx)."""
    for d in _header_devices(ctx):
        L.check(L.lib().vexb_program_header_push(d, text.encode()))


def pop_program_header(ctx: Context):
    """Restores the program header each device of ctx had before the last push."""
    for d in _header_devices(ctx):
        L.check(L.lib().vexb_program_header_pop(d))


def program_header(dev: int) -> str:
    """The effective program header of device `dev` ("" when none was pushed)."""
    n = C.c_size_t(0)
    L.check(L.lib().vexb_program_header_get(dev, None, C.byref(n)))
    buf = C.create_string_buffer(n.value)
    L.check(L.lib().vexb_program_header_get(dev, buf, C.byref(n)))
    return buf.value.decode()


def _mkfunc(op):
    return lambda *args: Func(op, *args)


sin, cos, tan, asin, acos, atan = (_mkfunc(o) for o in ("SIN", "COS", "TAN", "ASIN", "ACOS", "ATAN"))
sinh, cosh, tanh, exp, exp2, log = (_mkfunc(o) for o in ("SINH", "COSH", "TANH", "EXP", "EXP2", "LOG"))
log2, log10, sqrt, rsqrt, cbrt, fabs = (_mkfunc(o) for o in ("LOG2", "LOG10", "SQRT", "RSQRT", "CBRT", "FABS"))
floor, ceil, round_, trunc = (_mkfunc(o) for o in ("FLOOR", "CEIL", "ROUND", "TRUNC"))
pow_, atan2, fmod, hypot, fmin, fmax, fma = (_mkfunc(o) for o in ("POW", "ATAN2", "FMOD", "HYPOT", "FMIN", "FMAX", "FMA"))


def wrap(x) -> Node:
    if isinstance(x, Node):
        return x
    if isinstance(x, Pointer):
        raise TypeError("a raw_pointer is only indexed, offset by an integer, dereferenced or passed to a user function")
    if isinstance(x, SpMVTerm) and isinstance(x.A, SpMatCCSR) and isinstance(x.x, vector):
        return CcsrProduct(x.A, x.x, x.scale)                  # a CCSR product where an operand goes
    return Scalar(x)


class _Lowering:
    def __init__(self, part: int, part_start: int):
        self.e = L.Expr()
        self.part, self.part_start = part, part_start
        self.size = None
        self.ctx = None
        # assignments only: the one matrix whose sliced-ELL strips this expression may take as terminals (the generated
        # kernel sweeps in the storage order of one strip); False where such strips are not taken at all
        self.sweep = False
        # assignments only: the target vector; a CCSR product of it is evaluated into a temporary (kept here until the
        # launch is enqueued)
        self.target = None
        self.keep = []
        # temporaries (Temp): code[0, n_prefix) holds their definitions, each ending with its TDEF; slot k of `temps` is
        # (tag, dtype, definition by content, node)
        self.n_prefix = 0
        self.temps = []
        # raw pointers: the device they live on, and the vectors seen (each must have one slice on that device)
        self.ptr_dev = None
        self.vec_seen = []

    def see(self, v=None, ptr_vec=None):
        """Record a vector (or the vector behind a pointer) of the expression, and refuse a pointer next to a vector of
        several slices or of another device, before anything is launched."""
        if v is not None:
            self.vec_seen.append(v)
        if ptr_vec is not None:
            d = ptr_vec.ctx.devs[ptr_vec.ctx.local[0]]
            if self.ptr_dev is not None and self.ptr_dev != d:
                raise ValueError("raw pointers of one expression must live on one device")
            self.ptr_dev = d
        if self.ptr_dev is not None:
            for w in self.vec_seen:
                if w.ctx.nparts != 1 or w.ctx.devs[w.ctx.local[0]] != self.ptr_dev:
                    raise ValueError("every vector of an expression with a raw_pointer must have one slice, on the pointer's device")

    def pointer(self, p: Pointer) -> int:
        """The pointer's terminal: its address, and its element count in pad[0..5] (a load outside reads 0)."""
        self.see(ptr_vec=p.vec)
        k = self.term(L.TERM_PTR, p.dtype, ptr=p.vec.bufs[p.vec.ctx.local[0]].value or 0)
        for b in range(6):
            self.e.term[k].pad[b] = (p.vec.n >> (8 * b)) & 0xff
        return k

    def term(self, kind, dtype, pad0: int = 0, **kw) -> int:
        k = self.e.n_terms
        if k >= L.MAX_TERMS:
            raise ValueError("expression has too many terminals")
        t = self.e.term[k]
        t.kind, t.dtype = kind, dtype
        t.pad[0] = pad0
        for name, v in kw.items():
            setattr(t.v, name, v)
        self.e.n_terms = k + 1
        return k

    def emit(self, op, typ, arg=0):
        k = self.e.n_code
        if k >= L.MAX_CODE:
            raise ValueError("expression is too long")
        ins = self.e.code[k]
        ins.op, ins.type, ins.arg = L.OP[op], typ, arg
        self.e.n_code = k + 1

    def cvt(self, frm, to):
        if frm != to:
            self.emit("CVT", to, frm)

    def lower(self, n: Node):
        if isinstance(n, vector):
            if self.size is None:
                self.size, self.ctx = n.n, n.ctx
            elif n.n != self.size:
                raise ValueError("vectors of different sizes in one expression")     # VEXCL_CHECK_SIZES, operations.hpp:1824-1840
            self.see(n)
            self.emit("TERM", n.dtype, self.term(L.TERM_VEC, n.dtype, ptr=n.bufs[self.part].value or 0))
        elif isinstance(n, Load):
            # the index: every offset widened to int64 on its own (signed types sign-extended, unsigned zero-extended),
            # then added; *p reads element 0
            if not n.p.offsets:
                self.lower(Scalar(0, L.I64))
            for j, (sign, o) in enumerate(n.p.offsets):
                self.lower(o); self.cvt(o.dtype, L.I64)
                if j:
                    self.emit("ADD" if sign > 0 else "SUB", L.I64)
                elif sign < 0:
                    self.emit("NEG", L.I64)
            self.emit("LOAD", n.dtype, self.pointer(n.p))
        elif isinstance(n, InlineSpMV):
            if self.size is None:
                self.size, self.ctx = n.A.n, n.A.ctx
            strip = n.strip(self.part)
            if strip is None and (self.sweep is None or self.sweep is n.A):
                strip = n.strip(self.part, sweep=True)
                if strip is not None:
                    self.sweep = n.A
            if strip is not None:
                # row i of A*x as a terminal: the row loop is generated into this expression's kernel (VEXB_TERM_SPMV)
                xs = self.term(L.TERM_VEC, n.dtype, ptr=n.x.bufs[self.part].value or 0)
                self.emit("TERM", n.dtype, self.term(L.TERM_SPMV, n.dtype, pad0=xs, ptr=strip))
            else:
                self.lower(n.temporary())
        elif isinstance(n, CcsrProduct):
            if self.size is None:
                self.size, self.ctx = n.A.n, n.A.ctx
            if n.scale != 1.0:
                self.lower(Scalar(n.scale, n.dtype))
            if n.x is self.target:
                tmp = n.temporary()                     # x[i] written while other threads read x[i + col[j]] would race
                self.keep.append(tmp)
                self.lower(tmp)
            else:
                # row i of A*x as a terminal: the CCSR row loop is generated into this expression's kernel (VEXB_TERM_CCSR)
                xs = self.term(L.TERM_VEC, n.dtype, ptr=n.x.bufs[self.part].value or 0)
                k = self.term(L.TERM_CCSR, n.dtype, pad0=xs, ptr=n.A.h.value)
                self.e.term[k].pad[1] = n.A.idx_bytes
                self.emit("TERM", n.dtype, k)
            if n.scale != 1.0:
                self.emit("MUL", n.dtype)
        elif isinstance(n, Scalar):
            field = {L.F64: "f64", L.F32: "f32", L.I32: "i32", L.U32: "u32", L.I64: "i64", L.U64: "u64"}[n.dtype]
            self.emit("TERM", n.dtype, self.term(L.TERM_SCALAR, n.dtype, **{field: n.value}))
        elif isinstance(n, ElementIndex):
            self.emit("TERM", L.U64, self.term(L.TERM_INDEX, L.U64, i64=n.offset))
        elif isinstance(n, Unary):
            self.lower(n.a)
            self.emit(n.op, n.a.dtype)
        elif isinstance(n, Func):
            for a in n.args:
                self.lower(a); self.cvt(a.dtype, n.dtype)
            self.emit(n.op, n.dtype)
        elif isinstance(n, Binary):
            self.lower(n.a); self.cvt(n.a.dtype, n.ctype)
            self.lower(n.b); self.cvt(n.b.dtype, n.ctype)
            self.emit(n.op, n.ctype)
        elif isinstance(n, Call):
            for a, t in zip(n.args, n.fn.arg_types):
                if isinstance(a, Pointer):
                    self.emit("TERM", L.PTR(a.dtype), self.pointer(a))       # the pointer itself (Call checked the type)
                    continue
                self.lower(a); self.cvt(a.dtype, t)
            self.emit("CALL", n.fn.ret, n.fn.id)
        elif isinstance(n, Temp):
            self.temp(n)
        elif isinstance(n, Select):
            self.lower(n.cond)
            if n.cond.dtype != L.I32:                     # any arithmetic condition: (c != 0)
                zero = Scalar(0.0 if _is_float(n.cond.dtype) else 0, n.cond.dtype)
                self.lower(zero); self.emit("NE", n.cond.dtype)
            self.lower(n.a); self.cvt(n.a.dtype, n.dtype)
            self.lower(n.b); self.cvt(n.b.dtype, n.dtype)
            self.emit("SELECT", n.dtype)
        else:
            raise TypeError(f"cannot lower {type(n)}")

    def temp(self, n: Temp):
        """Lower the definition where the temporary is first used, then move it to the end of the prefix; a later use of
        the tag drops its lowering again (when it is the same program) and reads the same slot."""
        for k, (tag, typ, dk, node) in enumerate(self.temps):
            if node is n:                       # the same node again: no second lowering (nor product temporary)
                self.emit("TREF", n.dtype, k)
                return
        rel, terms = self.e.n_code - self.n_prefix, self.e.n_terms
        self.lower(n.a)
        self.cvt(n.a.dtype, n.dtype)
        frm = self.n_prefix + rel               # nested temporaries have moved into the prefix meanwhile
        d = self._definition(frm, self.e.n_code)
        for k, (tag, typ, dk, node) in enumerate(self.temps):
            if tag == n.tag:
                if dk != d or typ != n.dtype:
                    raise ValueError(f"make_temp({tag}): one tag names two different expressions")
                self.e.n_code = frm
                for j in range(terms, self.e.n_terms):
                    C.memset(C.addressof(self.e.term[j]), 0, C.sizeof(L.Term))
                self.e.n_terms = terms
                self.emit("TREF", n.dtype, k)
                return
        if len(self.temps) >= L.MAX_TEMPS:
            raise ValueError("expression has too many temporaries")
        self.emit("TDEF", n.dtype, len(self.temps))
        code = [(c.op, c.type, c.arg) for c in self.e.code[self.n_prefix:self.e.n_code]]
        cut = frm - self.n_prefix
        for j, (op, typ, arg) in enumerate(code[cut:] + code[:cut]):
            ins = self.e.code[self.n_prefix + j]
            ins.op, ins.type, ins.arg = op, typ, arg
        self.n_prefix += self.e.n_code - frm
        self.temps.append((n.tag, n.dtype, d, n))
        self.emit("TREF", n.dtype, len(self.temps) - 1)

    def _definition(self, frm, to) -> bytes:
        """code[frm, to) with every terminal by content (a product's x too)."""
        out = []
        for pc in range(frm, to):
            c = self.e.code[pc]
            out.append(bytes((c.op, c.type)))
            if c.op not in (L.OP["TERM"], L.OP["LOAD"]):
                out.append(c.arg.to_bytes(2, "little"))
                continue
            t = self.e.term[c.arg]
            raw = bytearray(C.string_at(C.addressof(t), C.sizeof(L.Term)))
            if t.kind in (L.TERM_SPMV, L.TERM_CCSR):
                raw[2] = 0
                raw += C.string_at(C.addressof(self.e.term[t.pad[0]]), C.sizeof(L.Term))
            out.append(bytes(raw))
        return b"".join(out)


def _has_call(n) -> bool:
    if isinstance(n, (Call, InlineSpMV, CcsrProduct)):
        return True
    kids = [getattr(n, c, None) for c in ("a", "b", "cond")] + list(getattr(n, "args", []))
    return any(isinstance(k, Node) and _has_call(k) for k in kids)


def _temporary(ctx, expr, n):
    """The expression evaluated into a vector of its own type (one extra pass): what a reduction folds when it cannot be
    served in one kernel."""
    tmp = vector(ctx, n, _VEXB2NP[expr.dtype])
    tmp._assign(L.SET, expr, sweep=False)
    return tmp


def _has_product_temporary(n, part) -> bool:
    """An inlined product whose strips cannot be inlined (halo, sliced ELL, float values, ...) is evaluated into a
    temporary product when lowered; a reduction of such an expression keeps the temporary of the whole expression."""
    if isinstance(n, InlineSpMV):
        return n.strip(part) is None
    kids = [getattr(n, c, None) for c in ("a", "b", "cond")] + list(getattr(n, "args", []))
    return any(isinstance(k, Node) and _has_product_temporary(k, part) for k in kids)


def _reduce_in_one_pass(ctx, expr, n):
    """The expression a Reductor hands to vexb_reduce_all / vexb_reduce_multi.  User functions and inlined sparse
    products are folded by one kernel generated for the request (bit-identical to reducing their temporary), so the
    expression goes as it is, unless it holds a product that cannot be inlined."""
    if _has_call(expr) and _has_product_temporary(expr, ctx.local[0]):
        return _temporary(ctx, expr, n)
    return expr


def _find_props(n: Node):
    """(ctx, size) of the first vector terminal (get_expression_properties, operations.hpp:1411)."""
    if isinstance(n, vector):
        return n.ctx, n.n
    if isinstance(n, (InlineSpMV, CcsrProduct)):
        return n.A.ctx, n.A.n
    for child in ("a", "b", "cond"):
        c = getattr(n, child, None)
        if isinstance(c, Node):
            r = _find_props(c)
            if r:
                return r
    for c in getattr(n, "args", []):
        r = _find_props(c)
        if r:
            return r
    return None


# ------------------------------------------------------------------------------------------- inlined sparse products
class InlineSpMV(Node):
    """`A * x` as a terminal of a vector expression: vex::make_inline(A * x) (spmat/inline_spmv.hpp:68-76) and the
    vex::sparse product terminal (sparse/product.hpp:45-130).  When the strips have no halo the row loop is generated into
    the consumer's kernel (VEXB_TERM_SPMV); otherwise the product is evaluated into a temporary when the expression is
    lowered.  A fresh node per use."""

    def __init__(self, A, x):
        if x.n != A.m:
            raise ValueError("inline product: vector size does not match the matrix")
        self.A, self.x, self.dtype = A, x, x.dtype
        self._tmp = None

    def strip(self, part, sweep=False):
        """The strip of `part` as a terminal: thread per row (vexb_dspmat_inline_strip), or with sweep=True a sliced-ELL
        strip for a storage-order sweep (vexb_dspmat_sweep_strip, assignments only)."""
        if not _is_float(self.dtype) or not hasattr(self.A, "parts"):
            return None
        query = L.lib().vexb_dspmat_sweep_strip if sweep else L.lib().vexb_dspmat_inline_strip
        h = C.c_void_p()
        L.check(query(self.A.parts[part], C.byref(h)))
        if not h.value:
            return None
        # all or nothing: an expression is lowered once per slot, and every slot must see the same kind of terminal
        for k in self.A.ctx.local:
            hk = C.c_void_p()
            L.check(query(self.A.parts[k], C.byref(hk)))
            if not hk.value:
                return None
        return h.value

    def temporary(self):
        if self._tmp is None:
            self._tmp = vector(self.A.ctx, self.A.n, self.x.np_dtype)
            self.A.apply(self.x, self._tmp, 1.0, False)
        return self._tmp


def make_inline(term):
    """vex::make_inline(A * x): the (unscaled) product as an expression terminal."""
    if not isinstance(term, SpMVTerm) or term.scale != 1.0:
        raise ValueError("make_inline: scale the inlined product inside the expression instead")
    if isinstance(term.A, SpMatCCSR):
        return CcsrProduct(term.A, term.x)
    return InlineSpMV(term.A, term.x)


class CcsrProduct(Node):
    """`A * x` of a SpMatCCSR where an operand goes -- vx.sin(A * x), x * (A * x), y *= A * x, user function arguments,
    if_else, Reductor calls, make_inline(A * x): the reference's ccsr_product terminal (spmat/ccsr.hpp:88-270).  Lowered
    to VEXB_TERM_CCSR, whose row loop is generated into the consumer's kernel (same bits as a temporary from A.apply),
    scaled inside the expression when it carries a scale.  When x is the assignment's target the product is evaluated
    into a temporary first."""

    def __init__(self, A, x, scale=1.0):
        if x.n != A.n:
            raise ValueError("SpMatCCSR product: vector size does not match the matrix")
        if x.dtype != A.val_dtype:
            raise TypeError("SpMatCCSR product: the vector's type differs from the matrix's value type")
        self.A, self.x, self.scale, self.dtype = A, x, scale, A.val_dtype

    def temporary(self):
        tmp = vector(self.A.ctx, self.A.n, self.x.np_dtype)
        self.A.apply(self.x, tmp, 1.0, False)
        return tmp


# ------------------------------------------------------------------------------------------- SpMV additive terms
class SpMVTerm:
    """`A * x`, possibly scaled: the additive_operator of operations.hpp:759-776."""
    __array_ufunc__ = None
    def __init__(self, A, x, scale=1.0):
        self.A, self.x, self.scale = A, x, scale

    def _operand(self, o):
        """A CCSR product meeting another expression (not a scale) becomes an operand: CcsrProduct."""
        return isinstance(self.A, SpMatCCSR) and isinstance(o, (Node, SpMVTerm))

    def __mul__(self, s): return wrap(self) * s if self._operand(s) else SpMVTerm(self.A, self.x, self.scale * s)
    def __rmul__(self, s): return s * wrap(self) if self._operand(s) else SpMVTerm(self.A, self.x, self.scale * s)
    def __truediv__(self, s): return wrap(self) / s if self._operand(s) else SpMVTerm(self.A, self.x, self.scale / s)
    def __neg__(self): return SpMVTerm(self.A, self.x, -self.scale)

    def _cmp(self, op, o):
        if not isinstance(self.A, SpMatCCSR):
            return NotImplemented
        return Node._bin(wrap(self), op, o)

    def __lt__(self, o): return self._cmp("LT", o)
    def __gt__(self, o): return self._cmp("GT", o)
    def __le__(self, o): return self._cmp("LE", o)
    def __ge__(self, o): return self._cmp("GE", o)
    def __add__(self, o): return Mixed(None, [self]) + o
    def __radd__(self, o): return Mixed(None, [self]).__radd__(o)
    def __sub__(self, o): return Mixed(None, [self]) - o
    def __rsub__(self, o): return Mixed(None, [self]).__rsub__(o)


class Mixed:
    """vector expression + additive terms, split as vector.hpp:758-763 / operations.hpp:1463-1576."""
    __array_ufunc__ = None
    def __init__(self, vec: Optional[Node], terms):
        self.vec, self.terms = vec, list(terms)

    @staticmethod
    def of(x):
        if isinstance(x, Mixed): return x
        if isinstance(x, SpMVTerm): return Mixed(None, [x])
        return Mixed(wrap(x), [])

    def _combine(self, o, sign):
        o = Mixed.of(o)
        if self.vec is None:
            vec = o.vec if sign > 0 or o.vec is None else -o.vec
        elif o.vec is None:
            vec = self.vec
        else:
            vec = self.vec + o.vec if sign > 0 else self.vec - o.vec
        return Mixed(vec, self.terms + [t if sign > 0 else -t for t in o.terms])

    def __add__(self, o): return self._combine(o, +1)
    def __radd__(self, o): return Mixed.of(o)._combine(self, +1)
    def __sub__(self, o): return self._combine(o, -1)
    def __rsub__(self, o): return Mixed.of(o)._combine(self, -1)


def _node_add_mixed(self, o):
    if isinstance(o, Pointer):
        return o + self                                # i + p: pointer arithmetic, as in C
    return Mixed.of(self) + o if isinstance(o, (SpMVTerm, Mixed)) else Node._bin(self, "ADD", o)


def _node_sub_mixed(self, o):
    return Mixed.of(self) - o if isinstance(o, (SpMVTerm, Mixed)) else Node._bin(self, "SUB", o)


Node.__add__ = _node_add_mixed
Node.__sub__ = _node_sub_mixed


# ------------------------------------------------------------------------------------------- vector
class vector(Node):
    """vex::vector<T>: n elements split into contiguous slices, one per context slot."""

    def __init__(self, ctx: Context, data, dtype=None):
        lib = L.lib()
        self.ctx = ctx
        host = None
        if isinstance(data, (int, np.integer)):
            self.n = int(data)
            self.np_dtype = np.dtype(dtype or np.float64)
        else:
            host = np.ascontiguousarray(data, dtype=dtype)
            self.n = host.size
            self.np_dtype = host.dtype
        self.dtype = _vdt(self.np_dtype)
        self.part = ctx.partition(self.n)
        self.bufs = {}
        es = self.np_dtype.itemsize
        for k in ctx.local:
            p = C.c_void_p()
            L.check(lib.vexb_malloc(ctx.devs[k], self.part_size(k) * es, C.byref(p)))   # vector.hpp:918-928
            self.bufs[k] = p
        if host is not None:
            self.write(host)

    def __del__(self):
        try:
            lib = L.lib()
            for k, p in self.bufs.items():
                lib.vexb_free(self.ctx.devs[k], p)
        except Exception:
            pass

    def _bufarr(self):
        """The device pointers of the local slices as a C array (cached: the buffers live as long as the vector)."""
        a = self.__dict__.get("_bufarr_c")
        if a is None:
            a = self._bufarr_c = self.ctx._arr(self.bufs)
        return a

    def size(self): return self.n
    def nparts(self): return self.ctx.nparts
    def part_size(self, k): return int(self.part[k + 1] - self.part[k])
    def part_start(self, k): return int(self.part[k])
    def __len__(self): return self.n

    def write(self, host: np.ndarray, local_only: bool = False):
        """Host -> device.  `host` is the full vector (or, with local_only, just this rank's slice)."""
        lib = L.lib()
        host = np.ascontiguousarray(host, dtype=self.np_dtype)
        es = self.np_dtype.itemsize
        for k in self.ctx.local:
            lo, n = (0, self.part_size(k)) if local_only else (self.part_start(k), self.part_size(k))
            if n:
                src = host[lo:lo + n]
                L.check(lib.vexb_h2d(self.ctx.devs[k], self.bufs[k], src.ctypes.data, n * es, self.ctx.streams[k], 1))

    def read(self) -> np.ndarray:
        """Device -> host: the full vector in single-process mode, the local slice in distributed mode."""
        lib = L.lib()
        es = self.np_dtype.itemsize
        if self.ctx.is_distributed:
            k = self.ctx.local[0]
            out = np.empty(self.part_size(k), dtype=self.np_dtype)
            if out.size:
                L.check(lib.vexb_d2h(self.ctx.devs[k], out.ctypes.data, self.bufs[k], out.size * es, self.ctx.streams[k], 1))
            return out
        out = np.empty(self.n, dtype=self.np_dtype)
        for k in self.ctx.local:
            lo, n = self.part_start(k), self.part_size(k)
            if n:
                L.check(lib.vexb_d2h(self.ctx.devs[k], out[lo:].ctypes.data, self.bufs[k], n * es, self.ctx.streams[k], 1))
        return out

    def __getitem__(self, i: int):
        """Element read = 1-element copy (vector.hpp:232-245); only for locally held elements."""
        if not 0 <= i < self.n:
            raise IndexError(i)                                 # vector::at, vector.hpp:588-600
        k = int(np.searchsorted(self.part, i, side="right") - 1)
        while self.part_size(k) == 0:
            k += 1
        out = np.empty(1, dtype=self.np_dtype)
        es = self.np_dtype.itemsize
        L.check(L.lib().vexb_d2h(self.ctx.devs[k], out.ctypes.data, C.c_void_p(self.bufs[k].value + (i - self.part_start(k)) * es),
                                 es, self.ctx.streams[k], 1))
        return out[0]

    # -- assignment family (vector.hpp:666-801) ------------------------------------------------
    def _assign(self, op: int, rhs, sweep=True):
        if isinstance(rhs, SpMVTerm) and isinstance(rhs.A, SpMatCCSR) and op not in (L.SET, L.ADD, L.SUB):
            rhs = wrap(rhs)                 # y *= A*x: the product as an operand; =, += and -= keep the additive path
        if isinstance(rhs, (SpMVTerm, Mixed)):
            return self._assign_mixed(op, Mixed.of(rhs))
        rhs = wrap(rhs)
        lib = L.lib()
        for k in self.ctx.local:
            low = _Lowering(k, self.part_start(k))
            low.size = self.n
            low.target = self
            low.sweep = None if sweep else False
            low.see(self)
            low.lower(rhs)
            code = lib.vexb_eval(self.ctx.devs[k], self.ctx.streams[k], self.bufs[k], self.dtype, op,
                                 C.byref(low.e), self.part_size(k), self.part_start(k))
            copies = _redirect_pointers(low.e, [self]) if code == L.ERR_UNSUPPORTED else []
            if copies:
                # a pointer into the target: threads would read elements others overwrite, so every read goes to a copy
                code = lib.vexb_eval(self.ctx.devs[k], self.ctx.streams[k], self.bufs[k], self.dtype, op,
                                     C.byref(low.e), self.part_size(k), self.part_start(k))
            L.check(code)
        return self

    def _assign_mixed(self, op: int, m: Mixed):
        if op not in (L.SET, L.ADD, L.SUB):
            raise TypeError("additive operators only combine with =, += and -=")
        # every product inlinable (strips without a halo): the whole right-hand side is ONE generated kernel, e.g. `y = x + A*x`
        # reads A and x once and writes y once.  Same operation order as the unfused path below for `=`.
        if (m.vec is not None or len(m.terms) > 1) and len(m.terms) <= 6 and _is_float(self.dtype) and getattr(self.ctx, "fuse_products", True):
            nodes = [InlineSpMV(t.A, t.x) if isinstance(t.A, SpMat) and isinstance(t.x, vector) and t.x.n == t.A.m else None for t in m.terms]
            k0 = self.ctx.local[0]
            if all(nd is not None and (nd.strip(k0) is not None or nd.strip(k0, sweep=True) is not None) for nd in nodes):
                expr = m.vec
                for t, nd in zip(m.terms, nodes):
                    prod = Binary("MUL", Scalar(float(t.scale), self.dtype), nd)
                    expr = prod if expr is None else Binary("ADD", wrap(expr), prod)
                return self._assign(op, expr)
        sign = -1.0 if op == L.SUB else 1.0
        append = op != L.SET
        if m.vec is not None:
            self._assign(op, m.vec)          # vector part first ...
            append = True
        for t in m.terms:                    # ... then each additive term (vector.hpp:758-763)
            t.A.apply(t.x, self, sign * t.scale, append)
            append = True
        return self

    def assign(self, rhs): return self._assign(L.SET, rhs)
    def __iadd__(self, rhs): return self._assign(L.ADD, rhs)
    def __isub__(self, rhs): return self._assign(L.SUB, rhs)
    def __imul__(self, rhs): return self._assign(L.MUL, rhs)
    def __itruediv__(self, rhs): return self._assign(L.DIV, rhs)
    def __imod__(self, rhs): return self._assign(L.MOD, rhs)
    def __iand__(self, rhs): return self._assign(L.AND, rhs)
    def __ior__(self, rhs): return self._assign(L.OR, rhs)
    def __ixor__(self, rhs): return self._assign(L.XOR, rhs)
    def __ilshift__(self, rhs): return self._assign(L.LSH, rhs)
    def __irshift__(self, rhs): return self._assign(L.RSH, rhs)

    def eval_path(self, op: int, rhs) -> str:
        low = _Lowering(self.ctx.local[0], 0)
        low.size = self.n
        low.lower(wrap(rhs))
        buf = C.create_string_buffer(64)
        L.check(L.lib().vexb_eval_path(self.dtype, op, C.byref(low.e), buf, 64))
        return buf.value.decode()


def _redirect_pointers(e, targets) -> list:
    """Point every raw-pointer terminal of `e` that addresses one of `targets` at a device copy of that vector (what the
    back end asks for with VEXB_ERR_UNSUPPORTED: `x = p[(i + 1) % n]` with p = raw_pointer(x) then reads the old x).
    Returns the copies (to be kept until the launch is enqueued; freeing waits for the device), [] when none applies."""
    copies = []
    for v in targets:
        k = v.ctx.local[0]
        addr = v.bufs[k].value
        hits = [j for j in range(e.n_terms) if e.term[j].kind == L.TERM_PTR and e.term[j].v.ptr == addr]
        if not hits:
            continue
        cp = vector(v.ctx, v.n, v.np_dtype)
        L.check(L.lib().vexb_d2d(v.ctx.devs[k], cp.bufs[k], v.bufs[k], v.part_size(k) * v.np_dtype.itemsize, v.ctx.streams[k]))
        for j in hits:
            e.term[j].v.ptr = cp.bufs[k].value
        copies.append(cp)
    return copies


def _reduce_all_in_step(ctx, k, peer, dtype, kind, result, code, results):
    """A fused reduction that fails on slot k after earlier slots have launched would leave those kernels waiting for a
    peer that never comes and the mailbox epochs out of step: run the identity + the standalone combine on the slots that
    did not launch, then raise."""
    if code == L.OK:
        return
    msg = L.lib().vexb_last_error().decode(errors="replace")
    if peer is not None and len(ctx.local) > 1:
        lib = L.lib()
        for j in ctx.local[ctx.local.index(k):]:
            lib.vexb_reduce_identity(ctx.devs[j], ctx.streams[j], dtype, kind, results[j])
            lib.vexb_peer_allreduce(ctx.peers[j], ctx.streams[j], results[j], dtype, kind)
    raise L.VexbError(code, msg)


def check_peer_fault():
    """Raise if any kernel of this process gave up waiting for a peer GPU (its results are NaN / all-ones, never stale)."""
    e = C.c_uint64(0)
    L.lib().vexb_peer_fault(C.byref(e), 0)
    if e.value:
        raise L.VexbError(L.ERR_PEER, f"a peer GPU did not arrive within the time limit (epoch {e.value}); dependent results are poisoned")


# ------------------------------------------------------------------------------------------- Reductor
class Reductor:
    """vex::Reductor<T, RDC> (reductor.hpp:289-439).  kind: L.SUM, L.SUM_KAHAN, L.MAX, L.MIN, L.MINMAX."""

    def __init__(self, ctx: Context, dtype=np.float64, kind=L.SUM):
        """kind: one of L.SUM, L.SUM_KAHAN, L.MAX, L.MIN, L.MINMAX -- or a sequence of the first four:
        vex::CombineReductors<R...> (reductor.hpp:132-280), several reductions of one expression in one pass; the call
        then returns a tuple."""
        self.ctx, self.np_dtype, self.dtype = ctx, np.dtype(dtype), _vdt(dtype)
        self.kinds = list(kind) if isinstance(kind, (list, tuple)) else None
        self.kind = kind if self.kinds is None else None
        if self.kinds is not None and not (1 <= len(self.kinds) <= 16 and all(k in (L.SUM, L.SUM_KAHAN, L.MAX, L.MIN) for k in self.kinds)):
            raise ValueError("between 1 and 16 of SUM, SUM_KAHAN, MAX, MIN can be combined")

    def _combined(self, expr, n, part):
        """vexb_reduce_multi on every slot, then combine across slots (inside the kernel with a peer group)."""
        lib, ctx, K = L.lib(), self.ctx, len(self.kinds)
        ops = (C.c_int * K)(*self.kinds)
        es = self.np_dtype.itemsize
        fused = ctx.peers is not None and ctx.use_peer_reduce and ctx.nparts > 1
        res = {}
        for k in ctx.local:
            ws, r = ctx.workspace(k, K)
            low = _Lowering(k, int(part[k]))
            low.lower(expr)
            code = lib.vexb_reduce_multi(ctx.devs[k], ctx.streams[k], C.byref(low.e), self.dtype, int(part[k + 1] - part[k]), int(part[k]),
                                         K, ops, r, ws, ctx.peers[k] if fused else None)
            if code == L.ERR_UNSUPPORTED and k == ctx.local[0] and _has_call(expr):
                return self._combined(_temporary(ctx, expr, n), n, part)       # no NVRTC: reduce a temporary
            L.check(code)
            res[k] = r
        out = np.empty(K, dtype=self.np_dtype)
        k0 = ctx.local[0]
        if ctx.nparts > 1 and not fused and ctx.comms is not None:
            for j, op in enumerate(self.kinds):
                bufs = {k: C.c_void_p(res[k].value + j * es) for k in ctx.local}
                L.check(lib.vexb_comm_allreduce(len(ctx.local), ctx._arr(ctx.comms), ctx._arr(bufs), ctx._arr(ctx.streams), 1, self.dtype, op))
        if ctx.nparts == 1 or fused or ctx.comms is not None:
            L.check(lib.vexb_reduce_fetch(ctx.devs[k0], ctx.streams[k0], res[k0], self.dtype, K, out.ctypes.data))
            return tuple(out)
        if ctx.is_distributed:
            raise RuntimeError("distributed context without a communicator")
        acc = None
        for k in ctx.local:                                        # device order, like reductor.hpp:420-436
            L.check(lib.vexb_reduce_fetch(ctx.devs[k], ctx.streams[k], res[k], self.dtype, K, out.ctypes.data))
            v = out.copy()
            if acc is None:
                acc = v
            else:
                for j, op in enumerate(self.kinds):
                    acc[j] = acc[j] + v[j] if op in (L.SUM, L.SUM_KAHAN) else max(acc[j], v[j]) if op == L.MAX else min(acc[j], v[j])
        return tuple(acc)

    def __call__(self, expr):
        lib = L.lib()
        ctx = self.ctx
        expr = wrap(expr)
        props = _find_props(expr)
        if props is None:
            raise ValueError("expression has no vector terminal")
        n = props[1]
        expr = _reduce_in_one_pass(ctx, expr, n)
        part = ctx.partition(n)
        if self.kinds is not None:
            return self._combined(expr, n, part)
        cnt = 2 if self.kind == L.MINMAX else 1
        res = {}
        for k in ctx.local:
            ws, r = ctx.workspace(k)
            low = _Lowering(k, int(part[k]))
            low.lower(expr)
            peer = ctx.peers[k] if (ctx.peers is not None and ctx.use_peer_reduce and ctx.nparts > 1) else None
            code = lib.vexb_reduce_all(ctx.devs[k], ctx.streams[k], C.byref(low.e), self.dtype, int(part[k + 1] - part[k]),
                                       int(part[k]), self.kind, r, ws, peer)
            if code == L.ERR_UNSUPPORTED and k == ctx.local[0] and _has_call(expr):
                return self(_temporary(ctx, expr, n))                          # no NVRTC: reduce a temporary
            _reduce_all_in_step(ctx, k, peer, self.dtype, self.kind, r, code, {j: ctx.workspace(j)[1] for j in ctx.local})
            res[k] = r
        out = np.empty(cnt, dtype=self.np_dtype)
        if ctx.nparts > 1 and ctx.peers is not None and ctx.use_peer_reduce:
            k = ctx.local[0]                                       # combined inside the kernel over peer memory
            L.check(lib.vexb_reduce_fetch(ctx.devs[k], ctx.streams[k], res[k], self.dtype, cnt, out.ctypes.data))
        elif ctx.nparts > 1 and ctx.comms is not None:
            # combine over NVLink (replaces the host fold, reductor.hpp:412-436)
            L.check(lib.vexb_comm_allreduce(len(ctx.local), ctx._arr(ctx.comms), ctx._arr(res), ctx._arr(ctx.streams),
                                            1, self.dtype, self.kind))
            k = ctx.local[0]
            L.check(lib.vexb_reduce_fetch(ctx.devs[k], ctx.streams[k], res[k], self.dtype, cnt, out.ctypes.data))
        else:
            if ctx.is_distributed and ctx.nparts > 1:
                raise RuntimeError("distributed context without a communicator")
            acc = None
            for k in ctx.local:                                    # device order, like reductor.hpp:420-436
                L.check(lib.vexb_reduce_fetch(ctx.devs[k], ctx.streams[k], res[k], self.dtype, cnt, out.ctypes.data))
                v = out.copy()
                if acc is None:
                    acc = v
                elif self.kind in (L.SUM, L.SUM_KAHAN):
                    acc = acc + v
                elif self.kind == L.MAX:
                    acc = np.maximum(acc, v)
                elif self.kind == L.MIN:
                    acc = np.minimum(acc, v)
                else:
                    acc = np.array([min(acc[0], v[0]), max(acc[1], v[1])], dtype=self.np_dtype)
            out = acc
        return (out[0], out[1]) if cnt == 2 else out[0]


# ------------------------------------------------------------------------------------------- SpMat
def _ip(a): return a.ctypes.data_as(C.c_void_p)


class SpMat:
    """vex::SpMat<val_t, col_t, idx_t> (spmat.hpp:56-386): CSR in, one strip per device, ghost exchange."""

    def __init__(self, ctx: Context, n: int, m: int, row, col, val, fmt: int = L.FMT_AUTO, strip: bool = False):
        """row/col/val: the whole matrix, or -- with strip=True, in distributed mode -- only this rank's
        rows [part[r], part[r+1]) with global column ids (row offsets may start anywhere)."""
        lib = L.lib()
        self.ctx, self.n, self.m, self.fmt = ctx, n, m, fmt
        self.row = np.ascontiguousarray(row)
        self.col = np.ascontiguousarray(col)
        self.val = np.ascontiguousarray(val)
        if self.row.dtype.itemsize not in (4, 8) or self.col.dtype.itemsize not in (4, 8):
            raise TypeError("row/col must be 32- or 64-bit integers")
        self.val_dtype = _vdt(self.val.dtype)
        self.part = ctx.partition(n)
        self.col_part = ctx.partition(m)                                        # spmat.hpp:74, :78
        rb, cb = self.row.dtype.itemsize, self.col.dtype.itemsize
        self.nnz = int(self.row[-1] - self.row[0]) if strip else int(self.row[n])
        # ghost columns of every part
        ghosts = {}
        self._strips = {}
        for k in ctx.local:
            r0, r1 = (0, int(self.part[k + 1] - self.part[k])) if strip else (int(self.part[k]), int(self.part[k + 1]))
            prow = self.row[r0:r1 + 1]
            j0 = int(prow[0]) if prow.size else 0
            base = int(self.row[0]) if strip else 0
            pcol = self.col[j0 - base:]
            pval = self.val[j0 - base:]
            self._strips[k] = (r1 - r0, prow, pcol, pval)
            cnt = C.c_size_t(0)
            if ctx.nparts > 1:
                L.check(lib.vexb_strip_ghost_cols(r1 - r0, _ip(prow), rb, _ip(pcol), cb, int(self.col_part[k]),
                                                  int(self.col_part[k + 1]), None, C.byref(cnt)))
                g = np.empty(cnt.value, dtype=np.int64)
                cap = C.c_size_t(cnt.value)
                L.check(lib.vexb_strip_ghost_cols(r1 - r0, _ip(prow), rb, _ip(pcol), cb, int(self.col_part[k]),
                                                  int(self.col_part[k + 1]), _ip(g), C.byref(cap)))
            else:
                g = np.empty(0, dtype=np.int64)
            ghosts[k] = g
        if ctx.is_distributed:
            all_g = ctx.allgather(ghosts[ctx.local[0]])
            ghosts = {k: np.ascontiguousarray(g, dtype=np.int64) for k, g in enumerate(all_g)}
        self.ghosts = ghosts
        off = np.zeros(ctx.nparts + 1, dtype=np.uint64)
        for k in range(ctx.nparts):
            off[k + 1] = off[k] + len(ghosts[k])
        cat = np.concatenate([ghosts[k] for k in range(ctx.nparts)]) if off[-1] else np.empty(0, np.int64)
        cat = np.ascontiguousarray(cat, dtype=np.int64)
        cp = (C.c_size_t * (ctx.nparts + 1))(*[int(x) for x in self.col_part])
        go = (C.c_size_t * (ctx.nparts + 1))(*[int(x) for x in off])
        self.plan = C.c_void_p()
        L.check(lib.vexb_halo_plan_create(ctx.nparts, cp, _ip(cat), go, C.byref(self.plan)))
        self.parts = {}
        for k in ctx.local:
            nrows, prow, pcol, pval = self._strips[k]
            h = C.c_void_p()
            L.check(lib.vexb_dspmat_create(ctx.devs[k], ctx.streams[k], k, self.plan, nrows, _ip(prow), rb, _ip(pcol), cb,
                                           _ip(pval), self.val_dtype, fmt, C.byref(h)))
            self.parts[k] = h
        self._strips = None
        self.peer_halo = False
        if ctx.nparts > 1 and ctx.nparts <= 16 and getattr(ctx, "peer_halo", False):
            self.peer_halo = self._connect_peer_halo()

    def _connect_peer_halo(self) -> bool:
        """Map the neighbours' ghost boxes (CUDA IPC between processes, peer access inside one).  All or nothing across
        the parts: if any part cannot connect, every part goes back to NCCL / copies (no rank may wait on a missing peer)."""
        lib, ctx = L.lib(), self.ctx
        if ctx.is_distributed:
            k = ctx.local[0]
            h = C.create_string_buffer(64)
            ok = lib.vexb_dspmat_halo_handle(self.parts[k], h) == L.OK
            allh = ctx.allgather(np.frombuffer(h.raw, dtype=np.uint8).copy())
            if ok:
                cat = b"".join(np.asarray(a, dtype=np.uint8).tobytes() for a in allh)
                ok = lib.vexb_dspmat_halo_connect(self.parts[k], C.create_string_buffer(cat, 64 * ctx.nparts)) == L.OK
            everybody = ctx.allgather(np.array([1 if ok else 0], dtype=np.int64))
            ok = all(int(np.asarray(a)[0]) == 1 for a in everybody)
        else:
            ok = lib.vexb_dspmat_halo_connect_local(len(ctx.local), ctx._arr(self.parts)) == L.OK
        if not ok:
            for h in self.parts.values():
                lib.vexb_dspmat_halo_disconnect(h)
        return ok

    def __del__(self):
        try:
            lib = L.lib()
            for h in self.parts.values():
                lib.vexb_dspmat_destroy(h)
            lib.vexb_halo_plan_destroy(self.plan)
        except Exception:
            pass

    def rows(self): return self.n
    def cols(self): return self.m
    def nonzeros(self): return self.nnz

    def info(self, k=None) -> L.DspmatInfo:
        info = L.DspmatInfo()
        L.check(L.lib().vexb_dspmat_get_info(self.parts[self.ctx.local[0] if k is None else k], C.byref(info)))
        return info

    def __mul__(self, x):
        if not isinstance(x, vector):
            return NotImplemented
        return SpMVTerm(self, x)

    def apply(self, x: vector, y: vector, alpha: float = 1.0, append: bool = False):
        """y = alpha*A*x  or  y += alpha*A*x  (spmat.hpp:120-185)."""
        ctx = self.ctx
        if x.n != self.m or y.n != self.n:
            raise ValueError("SpMat::apply: vector sizes do not match the matrix")
        fixed = self.__dict__.get("_apply_args")
        if fixed is None or fixed[3] is not ctx.streams:          # the handle tables never change: build them once
            fixed = self._apply_args = (len(ctx.local), ctx._arr(ctx.comms) if ctx.comms is not None else None, ctx._arr(self.parts),
                                        ctx.streams, ctx._arr(ctx.streams), L.lib().vexb_dspmat_apply)
        code = fixed[5](fixed[0], fixed[1], fixed[2], fixed[4], x._bufarr(), y._bufarr(), alpha, 1 if append else 0)
        if code:
            L.check(code)
        return y


def _spmat_apply_dot(self, x: "vector", y: "vector", out: "DeviceScalar", dot_with: Optional["vector"] = None,
                     alpha: float = 1.0, append: bool = False) -> bool:
    """y (=|+=) alpha*A*x and out = dot(dot_with or x, y) on every device.  The dot partials come out of the product kernel (plus a one-block fold launch) when the matrix has the
    peer-memory halo (or a single part) and a hybrid- or sliced-ELL interior (vexb_dspmat_apply_dot); otherwise the product followed
    by a device-resident reduction.  Returns True when the fused kernel ran."""
    ctx, lib = self.ctx, L.lib()
    w = x if dot_with is None else dot_with
    if x.n != self.m or y.n != self.n or w.n != self.n:
        raise ValueError("SpMat::apply_dot: vector sizes do not match the matrix")
    if getattr(self, "_fused_dot", True):
        peers = ctx._arr(ctx.peers) if (ctx.peers is not None and ctx.nparts > 1) else None
        if ctx.nparts == 1 or peers is not None:
            code = lib.vexb_dspmat_apply_dot(len(ctx.local), ctx._arr(self.parts), ctx._arr(ctx.streams), ctx._arr(x.bufs),
                                             ctx._arr(y.bufs), float(alpha), int(append), ctx._arr(w.bufs), ctx._arr(out.bufs), peers)
            if code == L.OK:
                return True
            if code != L.ERR_UNSUPPORTED:
                L.check(code)
        self._fused_dot = False                        # not available for this matrix: do not ask again
    self.apply(x, y, alpha, append)
    Reductor(ctx, w.np_dtype, L.SUM).device(w * y, out)
    return False


SpMat.apply_dot = _spmat_apply_dot


def _spmat_apply_multi(self, xs, ys, alpha: float = 1.0, append: bool = False):
    """ys[r] (=|+=) alpha*A*xs[r] for every r: vex::SpMat * vex::multivector.  Strips without a halo read the matrix once per
    group of up to four vectors (vexb_dspmat_apply_multi); the reference multiplies component by component."""
    ctx, nrhs = self.ctx, len(xs)
    if nrhs != len(ys) or nrhs < 1 or any(x.n != self.m for x in xs) or any(y.n != self.n for y in ys):
        raise ValueError("SpMat::apply_multi: vector counts or sizes do not match the matrix")
    xa = (C.c_void_p * (len(ctx.local) * nrhs))(*[xs[r].bufs[k] for k in ctx.local for r in range(nrhs)])
    ya = (C.c_void_p * (len(ctx.local) * nrhs))(*[ys[r].bufs[k] for k in ctx.local for r in range(nrhs)])
    comms = ctx._arr(ctx.comms) if ctx.comms is not None else None
    L.check(L.lib().vexb_dspmat_apply_multi(len(ctx.local), comms, ctx._arr(self.parts), ctx._arr(ctx.streams), nrhs, xa, ya,
                                            float(alpha), int(append)))
    return ys


SpMat.apply_multi = _spmat_apply_multi


class SpMatCCSR:
    """vex::SpMatCCSR<val_t, col_t, idx_t> (spmat/ccsr.hpp:54-86): unique rows with diagonal-relative columns.
    Single device, like the reference: the context must have one slot."""

    def __init__(self, ctx: Context, n: int, idx, row, col, val):
        if ctx.nparts != 1:
            raise ValueError("SpMatCCSR does not support multi-device contexts (ccsr.hpp:49-52)")
        self.ctx, self.n = ctx, int(n)
        idx, row = np.ascontiguousarray(idx), np.ascontiguousarray(row)
        col, val = np.ascontiguousarray(col), np.ascontiguousarray(val)
        if idx.dtype.itemsize not in (4, 8) or row.dtype.itemsize not in (4, 8) or col.dtype.itemsize not in (4, 8):
            raise TypeError("idx/row/col must be 32- or 64-bit integers")
        if col.dtype.kind != "i":
            raise TypeError("Column type for CCSR format has to be signed.")           # ccsr.hpp:56-57
        self.m = row.size - 1
        self.val_dtype = _vdt(val.dtype)
        self.h = C.c_void_p()
        k = ctx.local[0]
        L.check(L.lib().vexb_ccsr_create(ctx.devs[k], ctx.streams[k], self.n, self.m, _ip(idx), idx.dtype.itemsize,
                                         _ip(row), row.dtype.itemsize, _ip(col), col.dtype.itemsize, _ip(val),
                                         self.val_dtype, C.byref(self.h)))
        self.idx_bytes = self.info().idx_bytes              # width of idx on the device: part of a terminal's kernel shape

    def __del__(self):
        try:
            L.lib().vexb_ccsr_destroy(self.h)
        except Exception:
            pass

    def rows(self): return self.n
    def cols(self): return self.n

    def info(self) -> L.CcsrInfo:
        info = L.CcsrInfo()
        L.check(L.lib().vexb_ccsr_get_info(self.h, C.byref(info)))
        return info

    def __mul__(self, x):
        if not isinstance(x, vector):
            return NotImplemented
        return SpMVTerm(self, x)

    def apply(self, x: vector, y: vector, alpha: float = 1.0, append: bool = False):
        if x.n != self.n or y.n != self.n:
            raise ValueError("SpMatCCSR::apply: vector sizes do not match the matrix")
        k = self.ctx.local[0]
        L.check(L.lib().vexb_ccsr_spmv(self.ctx.devs[k], self.ctx.streams[k], self.h, x.bufs[k], y.bufs[k], float(alpha), int(append)))
        return y


class BlockMatrix:
    """vex::sparse::matrix<std::array<std::array<T,B>,B>> (the reference's custom value types, sparse/distributed.hpp:17-21):
    ptr/col count block rows and block columns, val has shape (nnzb, B, B), B = 2, 3 or 4.  x and y are plain vectors of
    m*B and n*B scalars -- the bytes of vex::vector<std::array<T,B>>.  Single device."""

    def __init__(self, ctx: Context, n: int, m: int, ptr, col, val):
        if ctx.nparts != 1:
            raise ValueError("block sparse matrices are only supported for single-device contexts")
        self.ctx, self.n, self.m = ctx, int(n), int(m)
        ptr, col, val = np.ascontiguousarray(ptr), np.ascontiguousarray(col), np.ascontiguousarray(val)
        if ptr.dtype.itemsize not in (4, 8) or col.dtype.itemsize not in (4, 8):
            raise TypeError("ptr/col must be 32- or 64-bit integers")
        if val.ndim != 3 or val.shape[1] != val.shape[2]:
            raise ValueError("val must have shape (nnzb, B, B)")
        self.block = int(val.shape[1])
        self.nnzb = int(val.shape[0])
        self.val_dtype = _vdt(val.dtype)
        self.h = C.c_void_p()
        k = ctx.local[0]
        L.check(L.lib().vexb_bsr_create(ctx.devs[k], ctx.streams[k], self.n, self.m, self.block, _ip(ptr), ptr.dtype.itemsize,
                                        _ip(col), col.dtype.itemsize, _ip(val), self.val_dtype, C.byref(self.h)))

    def __del__(self):
        try:
            L.lib().vexb_bspmat_destroy(self.h)
        except Exception:
            pass

    def rows(self): return self.n
    def cols(self): return self.m
    def nonzeros(self): return self.nnzb

    def info(self) -> L.BspmatInfo:
        info = L.BspmatInfo()
        L.check(L.lib().vexb_bspmat_get_info(self.h, C.byref(info)))
        return info

    def apply(self, x: vector, y: vector, alpha: float = 1.0, append: bool = False):
        """y = alpha*A*x  or  y += alpha*A*x, one launch."""
        if x.n != self.m * self.block or y.n != self.n * self.block:
            raise ValueError("BlockMatrix::apply: vector sizes do not match the matrix")
        if x.dtype != self.val_dtype or y.dtype != self.val_dtype:
            raise TypeError("BlockMatrix::apply: vectors must have the matrix's value type")
        k = self.ctx.local[0]
        L.check(L.lib().vexb_bspmv(self.ctx.devs[k], self.ctx.streams[k], self.h, x.bufs[k], y.bufs[k], float(alpha), int(append)))
        return y


class ComplexMatrix:
    """vex::sparse::matrix<std::complex<T>> (the reference's examples/complex_spmv.cpp): val is complex128 or complex64.  x
    and y are plain vectors of 2*m and 2*n scalars of the matching real type, the bytes of vex::vector<std::complex<T>>:
    vector(ctx, z.view(np.float64)).  alpha is real.  Single device."""

    def __init__(self, ctx: Context, n: int, m: int, ptr, col, val):
        if ctx.nparts != 1:
            raise ValueError("complex sparse matrices are only supported for single-device contexts")
        self.ctx, self.n, self.m = ctx, int(n), int(m)
        ptr, col, val = np.ascontiguousarray(ptr), np.ascontiguousarray(col), np.ascontiguousarray(val)
        if ptr.dtype.itemsize not in (4, 8) or col.dtype.itemsize not in (4, 8):
            raise TypeError("ptr/col must be 32- or 64-bit integers")
        if val.dtype not in (np.complex128, np.complex64) or val.ndim != 1:
            raise TypeError("val must be a 1-d complex128 or complex64 array")
        self.nnz = int(val.size)
        self.val_dtype = L.F64 if val.dtype == np.complex128 else L.F32
        self.h = C.c_void_p()
        k = ctx.local[0]
        L.check(L.lib().vexb_zsr_create(ctx.devs[k], ctx.streams[k], self.n, self.m, _ip(ptr), ptr.dtype.itemsize,
                                        _ip(col), col.dtype.itemsize, _ip(val), self.val_dtype, C.byref(self.h)))

    def __del__(self):
        try:
            L.lib().vexb_zspmat_destroy(self.h)
        except Exception:
            pass

    def rows(self): return self.n
    def cols(self): return self.m
    def nonzeros(self): return self.nnz

    def info(self) -> L.ZspmatInfo:
        info = L.ZspmatInfo()
        L.check(L.lib().vexb_zspmat_get_info(self.h, C.byref(info)))
        return info

    def apply(self, x: vector, y: vector, alpha: float = 1.0, append: bool = False):
        """y = alpha*A*x  or  y += alpha*A*x, one launch."""
        if x.n != 2 * self.m or y.n != 2 * self.n:
            raise ValueError("ComplexMatrix::apply: vector sizes do not match the matrix")
        if x.dtype != self.val_dtype or y.dtype != self.val_dtype:
            raise TypeError("ComplexMatrix::apply: vectors must have the real type of the matrix's values")
        k = self.ctx.local[0]
        L.check(L.lib().vexb_zspmv(self.ctx.devs[k], self.ctx.streams[k], self.h, x.bufs[k], y.bufs[k], float(alpha), int(append)))
        return y


class UserValueMatrix:
    """vex::sparse::matrix<V> of a user value type V with its spmv_ops_impl<V, X> (the reference's sparse/spmv_ops.hpp).
    val has shape (nnz, k): row j is the bytes of value j (k * itemsize bytes, a multiple of 4 up to 64).  val_type and
    rhs_type name the device types of V and X (e.g. "double4", "double2"), rhs_bytes is sizeof(X).  decl, product and
    append are the snippets of decl_accum_var(src, "sum"), append_product(src, "sum", "v", "xv") and append(src, "t",
    "sum").  x and y are plain vectors of scalars holding the bytes of m and n X.  Single device."""

    def __init__(self, ctx: Context, n: int, m: int, ptr, col, val, val_type: str, rhs_type: str, rhs_bytes: int,
                 decl: str, product: str, append: str):
        if ctx.nparts != 1:
            raise ValueError("sparse matrices of user value types are only supported for single-device contexts")
        self.ctx, self.n, self.m = ctx, int(n), int(m)
        ptr, col, val = np.ascontiguousarray(ptr), np.ascontiguousarray(col), np.ascontiguousarray(val)
        if ptr.dtype.itemsize not in (4, 8) or col.dtype.itemsize not in (4, 8):
            raise TypeError("ptr/col must be 32- or 64-bit integers")
        if val.ndim != 2:
            raise ValueError("val must have shape (nnz, k): one row of value bytes per stored entry")
        self.nnz = int(val.shape[0])
        self.val_bytes = int(val.shape[1] * val.dtype.itemsize)
        self.rhs_bytes = int(rhs_bytes)
        self._strs = [s.encode() for s in (val_type, rhs_type, decl, product, append)]      # kept alive for ops
        vt, rt, d, p, a = self._strs
        self.ops = L.UsrOps(vt, rt, self.rhs_bytes, d, p, a)
        self.h = C.c_void_p()
        k = ctx.local[0]
        L.check(L.lib().vexb_usr_create(ctx.devs[k], ctx.streams[k], self.n, self.m, _ip(ptr), ptr.dtype.itemsize,
                                        _ip(col), col.dtype.itemsize, _ip(val), self.val_bytes, C.byref(self.h)))

    def __del__(self):
        try:
            L.lib().vexb_usrmat_destroy(self.h)
        except Exception:
            pass

    def rows(self): return self.n
    def cols(self): return self.m
    def nonzeros(self): return self.nnz

    def info(self) -> L.UsrmatInfo:
        info = L.UsrmatInfo()
        L.check(L.lib().vexb_usrmat_get_info(self.h, C.byref(info)))
        return info

    def apply(self, x: vector, y: vector, append: bool = False):
        """y = A*x  or  y += A*x, one launch of the generated kernel (compiled at the first call on a device)."""
        xb, yb = x.n * x.np_dtype.itemsize, y.n * y.np_dtype.itemsize
        if xb != self.m * self.rhs_bytes or yb != self.n * self.rhs_bytes:
            raise ValueError("UserValueMatrix::apply: vector sizes do not match the matrix")
        k = self.ctx.local[0]
        L.check(L.lib().vexb_usr_spmv(self.ctx.devs[k], self.ctx.streams[k], self.h, C.byref(self.ops), x.bufs[k], y.bufs[k],
                                      int(append)))
        return y


class stencil:
    """vex::stencil<T> (stencil.hpp:168-330): `y = x * s`, `y += x * s`, `y = 42 * (x * s)`, ...
    y[i] = sum_k s[k] * x[clamp(i + k - center)]; with several slices the neighbours' edge elements are copied
    device to device into per-slice halo buffers first (stencil_base::exchange_halos, stencil.hpp:86-150)."""

    def __init__(self, ctx: Context, s, center: int, dtype=np.float64):
        if ctx.is_distributed:
            raise NotImplementedError("stencil: one process per GPU is not wired up yet")
        self.ctx = ctx
        self.s = np.ascontiguousarray(s, dtype=dtype)
        self.width, self.center = int(self.s.size), int(center)
        if not (self.width >= 1 and 0 <= self.center < self.width):
            raise ValueError("stencil needs width >= 1 and 0 <= center < width")      # stencil.hpp:70-74
        self.lhalo, self.rhalo = self.center, self.width - self.center - 1
        self.dtype = _vdt(self.s.dtype)
        lib, es = L.lib(), self.s.dtype.itemsize
        self.sdev, self.halo = {}, {}
        for k in ctx.local:
            p, h = C.c_void_p(), C.c_void_p()
            L.check(lib.vexb_malloc(ctx.devs[k], self.width * es, C.byref(p)))
            L.check(lib.vexb_h2d(ctx.devs[k], p, self.s.ctypes.data, self.width * es, ctx.streams[k], 1))
            L.check(lib.vexb_malloc(ctx.devs[k], max(self.width - 1, 1) * es, C.byref(h)))
            self.sdev[k], self.halo[k] = p, h

    def __del__(self):
        try:
            for k in self.sdev:
                L.lib().vexb_free(self.ctx.devs[k], self.sdev[k])
                L.lib().vexb_free(self.ctx.devs[k], self.halo[k])
        except Exception:
            pass

    def __mul__(self, x):
        return SpMVTerm(self, x) if isinstance(x, vector) else NotImplemented
    __rmul__ = __mul__

    def _fill(self, k, ptr, count, value):
        low = _Lowering(k, 0)
        low.size = count
        low.lower(Scalar(value, self.dtype))
        L.check(L.lib().vexb_eval(self.ctx.devs[k], self.ctx.streams[k], ptr, self.dtype, L.SET, C.byref(low.e), count, 0))

    def _gather(self, x: vector, k: int, dst_off: int, g0: int, g1: int):
        """Copy global elements [g0, g1) of x into slice k's halo buffer at element offset dst_off."""
        ctx, es, lib = self.ctx, self.s.dtype.itemsize, L.lib()
        for p in range(ctx.nparts):
            a, b = max(g0, x.part_start(p)), min(g1, x.part_start(p) + x.part_size(p))
            if a < b:
                L.check(lib.vexb_copy_peer(ctx.devs[k], C.c_void_p(self.halo[k].value + (dst_off + a - g0) * es), ctx.devs[p],
                                           C.c_void_p(x.bufs[p].value + (a - x.part_start(p)) * es), (b - a) * es, ctx.streams[k]))

    def exchange_halos(self, x: vector):
        """Returns {slice: (left pointer or None, right pointer or None)}."""
        ctx, n, es = self.ctx, x.n, self.s.dtype.itemsize
        sides = {k: (None, None) for k in ctx.local}
        if ctx.nparts <= 1 or self.width == 1:
            return sides
        ctx.finish()                                     # the neighbours' slices must be complete (stencil.hpp:113)
        for k in ctx.local:
            start, size = x.part_start(k), x.part_size(k)
            if not size:
                continue
            left = right = None
            if start > 0 and self.lhalo:
                g0 = start - self.lhalo
                if g0 < 0:                               # fewer elements before this slice than the stencil reaches
                    self._fill(k, self.halo[k], -g0, x[0])
                self._gather(x, k, max(0, -g0), max(g0, 0), start)
                left = self.halo[k]
            if start + size < n and self.rhalo:
                g0, g1 = start + size, min(start + size + self.rhalo, n)
                self._gather(x, k, self.lhalo, g0, g1)
                if g1 - g0 < self.rhalo:
                    self._fill(k, C.c_void_p(self.halo[k].value + (self.lhalo + g1 - g0) * es), self.rhalo - (g1 - g0), x[n - 1])
                right = C.c_void_p(self.halo[k].value + self.lhalo * es)
            sides[k] = (left, right)
        ctx.finish()                                     # nobody may overwrite x while a neighbour still copies from it
        return sides

    def apply(self, x: vector, y: vector, alpha: float = 1.0, append: bool = False):
        if x.n != y.n or x.dtype != self.dtype or y.dtype != self.dtype:
            raise ValueError("stencil: vectors must have the stencil's type and equal sizes")
        sides = self.exchange_halos(x)
        for k in self.ctx.local:
            left, right = sides[k]
            L.check(L.lib().vexb_stencil_apply(self.ctx.devs[k], self.ctx.streams[k], self.dtype, self.sdev[k], self.width,
                                               self.center, x.bufs[k], x.part_size(k), left, right, y.bufs[k], float(alpha), int(append)))
        return y


# ------------------------------------------------------------------------------------------- helpers for timing / host staging
class PinnedArray:
    """Page-locked host buffer exposed as a numpy array (.a)."""

    def __init__(self, n: int, dtype=np.float64):
        self.ptr = C.c_void_p()
        dt = np.dtype(dtype)
        L.check(L.lib().vexb_host_alloc(max(n, 1) * dt.itemsize, C.byref(self.ptr)))
        buf = (C.c_char * (max(n, 1) * dt.itemsize)).from_address(self.ptr.value)
        self.a = np.frombuffer(buf, dtype=dt, count=n)

    def __del__(self):
        try:
            self.a = None
            L.lib().vexb_host_free(self.ptr)
        except Exception:
            pass


def copy_h2d_async(v: vector, host: np.ndarray, k: Optional[int] = None):
    """Non-blocking host -> device copy of part k's slice (host holds exactly that slice)."""
    k = v.ctx.local[0] if k is None else k
    L.check(L.lib().vexb_h2d(v.ctx.devs[k], v.bufs[k], host.ctypes.data, v.part_size(k) * v.np_dtype.itemsize, v.ctx.streams[k], 0))


def copy_d2h_async(v: vector, host: np.ndarray, k: Optional[int] = None):
    k = v.ctx.local[0] if k is None else k
    L.check(L.lib().vexb_d2h(v.ctx.devs[k], host.ctypes.data, v.bufs[k], v.part_size(k) * v.np_dtype.itemsize, v.ctx.streams[k], 0))


class Event:
    def __init__(self, ctx: Context, k: Optional[int] = None):
        self.ctx, self.k = ctx, ctx.local[0] if k is None else k
        self.h = C.c_void_p()
        L.check(L.lib().vexb_event_create(ctx.devs[self.k], C.byref(self.h)))

    def record(self):
        L.check(L.lib().vexb_event_record(self.ctx.devs[self.k], self.h, self.ctx.streams[self.k]))

    def sync(self):
        L.check(L.lib().vexb_event_sync(self.ctx.devs[self.k], self.h))

    def elapsed_ms(self, later: "Event") -> float:
        ms = C.c_float()
        L.check(L.lib().vexb_event_elapsed_ms(self.h, later.h, C.byref(ms)))
        return ms.value


# ------------------------------------------------------------------------------------------- device-resident scalars, graphs
class DeviceScalar(Node):
    """One value per device slot, kept in device memory (VEXB_TERM_DSCALAR).  A Reductor can leave its
    result here (`Reductor.device`), scalar arithmetic on it is an n = 1 elementwise evaluation, and any
    vector expression can use it as a coefficient -- so an iteration such as CG needs no host round trip
    for alpha / beta and can be captured in a CUDA graph."""

    def __init__(self, ctx: Context, dtype=np.float64, value=0):
        lib = L.lib()
        self.ctx, self.np_dtype, self.dtype = ctx, np.dtype(dtype), _vdt(dtype)
        self.bufs = {}
        for k in ctx.local:
            p = C.c_void_p()
            L.check(lib.vexb_malloc(ctx.devs[k], 64, C.byref(p)))
            self.bufs[k] = p
        self.set(value)

    def __del__(self):
        try:
            for k, p in self.bufs.items():
                L.lib().vexb_free(self.ctx.devs[k], p)
        except Exception:
            pass

    def set(self, value):
        h = np.full(2, value, dtype=self.np_dtype)
        for k in self.ctx.local:
            L.check(L.lib().vexb_h2d(self.ctx.devs[k], self.bufs[k], h.ctypes.data, 2 * self.np_dtype.itemsize, self.ctx.streams[k], 1))

    def get(self):
        k = self.ctx.local[0]
        h = np.empty(1, dtype=self.np_dtype)
        L.check(L.lib().vexb_d2h(self.ctx.devs[k], h.ctypes.data, self.bufs[k], self.np_dtype.itemsize, self.ctx.streams[k], 1))
        check_peer_fault()
        return h[0]

    def assign(self, rhs):
        """self = scalar expression of DeviceScalars / constants (asynchronous, n = 1 on every slot)."""
        rhs = wrap(rhs)
        for k in self.ctx.local:
            low = _Lowering(k, 0)
            low.size = 1
            low.lower(rhs)
            L.check(L.lib().vexb_eval(self.ctx.devs[k], self.ctx.streams[k], self.bufs[k], self.dtype, L.SET, C.byref(low.e), 1, 0))
        return self


_lower_base = _Lowering.lower


def _lower_with_dscalar(self, n):
    if isinstance(n, DeviceScalar):
        self.emit("TERM", n.dtype, self.term(L.TERM_DSCALAR, n.dtype, ptr=n.bufs[self.part].value))
    else:
        _lower_base(self, n)


_Lowering.lower = _lower_with_dscalar


def _reduce_device(self, expr, out: DeviceScalar):
    """Reduce `expr` and leave the (all-reduced) result in `out` on every device; asynchronous."""
    lib = L.lib()
    ctx = self.ctx
    expr = wrap(expr)
    props = _find_props(expr)
    if props is None:
        raise ValueError("expression has no vector terminal")
    if self.kind == L.MINMAX:
        raise ValueError("MIN_MAX needs two result slots; use the host-returning call")
    expr = _reduce_in_one_pass(ctx, expr, props[1])
    part = ctx.partition(props[1])
    for k in ctx.local:
        ws, _ = ctx.workspace(k)
        low = _Lowering(k, int(part[k]))
        low.lower(expr)
        # with a peer group the combine across GPUs happens inside the reduction kernel (no NCCL call)
        peer = ctx.peers[k] if (ctx.peers is not None and ctx.use_peer_reduce) else None
        code = lib.vexb_reduce_all(ctx.devs[k], ctx.streams[k], C.byref(low.e), self.dtype, int(part[k + 1] - part[k]),
                                   int(part[k]), self.kind, out.bufs[k], ws, peer)
        if code == L.ERR_UNSUPPORTED and k == ctx.local[0] and _has_call(expr):
            return _reduce_device(self, _temporary(ctx, expr, props[1]), out)   # no NVRTC: reduce a temporary
        _reduce_all_in_step(ctx, k, peer, self.dtype, self.kind, out.bufs[k], code, out.bufs)
    if ctx.nparts > 1 and not (ctx.peers is not None and ctx.use_peer_reduce):
        if ctx.comms is None:
            raise RuntimeError("device-resident reductions over several slots need a communicator (NCCL)")
        L.check(lib.vexb_comm_allreduce(len(ctx.local), ctx._arr(ctx.comms), ctx._arr(out.bufs), ctx._arr(ctx.streams),
                                        1, self.dtype, self.kind))
    return out


Reductor.device = _reduce_device


class Graph:
    """Capture the asynchronous work issued by `fn()` on every local slot into CUDA graphs; replay with launch()."""

    def __init__(self, ctx: Context, fn):
        lib = L.lib()
        self.ctx = ctx
        for k in ctx.local:
            L.check(lib.vexb_graph_begin(ctx.devs[k], ctx.streams[k]))
        try:
            fn()
        finally:
            self.h = {}
            for k in ctx.local:
                g = C.c_void_p()
                L.check(lib.vexb_graph_end(ctx.devs[k], ctx.streams[k], C.byref(g)))
                self.h[k] = g

    def launch(self):
        for k in self.ctx.local:
            L.check(L.lib().vexb_graph_launch(self.h[k], self.ctx.streams[k]))

    def __del__(self):
        try:
            for g in self.h.values():
                L.lib().vexb_graph_destroy(g)
        except Exception:
            pass


def assign_multi(lhs, rhs, op: int = L.SET) -> bool:
    """vex::tie(lhs...) OP= std::tie(rhs...) (assign_multiexpression, vexcl/operations.hpp:2081-2185): every right-hand side is
    evaluated before any left-hand side is written.  One generated kernel per device slice when the back end has it
    (vexb_eval_multi; compiled in the background at the first use of the tuple of expressions), else component by
    component through temporaries.  Returns True when the fused kernel ran."""
    lhs, rhs = list(lhs), [wrap(r) for r in rhs]
    if len(lhs) != len(rhs) or not lhs:
        raise ValueError("assign_multi: one expression per target")
    ctx, n, dt = lhs[0].ctx, lhs[0].n, lhs[0].dtype
    if any(v.ctx is not ctx or v.n != n or v.dtype != dt for v in lhs):
        raise ValueError("assign_multi: targets must share context, size and type")
    lib = L.lib()
    N = len(lhs)
    fused = 2 <= N <= 8
    for k in ctx.local:
        if not fused:
            break
        lows = []
        for r in rhs:
            low = _Lowering(k, lhs[0].part_start(k))
            low.size = n
            for v in lhs:
                low.see(v)
            low.lower(r)
            lows.append(low)
        es = (C.POINTER(L.Expr) * N)(*[C.pointer(low.e) for low in lows])
        out = (C.c_void_p * N)(*[v.bufs[k] for v in lhs])
        handled = C.c_int(0)
        code = lib.vexb_eval_multi(ctx.devs[k], ctx.streams[k], N, out, dt, op, es, lhs[0].part_size(k), lhs[0].part_start(k), C.byref(handled))
        if code == L.ERR_UNSUPPORTED:
            # raw pointers into the targets read device copies instead (never component by component: that would race too)
            # (the component-by-component path below evaluates into temporaries first, so it reads the old targets as is)
            copies = [cp for low in lows for cp in _redirect_pointers(low.e, lhs)]
            if copies:
                code = lib.vexb_eval_multi(ctx.devs[k], ctx.streams[k], N, out, dt, op, es, lhs[0].part_size(k), lhs[0].part_start(k), C.byref(handled))
        L.check(code)
        if not handled.value:
            fused = False                       # the kernel is not there yet (first slice says so): nothing has been written
    if fused:
        return True
    tmp = [vector(ctx, n, dtype=lhs[0].np_dtype) for _ in range(N)]
    for t, r in zip(tmp, rhs):
        t.assign(r)
    for v, t in zip(lhs, tmp):
        v._assign(op, t)
    return False


# ------------------------------------------------------------------------------------------- sort
def _sort(keys: vector, vals: Optional[vector], descending: bool):
    """vexb_sort on every slice (on its own stream, workspace allocated per call and part), then, with several parts,
    the stable host merge of the sorted slices (vexb_sort_merge), written back: vex::sort's sort_sink (sort.hpp:2070-2116)."""
    ctx = keys.ctx
    if vals is not None and (vals.ctx is not ctx or vals.n != keys.n or not np.array_equal(vals.part, keys.part)):
        raise ValueError("Keys and values span different devices")
    if ctx.is_distributed:
        raise ValueError("sort needs every part of the vector in this process")
    lib = L.lib()
    vdt = -1 if vals is None else vals.dtype
    for k in ctx.local:
        n = keys.part_size(k)
        if n == 0:
            continue
        nb = C.c_size_t()
        L.check(lib.vexb_sort_workspace_bytes(n, keys.dtype, vdt, C.byref(nb)))
        ws = C.c_void_p()
        if nb.value:
            L.check(lib.vexb_malloc(ctx.devs[k], nb.value, C.byref(ws)))
        try:
            L.check(lib.vexb_sort(ctx.devs[k], ctx.streams[k], keys.bufs[k], keys.dtype, None if vals is None else vals.bufs[k],
                                  vdt, n, int(bool(descending)), ws, nb.value))
        finally:
            if ws.value:
                lib.vexb_free(ctx.devs[k], ws)
    if ctx.nparts == 1:
        return
    hk = keys.read()
    ok = np.empty_like(hk)
    hv = ov = None
    if vals is not None:
        hv = vals.read()
        ov = np.empty_like(hv)
    part = (C.c_size_t * (ctx.nparts + 1))(*[int(p) for p in keys.part])
    L.check(lib.vexb_sort_merge(ctx.nparts, part, hk.ctypes.data, keys.dtype, None if hv is None else hv.ctypes.data, vdt,
                                int(bool(descending)), ok.ctypes.data, None if ov is None else ov.ctypes.data))
    keys.write(ok)
    if vals is not None:
        vals.write(ov)


def sort(keys: vector, descending: bool = False):
    """vex::sort(keys[, vex::less / vex::greater]): a stable sort in place, ascending or descending.  Floating keys: -0.0
    equals +0.0, NaNs equal each other and follow +inf (numpy's and torch's order)."""
    _sort(keys, None, descending)


def sort_by_key(keys: vector, vals: vector, descending: bool = False):
    """vex::sort_by_key(keys, vals[, comparator]): sort keys stably in place and move vals with them."""
    _sort(keys, vals, descending)


# ------------------------------------------------------------------------------------------- scans
def _scan_identity(np_dtype):
    """The exact identity of the element type's add: -0.0 for floats (-0.0 + x == x, also for x = +0.0), 0 otherwise."""
    return np_dtype.type(-0.0) if np_dtype.kind == "f" else np_dtype.type(0)


def _as_element(value, np_dtype) -> np.ndarray:
    """`value` as one element of np_dtype; integers wrap, as the C++ conversion does."""
    a = np.asarray(value)
    if np_dtype.kind in "iu" and a.dtype.kind in "iu":
        return np.array([int(a) % (1 << (8 * np_dtype.itemsize))], dtype=np.uint64).astype(np_dtype)
    return np.array([a], dtype=np_dtype)


def _scan_workspace(ctx, k, n, dtype):
    lib = L.lib()
    nb = C.c_size_t()
    L.check(lib.vexb_scan_workspace_bytes(n, dtype, C.byref(nb)))
    ws = C.c_void_p()
    if nb.value:
        L.check(lib.vexb_malloc(ctx.devs[k], nb.value, C.byref(ws)))
    return ws, nb.value


def _element(vec: vector, k: int, i: int):
    """Element i of slice k (a blocking one-element read)."""
    out = np.empty(1, dtype=vec.np_dtype)
    es = vec.np_dtype.itemsize
    L.check(L.lib().vexb_d2h(vec.ctx.devs[k], out.ctypes.data, C.c_void_p(vec.bufs[k].value + i * es), es, vec.ctx.streams[k], 1))
    return out[0]


def _add_to_slice(vec: vector, k: int, value):
    """Slice k of vec += value, one launch of the expression path."""
    low = _Lowering(k, vec.part_start(k))
    low.size = vec.n
    low.target = vec
    low.sweep = None
    low.see(vec)
    low.lower(Scalar(value, vec.dtype))
    L.check(L.lib().vexb_eval(vec.ctx.devs[k], vec.ctx.streams[k], vec.bufs[k], vec.dtype, L.ADD, C.byref(low.e),
                              vec.part_size(k), vec.part_start(k)))


def _scan(inp: vector, out: vector, init, exclusive: bool):
    """vexb_scan on every slice; with several parts, the local totals are folded on the host in the element type and
    each carry is added to its slice (scan.hpp:426-518), with init counted once: only the first non-empty slice starts
    at init, the others at the identity."""
    ctx = inp.ctx
    if out.ctx is not ctx or out.dtype != inp.dtype or out.n != inp.n or not np.array_equal(out.part, inp.part):
        raise ValueError("Incompatible partitioning")
    if ctx.is_distributed:
        raise ValueError("scan needs every part of the vector in this process")
    lib = L.lib()
    dt = inp.np_dtype
    first = _as_element(init, dt)
    ident = np.array([_scan_identity(dt)], dtype=dt)
    several = ctx.nparts > 1
    # an exclusive scan in place overwrites each slice's last input, which its carry needs: read those first
    last_in = {k: _element(inp, k, inp.part_size(k) - 1) for k in ctx.local if several and exclusive and inp.part_size(k)}
    started = False
    for k in ctx.local:
        n = inp.part_size(k)
        if n == 0:
            continue
        ws, nb = _scan_workspace(ctx, k, n, inp.dtype)
        try:
            L.check(lib.vexb_scan(ctx.devs[k], ctx.streams[k], inp.bufs[k], out.bufs[k], inp.dtype, n, int(bool(exclusive)),
                                  (ident if started else first).ctypes.data, ws, nb))
        finally:
            if ws.value:
                lib.vexb_free(ctx.devs[k], ws)
        started = True
    if not several:
        return
    carry = None
    with np.errstate(over="ignore"):
        for k in ctx.local:
            n = out.part_size(k)
            if n == 0:
                continue
            total = _element(out, k, n - 1)
            if exclusive:
                total = dt.type(total + last_in[k])
            if carry is None:
                carry = total
            else:
                _add_to_slice(out, k, carry)
                carry = dt.type(carry + total)


def inclusive_scan(inp: vector, out: vector, init=0):
    """vex::inclusive_scan(in, out[, init]): out[i] = in[0] + ... + in[i].  `init` is not read, as in the reference,
    whose kernels ignore it for inclusive scans.  out may be inp.  Integer sums wrap; every float add is rounded."""
    _scan(inp, out, init, False)


def exclusive_scan(inp: vector, out: vector, init=0):
    """vex::exclusive_scan(in, out[, init]): out[0] = init (its own bits), out[i] = init + in[0] + ... + in[i-1].  out
    may be inp.  On several parts init is counted once (the reference adds it once per part)."""
    _scan(inp, out, init, True)


def _by_key_checks(keys: vector, ivals: vector, what: str):
    if keys.ctx.nparts != 1 or ivals.ctx.nparts != 1:
        raise ValueError(f"{what} is only supported for single device contexts")
    if keys.ctx.is_distributed:
        raise ValueError(f"{what} is only supported for single device contexts")
    if keys.n != ivals.n:
        raise ValueError("keys and values should have same size")


def _scan_by_key(keys: vector, ivals: vector, ovals: vector, init, exclusive: bool):
    _by_key_checks(keys, ivals, "scan_by_key")
    if ovals.ctx.nparts != 1 or ovals.n != ivals.n or ovals.dtype != ivals.dtype:
        raise ValueError("input and output should have same size")
    ctx = keys.ctx
    k = ctx.local[0]
    n = keys.n
    if n == 0:
        return
    if ovals.bufs[k].value == keys.bufs[k].value:
        raise ValueError("keys and ovals are the same buffer")
    lib = L.lib()
    first = _as_element(init, ivals.np_dtype)
    ws, nb = _scan_workspace(ctx, k, n, ivals.dtype)
    try:
        L.check(lib.vexb_scan_by_key(ctx.devs[k], ctx.streams[k], keys.bufs[k], keys.dtype, ivals.bufs[k], ovals.bufs[k],
                                     ivals.dtype, n, int(bool(exclusive)), first.ctypes.data, ws, nb))
    finally:
        if ws.value:
            lib.vexb_free(ctx.devs[k], ws)


def inclusive_scan_by_key(keys: vector, ivals: vector, ovals: vector, init=0):
    """vex::inclusive_scan_by_key(keys, ivals, ovals[, init]): the inclusive sum within every run of keys equal under
    == (-0.0 and +0.0 share a run, every NaN key is a run of its own).  `init` is not read, as in the reference.
    ovals may be ivals.  One-part vectors only."""
    _scan_by_key(keys, ivals, ovals, init, False)


def exclusive_scan_by_key(keys: vector, ivals: vector, ovals: vector, init=0):
    """vex::exclusive_scan_by_key(keys, ivals, ovals[, init]): the exclusive sum within every run of keys, each run
    starting at init.  ovals may be ivals.  One-part vectors only."""
    _scan_by_key(keys, ivals, ovals, init, True)


def reduce_by_key(ikeys: vector, ivals: vector):
    """vex::reduce_by_key(ikeys, ivals, okeys, ovals): (okeys, ovals) as new vectors with one element per run of keys
    equal under ==: okeys[j] holds the bits of the last key of run j and ovals[j] the sum of its values.  One-part
    vectors only."""
    _by_key_checks(ikeys, ivals, "reduce_by_key")
    ctx = ikeys.ctx
    k = ctx.local[0]
    n = ikeys.n
    lib = L.lib()
    ws, nb = _scan_workspace(ctx, k, n, ivals.dtype)
    try:
        runs = C.c_size_t()
        L.check(lib.vexb_reduce_by_key_count(ctx.devs[k], ctx.streams[k], ikeys.bufs[k], ikeys.dtype, ivals.bufs[k],
                                             ivals.dtype, n, ws, nb, C.byref(runs)))
        okeys, ovals = vector(ctx, runs.value, ikeys.np_dtype), vector(ctx, runs.value, ivals.np_dtype)
        L.check(lib.vexb_reduce_by_key_write(ctx.devs[k], ctx.streams[k], ikeys.bufs[k], ikeys.dtype, ivals.bufs[k],
                                             ivals.dtype, n, okeys.bufs[k], ovals.bufs[k], ws, nb))
    finally:
        if ws.value:
            lib.vexb_free(ctx.devs[k], ws)
    return okeys, ovals
