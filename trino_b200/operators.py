"""Host-side mirror of the reference's Operator / OperatorFactory interface over the C ABI.

The reference's host language is Java and there is no JDK in this environment, so the drop-in boundary is
the C ABI (include/trino_gpu.h); these classes are the Python equivalent of the thin Java operators in
java/ (see INTEGRATION.md) and keep the reference's names, argument meaning and error behaviour:

  Operator            M/operator/Operator.java:21-102  (needsInput/addInput/getOutput/finish/isFinished/close)
  OperatorFactory     M/operator/OperatorFactory.java:16-30 (createOperator/noMoreOperators/duplicate)
  HashAggregationOperatorFactory   M/operator/HashAggregationOperator.java:63-200
  AggregationOperatorFactory       M/operator/AggregationOperator.java:35-176 (no GROUP BY keys: one output row)
  HashBuilderOperatorFactory       M/operator/join/unspilled/HashBuilderOperator.java:55-140
  LookupJoinOperatorFactory        M/operator/join/unspilled/LookupJoinOperatorFactory.java
  FilterAndProjectOperatorFactory  M/operator/FilterAndProjectOperator.java:97-150
  PartitionedOutputOperatorFactory M/operator/output/PartitionedOutputOperator.java:52-140

Every method ends in a libtrino_gpu.so call; nothing here computes on the CPU.
"""
import ctypes as C

import numpy as np

from . import abi
from .page import AbiPage, Block, Page, RowBlock, compose_row_blocks, compose_state_blocks, flatten_row_blocks, flatten_state_blocks

_NP_OF_TYPE = {abi.INT64: np.int64, abi.INT32: np.int32, abi.INT16: np.int16, abi.INT8: np.int8, abi.FLOAT64: np.float64, abi.FLOAT32: np.float32}
_ELEM = {abi.INT64: 8, abi.INT32: 4, abi.INT16: 2, abi.INT8: 1, abi.FLOAT64: 8, abi.FLOAT32: 4}


def _i32(values):
    arr = (C.c_int32 * max(1, len(values)))(*values)
    return arr


class Context:
    """tgpu_ctx: one per (process, device, driver thread)."""

    def __init__(self, device=0):
        self.lib = abi.load_library()
        h = C.c_void_p()
        st = self.lib.tgpu_ctx_create(device, C.byref(h))
        if st != 0:
            raise abi.TrinoGpuError(st, self.lib.tgpu_status_name(st).decode(), self.lib.tgpu_last_error(None).decode())
        self.h = h
        self.device = device

    def check(self, st):
        if st != 0:
            raise abi.TrinoGpuError(st, self.lib.tgpu_status_name(st).decode(), self.lib.tgpu_last_error(self.h).decode())

    def close(self):
        if self.h:
            self.lib.tgpu_ctx_destroy(self.h)
            self.h = None

    def synchronize(self):
        self.check(self.lib.tgpu_ctx_synchronize(self.h))

    @property
    def kernel_launches(self):
        return self.lib.tgpu_ctx_kernel_launches(self.h)

    # ---- device memory
    def malloc(self, nbytes):
        p = C.c_void_p()
        self.check(self.lib.tgpu_malloc(self.h, nbytes, C.byref(p)))
        return p.value

    def free(self, ptr):
        self.check(self.lib.tgpu_free(self.h, C.c_void_p(ptr)))

    def to_device(self, arr):
        arr = np.ascontiguousarray(arr)
        p = self.malloc(max(arr.nbytes, 16))
        if arr.nbytes:
            self.check(self.lib.tgpu_memcpy_h2d(self.h, C.c_void_p(p), C.c_void_p(arr.ctypes.data), arr.nbytes))
        return p

    def to_host(self, ptr, dtype, count):
        out = np.empty(count, dtype=dtype)
        if out.nbytes:
            self.check(self.lib.tgpu_memcpy_d2h(self.h, C.c_void_p(out.ctypes.data), C.c_void_p(ptr), out.nbytes))
        return out

    def pinned_empty(self, count, dtype):
        p = C.c_void_p()
        nbytes = int(count) * np.dtype(dtype).itemsize
        st = self.lib.tgpu_host_alloc_pinned(max(nbytes, 16), C.byref(p))
        self.check(st)
        buf = (C.c_char * max(nbytes, 16)).from_address(p.value)
        arr = np.frombuffer(buf, dtype=dtype, count=count)
        self._pinned = getattr(self, "_pinned", [])
        self._pinned.append(p)   # freed with the process; pinned buffers live as long as the bench
        return arr

    def flush_l2(self):
        self.check(self.lib.tgpu_flush_l2(self.h))

    def timer_start(self):
        self.check(self.lib.tgpu_timer_start(self.h))

    def timer_stop_ms(self):
        ms = C.c_float()
        self.check(self.lib.tgpu_timer_stop_ms(self.h, C.byref(ms)))
        return ms.value

    def last_kernel_ms(self):
        ms = C.c_float()
        self.check(self.lib.tgpu_ctx_last_kernel_ms(self.h, C.byref(ms)))
        return ms.value

    # ---- output pages
    def page_to_host(self, pp, release=True, views_of=None):
        """device tgpu_page* -> host Page (numpy).  `views_of`: the host input Page of a by-reference probe; output columns
        without device data are views of its blocks (tgpu_page_passthrough_channel)."""
        dp = pp.contents
        n = dp.num_rows
        host_cols = (abi.Column * max(1, dp.num_columns))()
        keep = []
        for c in range(dp.num_columns):
            d = dp.columns[c]
            h = host_cols[c]
            h.type = d.type
            h.length = n
            if views_of is not None and n > 0 and not d.data:
                src = C.c_int32(-1)
                self.check(self.lib.tgpu_page_passthrough_channel(pp, c, C.byref(src)))
                if src.value < 0:
                    raise RuntimeError(f"output column {c} has no device data and is not a pass-through view")
                h.data = None
                keep.append(("view", views_of.get_block(src.value), None, None))
                continue
            valid = np.empty((n + 7) // 8 + 1, dtype=np.uint8)
            h.validity = valid.ctypes.data
            if d.type == abi.UTF8:
                nbytes = max(1, self.lib.tgpu_page_utf8_bytes(self.h, pp, c))
                # offsets may be absolute into a larger buffer: size the host buffer by the last offset
                offs = np.empty(n + 1, dtype=np.int32)
                if n:
                    self.check(self.lib.tgpu_memcpy_d2h(self.h, C.c_void_p(offs.ctypes.data), C.c_void_p(d.offsets), (n + 1) * 4))
                    nbytes = max(nbytes, int(offs[n]))
                data = np.zeros(nbytes, dtype=np.uint8)
                h.offsets = offs.ctypes.data
                h.data = data.ctypes.data
                keep.append((d.type, data, valid, offs))
            elif d.type == abi.INT128:
                data = np.empty((n, 2), dtype=np.int64)
                h.data = data.ctypes.data
                keep.append((d.type, data, valid, None))
            else:
                data = np.empty(n, dtype=_NP_OF_TYPE[d.type])
                h.data = data.ctypes.data
                keep.append((d.type, data, valid, None))
        hp = abi.Page(dp.num_columns, 0, n, C.cast(host_cols, C.POINTER(abi.Column)))
        self.check(self.lib.tgpu_page_copy_to_host(self.h, pp, C.byref(hp)))
        blocks = []
        for type_, data, valid, offs in keep:
            if type_ == "view":
                blocks.append(data)
                continue
            bits = np.unpackbits(valid, bitorder="little")[:n].astype(np.bool_)
            nulls = ~bits
            blocks.append(Block(type_, data, nulls if nulls.any() else None, offs))
        if release:
            self.lib.tgpu_page_release(self.h, pp)
        return Page(*blocks, position_count=n)


class DeviceColumn:
    """A column that already lives in HBM (bench / GPU->GPU chaining)."""

    def __init__(self, type_, ptr, length, validity=None, offsets=None):
        self.type, self.ptr, self.length, self.validity, self.offsets = type_, ptr, length, validity, offsets


class DevicePage:
    def __init__(self, columns, rows):
        self.columns = columns
        self.rows = rows
        self.abi_cols = (abi.Column * max(1, len(columns)))()
        for i, c in enumerate(columns):
            a = self.abi_cols[i]
            a.type, a.flags, a.length = c.type, 0, c.length
            a.data, a.offsets, a.validity = c.ptr, c.offsets, c.validity
        self.page = abi.Page(len(columns), abi.PAGE_DEVICE, rows, C.cast(self.abi_cols, C.POINTER(abi.Column)))

    def ref(self):
        return C.byref(self.page)


class DeviceOutputPage:
    """A library-owned output page left on the device."""

    def __init__(self, ctx, pp):
        self.ctx, self.pp = ctx, pp
        self.rows = pp.contents.num_rows
        self.num_columns = pp.contents.num_columns

    def column(self, c):
        d = self.pp.contents.columns[c]
        return DeviceColumn(d.type, d.data, d.length, d.validity, d.offsets)

    def as_device_page(self):
        return DevicePage([self.column(c) for c in range(self.num_columns)], self.rows)

    def to_host(self):
        return self.ctx.page_to_host(self.pp, release=False)

    def release(self):
        if self.pp:
            self.ctx.lib.tgpu_page_release(self.ctx.h, self.pp)
            self.pp = None


def _as_abi_page(page):
    if isinstance(page, (DevicePage, AbiPage)):
        return page
    if isinstance(page, DeviceOutputPage):
        return page.as_device_page()
    return AbiPage(page)


# =====================================================================================================
# Operator / OperatorFactory
# =====================================================================================================
class Operator:
    """M/operator/Operator.java:21-102"""

    def __init__(self, ctx, handle):
        self.ctx = ctx
        self.h = handle

    def needs_input(self):
        v = C.c_int()
        self.ctx.check(self.ctx.lib.tgpu_op_needs_input(self.h, C.byref(v)))
        return bool(v.value)

    def add_input(self, page):
        ap = _as_abi_page(page)
        self._last_input = page
        self.ctx.check(self.ctx.lib.tgpu_op_add_input(self.h, ap.ref()))

    def set_passthrough_by_reference(self, enable=True):
        """LookupJoinOperator only: host probe pages upload their join key alone; 1:1 outputs return the input blocks as views"""
        self.ctx.check(self.ctx.lib.tgpu_join_probe_set_passthrough_by_reference(self.h, int(enable)))
        self._by_reference = bool(enable)

    def get_output_device(self):
        pp = abi.PP()
        self.ctx.check(self.ctx.lib.tgpu_op_get_output(self.h, C.byref(pp)))
        return DeviceOutputPage(self.ctx, pp) if pp else None

    def get_output(self):
        pp = abi.PP()
        self.ctx.check(self.ctx.lib.tgpu_op_get_output(self.h, C.byref(pp)))
        views = getattr(self, "_last_input", None) if getattr(self, "_by_reference", False) else None
        if views is not None and not hasattr(views, "get_block"):
            views = None      # device-resident input pages are never by-reference
        return self.ctx.page_to_host(pp, views_of=views) if pp else None

    def finish(self):
        self.ctx.check(self.ctx.lib.tgpu_op_finish(self.h))

    def is_finished(self):
        v = C.c_int()
        self.ctx.check(self.ctx.lib.tgpu_op_is_finished(self.h, C.byref(v)))
        return bool(v.value)

    def memory_bytes(self):
        return self.ctx.lib.tgpu_op_memory_bytes(self.h)

    def close(self):
        if self.h:
            self.ctx.lib.tgpu_op_close(self.h)
            self.h = None


class OperatorFactory:
    """M/operator/OperatorFactory.java:16-30"""

    def __init__(self):
        self.closed = False

    def create_operator(self):
        if self.closed:
            raise RuntimeError("Factory is already closed")   # checkState(!closed) in every reference factory
        return self._create()

    def no_more_operators(self):
        self.closed = True

    def duplicate(self):
        raise NotImplementedError


# ---- expressions ----------------------------------------------------------------------------------
class Col:
    """dtype: (precision, scale) of a V_DECIMAL channel (a short decimal is an INT64 channel, a long one INT128)"""

    def __init__(self, channel, vtype, dtype=None):
        self.channel, self.vtype, self.dtype = channel, vtype, dtype


class Const:
    """value: int / float / bool, or str / bytes for V_VARCHAR (a str is taken as its UTF-8 bytes), or the unscaled int of a V_DECIMAL
    of type dtype = (precision, scale)"""

    def __init__(self, value, vtype, dtype=None):
        self.value, self.vtype, self.dtype = value, vtype, dtype


def _utf8(v):
    return v.encode() if isinstance(v, str) else bytes(v)


class Null:
    def __init__(self, vtype, dtype=None):
        self.vtype, self.dtype = vtype, dtype


def decimal_result_type(op, a, b=None, legacy=False):
    """the result DECIMAL(p, s) of a decimal operator under the reference's type rules (M/type/DecimalOperators.java: the default rules,
    or deprecated.legacy-arithmetic-decimal-operators with legacy=True)"""
    (ap, as_), (bp, bs) = a, (b if b is not None else (0, 0))
    if op in (abi.EX_MOV, abi.EX_NEG):
        return a
    if op in (abi.EX_ADD, abi.EX_SUB):
        if legacy:
            return min(38, max(ap - as_, bp - bs) + max(as_, bs) + 1), max(as_, bs)
        integral, raw = max(ap - as_, bp - bs), max(as_, bs)
        p = min(raw + integral + 1, 38)
        return p, min(raw, p - integral)
    if op == abi.EX_MUL:
        if legacy:
            return min(38, ap + bp), as_ + bs
        rp, rs = ap + bp + 1, as_ + bs
        integral = rp - rs
        return min(rp, 38), min(rs, 6 if integral > 32 else 38 - integral)
    if op == abi.EX_DIV:
        if legacy:
            return min(38, ap + bs + max(bs - as_, 0)), max(as_, bs)
        rs = max(6, as_ + bp + 1)
        rp = ap - as_ + bs + rs
        integral = rp - rs
        return min(rp, 38), min(rs, 6 if integral > 32 else 38 - integral)
    raise ValueError("no DECIMAL result type for op %d" % op)


class Call:
    """op: one of abi.EX_*; args: expressions.  vtype is the OPERAND type (result of comparisons is BOOLEAN).
    EX_IN takes in_list (str / bytes values for a VARCHAR operand, unscaled ints for a DECIMAL one); EX_LIKE takes the constant pattern
    and an optional one-character escape (str / bytes): `value LIKE pattern [ESCAPE escape]`.
    String functions: EX_LENGTH(s) gives BIGINT; EX_SUBSTR(s, start[, length]) with BIGINT start and length, EX_LTRIM / EX_RTRIM /
    EX_TRIM(s) and EX_CONCAT(a, b) give VARCHAR (see concat() for more than two pieces).
    DECIMAL: the result type of +, -, *, / follows the reference's default rules (legacy=True: the legacy ones) unless result_dtype gives
    it; EX_CAST_TO_DECIMAL needs result_dtype."""

    def __init__(self, op, *args, in_list=None, pattern=None, escape=None, result_dtype=None, legacy=False):
        self.op, self.args, self.in_list = op, list(args), in_list
        self.pattern, self.escape = pattern, escape
        a0 = args[0]
        self.operand_vtype = a0.vtype if not isinstance(a0, Call) else a0.result_vtype
        self.operand_dtypes = [getattr(x, "dtype", None) for x in args]
        self.dtype = None
        boolean_result = op in (abi.EX_EQ, abi.EX_NE, abi.EX_LT, abi.EX_LE, abi.EX_GT, abi.EX_GE, abi.EX_AND, abi.EX_OR, abi.EX_NOT,
                                abi.EX_IS_NULL, abi.EX_IS_NOT_NULL, abi.EX_BETWEEN, abi.EX_IN, abi.EX_LIKE)
        if boolean_result:
            self.result_vtype = abi.V_BOOLEAN
        elif op in (abi.EX_CAST_BIGINT_TO_DOUBLE, abi.EX_CAST_DECIMAL_TO_DOUBLE):
            self.result_vtype = abi.V_DOUBLE
        elif op in (abi.EX_CAST_DOUBLE_TO_BIGINT, abi.EX_CAST_DECIMAL_TO_BIGINT, abi.EX_LENGTH):
            self.result_vtype = abi.V_BIGINT
        elif op == abi.EX_CAST_TO_DECIMAL:
            if result_dtype is None:
                raise ValueError("a cast to DECIMAL needs result_dtype")
            self.result_vtype, self.dtype = abi.V_DECIMAL, tuple(result_dtype)
        else:
            self.result_vtype = self.operand_vtype
            if self.operand_vtype == abi.V_DECIMAL:
                self.dtype = tuple(result_dtype) if result_dtype is not None else decimal_result_type(
                    op, self.operand_dtypes[0], self.operand_dtypes[1] if len(args) > 1 else None, legacy)

    @property
    def vtype(self):
        return self.result_vtype


def concat(*args):
    """concat(x1, ..., xn) and x1 || ... || xn as the left-deep chain of binary EX_CONCATs the library evaluates (the same value and the
    same error as the variadic call)"""
    if len(args) < 2:
        raise ValueError("There must be two or more concatenation arguments")
    e = Call(abi.EX_CONCAT, args[0], args[1])
    for a in args[2:]:
        e = Call(abi.EX_CONCAT, e, a)
    return e


# ---- conditional special forms (SqlToRowExpressionTranslator.java:280-400) --------------------------------------------------------
# The branches of one form have one type: the planner has already coerced them to the result type.  IF and the binary COALESCE are
# instructions (abi.EX_IF, abi.EX_COALESCE); CASE, the simple CASE, NULLIF and a longer COALESCE keep the tree as written (the reference
# evaluator reads it) and carry in `lowered` the tree of IF / COALESCE / EQ nodes PageProcessorProgram compiles.  A node that appears
# twice in `lowered` (the simple CASE's value, NULLIF's first argument) is evaluated once.  VARCHAR results are not evaluated on the GPU.
def _branch_type(*exprs):
    """(vtype, dtype) of a form's result: its first branch that is not a bare NULL, else its first"""
    for e in exprs:
        if not isinstance(e, Null):
            return e.vtype, getattr(e, "dtype", None)
    return exprs[0].vtype, getattr(exprs[0], "dtype", None)


class If:
    """IF(cond, then[, else_]): then when cond is TRUE, otherwise else_ (NULL when missing); cond is BOOLEAN"""
    lowered = None

    def __init__(self, cond, then, else_=None):
        self.vtype, self.dtype = _branch_type(then, else_) if else_ is not None else _branch_type(then)
        self.cond, self.then = cond, then
        self.else_ = else_ if else_ is not None else Null(self.vtype, self.dtype)


class Case:
    """searched CASE WHEN cond1 THEN r1 ... [ELSE else_] END: whens = [(cond, result), ...]; lowered to the right-deep IF chain"""

    def __init__(self, whens, else_=None):
        if not whens:
            raise ValueError("CASE needs at least one WHEN")
        self.whens, self.else_ = [tuple(w) for w in whens], else_
        self.vtype, self.dtype = _branch_type(*[r for _, r in self.whens], *([else_] if else_ is not None else []))
        e = else_
        for c, r in reversed(self.whens):
            e = If(c, r, e)
        self.lowered = e


class Switch:
    """simple CASE value WHEN w1 THEN r1 ... [ELSE else_] END: whens = [(w, result), ...], each w of value's type.  Lowered to
    IF(value = w1, r1, IF(value = w2, r2, ... else_)) with value the first operand of every EQ: value's error comes first, and a NULL
    value makes every EQ NULL without reading any w's error, as SwitchCodeGenerator does"""

    def __init__(self, value, whens, else_=None):
        if not whens:
            raise ValueError("CASE needs at least one WHEN")
        self.value, self.whens, self.else_ = value, [tuple(w) for w in whens], else_
        self.vtype, self.dtype = _branch_type(*[r for _, r in self.whens], *([else_] if else_ is not None else []))
        e = else_
        for w, r in reversed(self.whens):
            e = If(Call(abi.EX_EQ, value, w), r, e)
        self.lowered = e


class Coalesce:
    """COALESCE(a1, ..., an): the first non-NULL argument.  More than two arguments lower to COALESCE(a1, COALESCE(a2, ...))"""

    def __init__(self, *args):
        if len(args) < 2:
            raise ValueError("COALESCE needs at least two arguments")
        self.args = list(args)
        self.vtype, self.dtype = _branch_type(*args)
        self.lowered = Coalesce(args[0], Coalesce(*args[1:])) if len(args) > 2 else None


def _cast(e, vtype, dtype=None):
    """e as (vtype, dtype): the cast the planner puts around a comparison operand of another type"""
    ev, ed = e.vtype, getattr(e, "dtype", None)
    if ev == vtype and (vtype != abi.V_DECIMAL or tuple(ed) == tuple(dtype)):
        return e
    if ev == abi.V_BIGINT and vtype == abi.V_DOUBLE:
        return Call(abi.EX_CAST_BIGINT_TO_DOUBLE, e)
    if ev == abi.V_DECIMAL and vtype == abi.V_DOUBLE:
        return Call(abi.EX_CAST_DECIMAL_TO_DOUBLE, e)
    if ev in (abi.V_BIGINT, abi.V_DECIMAL) and vtype == abi.V_DECIMAL:
        return Call(abi.EX_CAST_TO_DECIMAL, e, result_dtype=dtype)
    raise ValueError("no cast from vtype %d to vtype %d" % (ev, vtype))


class NullIf:
    """NULLIF(a, b): NULL when a = b, otherwise a.  compare_as: the common type of the comparison when it is not a's, as a vtype or
    (vtype, dtype).  Lowered to IF(cast(a) = cast(b), NULL, a) with a evaluated once: a NULL a stops the EQ before b, so b raises
    nothing, as NullIfCodeGenerator does"""

    def __init__(self, a, b, compare_as=None):
        self.a, self.b = a, b
        self.vtype, self.dtype = a.vtype, getattr(a, "dtype", None)
        if compare_as is None:
            cv, cd = self.vtype, self.dtype
        elif isinstance(compare_as, int):
            cv, cd = compare_as, None
        else:
            cv, cd = compare_as
        self.compare_as = (cv, cd)
        self.lowered = If(Call(abi.EX_EQ, _cast(a, cv, cd), _cast(b, cv, cd)), Null(self.vtype, self.dtype), a)


def _lower(e):
    while getattr(e, "lowered", None) is not None:
        e = e.lowered
    return e


def _children(e):
    """the operands of an instruction node (after _lower)"""
    if isinstance(e, Call):
        return e.args
    if isinstance(e, If):
        return [e.cond, e.then, e.else_]
    if isinstance(e, Coalesce):
        return e.args
    return []


def _count_reads(e, reads):
    """reads[id(node)]: how many instruction operands read each node of the tree below e (once per edge); each node is visited once"""
    for c in _children(e):
        c = _lower(c)
        first = id(c) not in reads
        reads[id(c)] = reads.get(id(c), 0) + 1
        if first:
            _count_reads(c, reads)


class PageProcessorProgram:
    """Compiles expression trees (the RowExpressions of LocalExecutionPlanner.java:2111-2114) to the three-address
    tgpu_expr_program.  `projections`: ints pass a channel through, expressions are computed."""

    def __init__(self, filter_expr, projections):
        self.insns = []
        self.in_lists = []
        self.strings = []          # VARCHAR constants (bytes), indexed by TGPU_OPND_CONST imm and VARCHAR IN-list values
        self.like_patterns = []    # (pattern bytes, escape bytes)
        self.signatures = []       # per instruction: ((p, s) of a, b, c, result) or None
        self.decimal_constants = []   # long DECIMAL constants (python ints), indexed by a long constant's imm and long IN-list values
        self.live = set()
        self.filter_temp = -1
        self.num_filter_insns = 0
        if filter_expr is not None:
            opnd = self._emit(filter_expr)
            if opnd[0] != abi.OPND_TEMP:
                t = self._alloc()
                self._push(abi.EX_MOV, abi.V_BOOLEAN, t, opnd)
                opnd = (abi.OPND_TEMP, t, 0)
            self.filter_temp = opnd[1]
            self.num_filter_insns = len(self.insns)
        self.projections = []
        for p in projections:
            if isinstance(p, int):
                self.projections.append((0, p, 0))
                continue
            vt = p.vtype
            opnd = self._emit(p)
            if opnd[0] != abi.OPND_TEMP or opnd[1] == self.filter_temp:
                t = self._alloc()
                dt = p.dtype if vt == abi.V_DECIMAL else None
                self._push(abi.EX_MOV, vt, t, opnd, sig=(dt, None, None, dt) if dt else None)
                opnd = (abi.OPND_TEMP, t, 0)
            self.projections.append((1, opnd[1], vt))
        self._build()

    def _alloc(self):
        for t in range(8):
            if t not in self.live:
                self.live.add(t)
                return t
        raise ValueError("expression needs more than 8 temporaries")

    def _push(self, op, vtype, dst, a, b=None, c=None, sig=None):
        self.insns.append((op, vtype, dst, a, b or (abi.OPND_NONE, 0, 0), c or (abi.OPND_NONE, 0, 0)))
        self.signatures.append(sig)

    def _decimal(self, value, dtype):
        """a DECIMAL constant: a short one is its unscaled value, a long one an index into decimal_constants"""
        if dtype[0] <= 18:
            return int(value)
        if value not in self.decimal_constants:
            self.decimal_constants.append(int(value))
        return self.decimal_constants.index(value)

    def _string(self, v):
        b = _utf8(v)
        if b not in self.strings:
            self.strings.append(b)
        return self.strings.index(b)

    def _emit(self, e):
        """one tree (the filter or a projection): a node read by several operands within it is emitted once, at its first use, and its
        temp is freed after its last reader"""
        self._reads, self._done = {}, {}
        _count_reads(_lower(e), self._reads)
        return self._emit_node(e)

    def _emit_node(self, e):
        e = _lower(e)
        if id(e) in self._done:
            return self._done[id(e)]
        if isinstance(e, Col):
            return (abi.OPND_COLUMN, e.channel, 0)
        if isinstance(e, Const) and e.vtype == abi.V_VARCHAR:
            return (abi.OPND_CONST, 0, self._string(e.value))
        if isinstance(e, Const) and e.vtype == abi.V_DECIMAL:
            return (abi.OPND_CONST, 0, self._decimal(e.value, e.dtype))
        if isinstance(e, Const):
            imm = abi.Imm()
            if e.vtype == abi.V_DOUBLE:
                imm.f64 = float(e.value)
            else:
                imm.i64 = int(e.value)
            return (abi.OPND_CONST, 0, imm.i64)
        if isinstance(e, Null):
            return (abi.OPND_NULL, 0, 0)
        if isinstance(e, (If, Coalesce)):
            kids = [_lower(k) for k in _children(e)]
            ops = [self._emit_node(k) for k in kids]
            self._release(kids, ops)
            dst = self._alloc()
            sig = None
            if e.vtype == abi.V_DECIMAL:
                dts = [getattr(k, "dtype", None) or e.dtype for k in kids]
                sig = (None, dts[1], dts[2], e.dtype) if isinstance(e, If) else (dts[0], dts[1], None, e.dtype)
            self._push(abi.EX_IF if isinstance(e, If) else abi.EX_COALESCE, e.vtype, dst, *ops, sig=sig)
            self._done[id(e)] = (abi.OPND_TEMP, dst, 0)
            return self._done[id(e)]
        kids = [_lower(a) for a in e.args]
        ops = [self._emit_node(a) for a in kids]
        b = None
        if e.op == abi.EX_LIKE:
            self.like_patterns.append((_utf8(e.pattern), b"" if e.escape is None else _utf8(e.escape)))
            b = (abi.OPND_CONST, 0, len(self.like_patterns) - 1)
        elif e.op == abi.EX_IN and e.operand_vtype == abi.V_DECIMAL:
            self.in_lists.append([self._decimal(v, e.operand_dtypes[0]) for v in e.in_list])
            b = (abi.OPND_CONST, 0, len(self.in_lists) - 1)
        elif e.op == abi.EX_IN and e.operand_vtype == abi.V_VARCHAR:
            self.in_lists.append([self._string(v) for v in e.in_list])
            b = (abi.OPND_CONST, 0, len(self.in_lists) - 1)
        elif e.op == abi.EX_IN:
            vals = []
            for v in e.in_list:
                imm = abi.Imm()
                if e.operand_vtype == abi.V_DOUBLE:
                    imm.f64 = float(v)
                else:
                    imm.i64 = int(v)
                vals.append(imm.i64)
            self.in_lists.append(vals)
            b = (abi.OPND_CONST, 0, len(self.in_lists) - 1)
        self._release(kids, ops)
        dst = self._alloc()
        sig = None
        if e.operand_vtype == abi.V_DECIMAL or e.dtype is not None:
            dts = (e.operand_dtypes + [None, None, None])[:3] if e.operand_vtype == abi.V_DECIMAL else [None, None, None]
            if e.op == abi.EX_IN:
                dts = [dts[0], None, None]
            sig = (dts[0], dts[1], dts[2], e.dtype)
        self._push(e.op, e.operand_vtype, dst, ops[0], b if b else (ops[1] if len(ops) > 1 else None), ops[2] if len(ops) > 2 else None, sig=sig)
        self._done[id(e)] = (abi.OPND_TEMP, dst, 0)
        return self._done[id(e)]

    def _release(self, kids, ops):
        """operand temps die after their last reader (the filter's temp lives on: projections are emitted after it)"""
        for k, o in zip(kids, ops):
            if o[0] == abi.OPND_TEMP and o[1] != self.filter_temp:
                self._reads[id(k)] -= 1
                if self._reads[id(k)] == 0:
                    self.live.discard(o[1])

    def _build(self):
        n = len(self.insns)
        if n > 64:
            raise ValueError("expression needs more than 64 instructions")
        self._insns = (abi.ExprInsn * max(1, n))()
        for i, (op, vt, dst, a, b, c) in enumerate(self.insns):
            ins = self._insns[i]
            ins.op, ins.vtype, ins.dst = op, vt, dst
            for fld, o in (("a", a), ("b", b), ("c", c)):
                f = getattr(ins, fld)
                f.kind, f.index = o[0], o[1]
                f.imm.i64 = o[2]
        self._projs = (abi.Projection * max(1, len(self.projections)))()
        for i, (k, idx, vt) in enumerate(self.projections):
            self._projs[i].kind, self._projs[i].index, self._projs[i].vtype = k, idx, vt
        self._lists = (abi.InList * max(1, len(self.in_lists)))()
        self._list_bufs = []
        for i, vals in enumerate(self.in_lists):
            buf = (C.c_int64 * max(1, len(vals)))(*vals)
            self._list_bufs.append(buf)
            self._lists[i].count = len(vals)
            self._lists[i].values = C.cast(buf, C.POINTER(C.c_int64))
        # the pool's and the patterns' bytes stay alive with the program
        self._str_bufs = [C.create_string_buffer(b, max(1, len(b))) for b in self.strings]
        self._strs = (abi.Bytes * max(1, len(self.strings)))()
        for i, b in enumerate(self.strings):
            self._strs[i].length, self._strs[i].data = len(b), C.cast(self._str_bufs[i], C.c_void_p)
        self._likes = (abi.LikePattern * max(1, len(self.like_patterns)))()
        for i, (pat, esc) in enumerate(self.like_patterns):
            pb, eb = C.create_string_buffer(pat, max(1, len(pat))), C.create_string_buffer(esc, max(1, len(esc)))
            self._str_bufs += [pb, eb]
            self._likes[i].pattern.length, self._likes[i].pattern.data = len(pat), C.cast(pb, C.c_void_p)
            self._likes[i].escape.length, self._likes[i].escape.data = len(esc), C.cast(eb, C.c_void_p)
        self.struct = abi.ExprProgram(n, C.cast(self._insns, C.POINTER(abi.ExprInsn)), self.filter_temp, self.num_filter_insns,
                                      len(self.projections), C.cast(self._projs, C.POINTER(abi.Projection)),
                                      len(self.in_lists), C.cast(self._lists, C.POINTER(abi.InList)),
                                      len(self.strings), C.cast(self._strs, C.POINTER(abi.Bytes)),
                                      len(self.like_patterns), C.cast(self._likes, C.POINTER(abi.LikePattern)))
        if any(sig is not None for sig in self.signatures):
            self._sigs = (abi.DecimalSignature * max(1, n))()
            for i, sig in enumerate(self.signatures):
                for fld, dt in zip(("a", "b", "c", "result"), sig or ()):
                    if dt is not None:
                        getattr(self._sigs[i], fld).precision, getattr(self._sigs[i], fld).scale = dt
            words = []
            for v in self.decimal_constants:
                u = v & ((1 << 128) - 1)
                words += [u >> 64, u & ((1 << 64) - 1)]
            self._dec_consts = (C.c_int64 * max(1, len(words)))(*[w - (1 << 64) if w >= (1 << 63) else w for w in words])
            self.struct.decimal_signatures = C.cast(self._sigs, C.POINTER(abi.DecimalSignature))
            self.struct.num_decimal_constants = len(self.decimal_constants)
            self.struct.decimal_constants = C.cast(self._dec_consts, C.POINTER(C.c_int64))


class FilterAndProjectOperatorFactory(OperatorFactory):
    def __init__(self, ctx, program):
        super().__init__()
        self.ctx, self.program = ctx, program

    def _create(self):
        h = C.c_void_p()
        self.ctx.check(self.ctx.lib.tgpu_filter_project_create(self.ctx.h, C.byref(self.program.struct), C.byref(h)))
        return Operator(self.ctx, h)

    def duplicate(self):
        return FilterAndProjectOperatorFactory(self.ctx, self.program)


# ---- aggregation ------------------------------------------------------------------------------------
class Aggregator:
    """One AggregatorFactory (M/operator/aggregation/AggregatorFactory.java:40-58): function + input/mask channels."""

    def __init__(self, function, input_channel=-1, mask_channel=-1, result_type=0):
        """result_type: tgpu_type of an avg(decimal) result (INT64 short / INT128 long decimal) where the input does not tell (FINAL step)"""
        self.function, self.input_channel, self.mask_channel, self.result_type = function, input_channel, mask_channel, result_type


class _StateOperator(Operator):
    """An aggregation operator whose intermediate states may be ROW-typed / VARBINARY on the Java side"""
    # ROW-typed intermediate states (AccumulatorCompiler.java:687-760): set by the factory when the neighbouring stage is a Java
    # operator that speaks the reference's state types.  in_first: flat channel of each original input channel; out_widths: see
    # page.compose_row_blocks
    _out_widths = None
    _in_decimal = None            # {input channel (the plan's numbering): "decimal_sum" | "decimal_avg"}: VARBINARY decimal states to unpack

    def add_input(self, page):
        if hasattr(page, "blocks") and (self._in_decimal or any(isinstance(b, RowBlock) for b in page.blocks)):
            page = flatten_state_blocks(page, self._in_decimal or {})
        super().add_input(page)

    def get_output(self):
        out = super().get_output()
        if out is not None and self._out_widths is not None:
            out = compose_state_blocks(out, self._out_widths)
        return out


class HashAggregationOperator(_StateOperator):
    def group_count(self):
        v = C.c_int64()
        self.ctx.check(self.ctx.lib.tgpu_agg_group_count(self.h, C.byref(v)))
        return v.value

    def rows_with_partial_aggregation_disabled(self):
        """AggregationMetrics.INPUT_ROWS_WITH_PARTIAL_AGGREGATION_DISABLED_METRIC_NAME"""
        v = C.c_int64()
        self.ctx.check(self.ctx.lib.tgpu_agg_rows_with_partial_aggregation_disabled(self.h, C.byref(v)))
        return v.value


class PartialAggregationController:
    """M/operator/aggregation/partial/PartialAggregationController.java:35-103 - the object lives in the native library (the operators
    report their flushes to it themselves); needs no GPU."""

    def __init__(self, lib, max_partial_memory, unique_rows_ratio_threshold):
        self.lib, self.max_partial_memory, self.threshold = lib, int(max_partial_memory), float(unique_rows_ratio_threshold)
        h = C.c_void_p()
        rc = lib.tgpu_partial_agg_controller_create(self.max_partial_memory, self.threshold, C.byref(h))
        if rc != 0:
            raise abi.TrinoGpuError(rc, "INVALID_ARGUMENT", "tgpu_partial_agg_controller_create failed")
        self.h = h

    def is_partial_aggregation_disabled(self):
        return bool(self.lib.tgpu_partial_agg_controller_is_disabled(self.h))

    def on_flush(self, bytes_processed, rows_processed, unique_rows_produced=None):
        """unique_rows_produced None = OptionalLong.empty()"""
        self.lib.tgpu_partial_agg_controller_on_flush(self.h, int(bytes_processed), int(rows_processed),
                                                      -1 if unique_rows_produced is None else int(unique_rows_produced))

    def duplicate(self):
        return PartialAggregationController(self.lib, self.max_partial_memory, self.threshold)

    def close(self):
        if self.h:
            self.lib.tgpu_partial_agg_controller_destroy(self.h)
            self.h = None


_FLAT_STATE = {abi.AGG_AVG: 2, abi.AGG_SUM_DECIMAL: 2, abi.AGG_AVG_DECIMAL: 3,           # flat state columns per function (default 1)
               abi.AGG_VAR_SAMP: 3, abi.AGG_VAR_POP: 3, abi.AGG_STDDEV_SAMP: 3, abi.AGG_STDDEV_POP: 3}   # ROW(count, m2, mean)
_DECIMAL_STATE = {abi.AGG_SUM_DECIMAL: "decimal_sum", abi.AGG_AVG_DECIMAL: "decimal_avg"}


def _state_widths(aggregators):
    """the reference's state type per aggregate: ROW(BIGINT, DOUBLE) for avg (2 flat columns), ROW(BIGINT, DOUBLE, DOUBLE) for the
    variance family (3), VARBINARY for the decimal states"""
    return [_DECIMAL_STATE.get(a.function, _FLAT_STATE.get(a.function, 1)) for a in aggregators]


def _flat_channels(aggregators, channels):
    """channels numbered as the Java plan numbers them (one channel per ROW state) -> the flattened page's channels the library sees"""
    wide = {a.input_channel: _FLAT_STATE[a.function] for a in aggregators if a.function in _FLAT_STATE}
    top = max(list(channels) + [0])
    first, at = [], 0
    for c in range(top + 1):
        first.append(at)
        at += wide.get(c, 1)
    return [first[c] if c >= 0 else c for c in channels]


def _agg_fns(aggregators, inputs):
    fns = (abi.AggFn * max(1, len(aggregators)))()
    for i, a in enumerate(aggregators):
        fns[i].function, fns[i].input_channel, fns[i].mask_channel = a.function, inputs[i], a.mask_channel
        fns[i].reserved = getattr(a, "result_type", 0)
    return fns


class HashAggregationOperatorFactory(OperatorFactory):
    def __init__(self, ctx, group_by_channels, step, aggregators, expected_groups=10_000, max_partial_memory=0, pre=None,
                 global_aggregation_group_ids=(), group_id_channel=None, input_types=None, partial_aggregation_controller=None,
                 row_typed_states=False):
        """global_aggregation_group_ids / group_id_channel (a group-by CHANNEL, like the reference's groupIdChannel) / input_types (tgpu_type
        per input channel): the default rows of global grouping sets over empty input (HashAggregationOperator.java:537-567)"""
        super().__init__()
        self.ctx, self.group_by_channels, self.step, self.aggregators = ctx, list(group_by_channels), step, list(aggregators)
        self.expected_groups, self.max_partial_memory, self.pre = expected_groups, max_partial_memory, pre
        self.global_ids, self.group_id_channel, self.input_types = list(global_aggregation_group_ids), group_id_channel, input_types
        self.controller = partial_aggregation_controller
        self.row_typed_states = row_typed_states

    def _create(self):
        from_state = self.step in (abi.STEP_FINAL, abi.STEP_INTERMEDIATE)
        to_state = self.step in (abi.STEP_PARTIAL, abi.STEP_INTERMEDIATE)
        keys_list, agg_inputs = list(self.group_by_channels), [a.input_channel for a in self.aggregators]
        if self.row_typed_states and from_state:
            # channels are numbered as the Java plan numbers them (one channel per ROW state); the library sees the flattened page
            flat = _flat_channels(self.aggregators, keys_list + agg_inputs)
            keys_list, agg_inputs = flat[:len(keys_list)], flat[len(keys_list):]
        keys = _i32(keys_list)
        fns = _agg_fns(self.aggregators, agg_inputs)
        gids = _i32(self.global_ids)
        types = _i32(list(self.input_types or []))
        spec = abi.AggSpec(len(self.group_by_channels), C.cast(keys, C.POINTER(C.c_int32)), self.step, len(self.aggregators),
                           C.cast(fns, C.POINTER(abi.AggFn)), self.expected_groups, self.max_partial_memory,
                           C.pointer(self.pre.struct) if self.pre is not None else None,
                           len(self.global_ids), C.cast(gids, C.POINTER(C.c_int32)),
                           self.group_by_channels.index(self.group_id_channel) if self.group_id_channel is not None else -1,
                           len(self.input_types or []), C.cast(types, C.POINTER(C.c_int32)),
                           self.controller.h if self.controller is not None else None)
        h = C.c_void_p()
        self.ctx.check(self.ctx.lib.tgpu_agg_create(self.ctx.h, C.byref(spec), C.byref(h)))
        op = HashAggregationOperator(self.ctx, h)
        if self.row_typed_states and to_state:
            op._out_widths = [1] * len(self.group_by_channels) + _state_widths(self.aggregators)
        if self.row_typed_states and from_state:
            op._in_decimal = {a.input_channel: _DECIMAL_STATE[a.function] for a in self.aggregators if a.function in _DECIMAL_STATE}
        return op

    def duplicate(self):
        return HashAggregationOperatorFactory(self.ctx, self.group_by_channels, self.step, self.aggregators, self.expected_groups,
                                              self.max_partial_memory, self.pre, self.global_ids, self.group_id_channel, self.input_types,
                                              # HashAggregationOperatorFactory.duplicate :238: a fresh controller for the duplicated plan node
                                              self.controller.duplicate() if self.controller is not None else None, self.row_typed_states)


class AggregationOperator(_StateOperator):
    """M/operator/AggregationOperator.java:35-176: needs input until finish(), then exactly one page of one row"""


class AggregationOperatorFactory(OperatorFactory):
    """AggregationOperatorFactory (M/operator/AggregationOperator.java:43-88), the operator of aggregations without GROUP BY keys.
    input_types: tgpu_type of every input channel of the pages the library sees (for a FINAL step over ROW-typed states: of the
    flattened state columns); required, they shape the output row when no page arrives.  pre: a fused PageProcessorProgram (raw steps)."""

    def __init__(self, ctx, step, aggregators, pre=None, input_types=None, row_typed_states=False):
        super().__init__()
        if input_types is None:
            raise ValueError("AggregationOperatorFactory needs input_types")
        self.ctx, self.step, self.aggregators, self.pre = ctx, step, list(aggregators), pre
        self.input_types, self.row_typed_states = list(input_types), row_typed_states

    def _create(self):
        from_state = self.step in (abi.STEP_FINAL, abi.STEP_INTERMEDIATE)
        to_state = self.step in (abi.STEP_PARTIAL, abi.STEP_INTERMEDIATE)
        agg_inputs = [a.input_channel for a in self.aggregators]
        if self.row_typed_states and from_state:
            agg_inputs = _flat_channels(self.aggregators, agg_inputs)
        fns = _agg_fns(self.aggregators, agg_inputs)
        types = _i32(self.input_types)
        spec = abi.AggSpec(0, None, self.step, len(self.aggregators), C.cast(fns, C.POINTER(abi.AggFn)), 1, 0,
                           C.pointer(self.pre.struct) if self.pre is not None else None, 0, None, -1,
                           len(self.input_types), C.cast(types, C.POINTER(C.c_int32)), None)
        h = C.c_void_p()
        self.ctx.check(self.ctx.lib.tgpu_aggregation_create(self.ctx.h, C.byref(spec), C.byref(h)))
        op = AggregationOperator(self.ctx, h)
        if self.row_typed_states and to_state:
            op._out_widths = _state_widths(self.aggregators)
        if self.row_typed_states and from_state:
            op._in_decimal = {a.input_channel: _DECIMAL_STATE[a.function] for a in self.aggregators if a.function in _DECIMAL_STATE}
        return op

    def duplicate(self):
        return AggregationOperatorFactory(self.ctx, self.step, self.aggregators, self.pre, self.input_types, self.row_typed_states)


class GroupByHash:
    """M/operator/GroupByHash.java: getGroupIds / getGroupCount over a persistent device table."""

    def __init__(self, ctx, key_channels, expected_size=10_000):
        self.ctx = ctx
        keys = _i32(list(key_channels))
        h = C.c_void_p()
        ctx.check(ctx.lib.tgpu_groupby_hash_create(ctx.h, len(key_channels), C.cast(keys, C.POINTER(C.c_int32)), expected_size, C.byref(h)))
        self.h = h

    def get_group_ids(self, page):
        ap = _as_abi_page(page)
        out = np.empty(page.position_count, dtype=np.int32)
        self.ctx.check(self.ctx.lib.tgpu_groupby_hash_get_group_ids(self.h, ap.ref(), C.c_void_p(out.ctypes.data)))
        return out

    def get_group_count(self):
        v = C.c_int64()
        self.ctx.check(self.ctx.lib.tgpu_agg_group_count(self.h, C.byref(v)))
        return v.value

    def close(self):
        if self.h:
            self.ctx.lib.tgpu_op_close(self.h)
            self.h = None


# ---- join -------------------------------------------------------------------------------------------
class LookupSource:
    """M/operator/join/LookupSource.java:24-68 (device table handle)."""

    def __init__(self, ctx, handle):
        self.ctx, self.h = ctx, handle

    def get_join_position_count(self):
        return self.ctx.lib.tgpu_lookup_position_count(self.h)

    def get_in_memory_size_in_bytes(self):
        return self.ctx.lib.tgpu_lookup_memory_bytes(self.h)

    def has_position_links(self):
        return bool(self.ctx.lib.tgpu_lookup_has_duplicates(self.h))

    def get_join_positions(self, keys_page):
        ap = _as_abi_page(keys_page)
        n = keys_page.position_count
        out = np.empty(n, dtype=np.int32)
        self.ctx.check(self.ctx.lib.tgpu_lookup_get_join_positions(self.ctx.h, self.h, ap.ref(), C.c_void_p(out.ctypes.data)))
        return out

    def get_join_positions_device(self, device_page, out_ptr):
        self.ctx.check(self.ctx.lib.tgpu_lookup_get_join_positions(self.ctx.h, self.h, device_page.ref(), C.c_void_p(out_ptr)))

    def key_domain(self, max_values):
        """DynamicFilterSourceOperator / JoinDomainBuilder: (min, max, distinct count, sorted values or None, has_null) of the
        build-side join key; values are None when there are more than max_values distinct keys (range fallback)."""
        lo, hi, cnt, has_null = C.c_int64(), C.c_int64(), C.c_int64(), C.c_int32()
        vals = np.empty(max(max_values, 1), dtype=np.int64)
        self.ctx.check(self.ctx.lib.tgpu_lookup_key_domain(self.ctx.h, self.h, max_values, C.byref(lo), C.byref(hi), C.byref(cnt),
                                                            vals.ctypes.data_as(C.POINTER(C.c_int64)), C.byref(has_null)))
        values = vals[:cnt.value].copy() if cnt.value <= max_values else None
        return lo.value, hi.value, cnt.value, values, bool(has_null.value)

    def position_links(self):
        out = np.empty(self.get_join_position_count(), dtype=np.int32)
        self.ctx.check(self.ctx.lib.tgpu_lookup_copy_position_links(self.ctx.h, self.h, C.c_void_p(out.ctypes.data)))
        return out

    def close(self):
        if self.h:
            self.ctx.lib.tgpu_lookup_release(self.h)
            self.h = None


class JoinBridge:
    """The JoinBridgeManager / PartitionedLookupSourceFactory hand-off (PartitionedLookupSourceFactory.java:100,126):
    the build operator lends its LookupSource, probe operators take it once it is there."""

    def __init__(self):
        self.lookup_source = None

    def lend(self, lookup_source):
        self.lookup_source = lookup_source

    def is_built(self):
        return self.lookup_source is not None


class HashBuilderOperator(Operator):
    def __init__(self, ctx, handle, bridge):
        super().__init__(ctx, handle)
        self.bridge = bridge

    def finish(self):
        super().finish()
        if not self.bridge.is_built():
            lk = C.c_void_p()
            self.ctx.check(self.ctx.lib.tgpu_join_build_get_lookup(self.h, C.byref(lk)))
            self.bridge.lend(LookupSource(self.ctx, lk))


class HashBuilderOperatorFactory(OperatorFactory):
    def __init__(self, ctx, bridge, hash_channels, output_channels, expected_positions=10_000, filter=None, num_build_channels=None):
        """filter: the join filter function (filterFunctionFactory) as an expression tree over the join-sources layout - build channels
        0 .. num_build_channels-1, then the probe channels; num_build_channels = buildLayout.size(), required with a filter"""
        super().__init__()
        self.ctx, self.bridge = ctx, bridge
        self.hash_channels, self.output_channels, self.expected_positions = list(hash_channels), list(output_channels), expected_positions
        self.filter, self.num_build_channels = filter, num_build_channels
        self.filter_program = None
        if filter is not None:
            if num_build_channels is None:
                raise ValueError("a join filter needs num_build_channels (the build layout's size)")
            self.filter_program = PageProcessorProgram(filter, [])

    def _create(self):
        kc, oc = _i32(self.hash_channels), _i32(self.output_channels)
        spec = abi.JoinBuildSpec(len(self.hash_channels), C.cast(kc, C.POINTER(C.c_int32)), len(self.output_channels),
                                 C.cast(oc, C.POINTER(C.c_int32)), self.expected_positions)
        h = C.c_void_p()
        if self.filter_program is None:
            self.ctx.check(self.ctx.lib.tgpu_join_build_create(self.ctx.h, C.byref(spec), C.byref(h)))
        else:
            self.ctx.check(self.ctx.lib.tgpu_join_build_create_filtered(self.ctx.h, C.byref(spec), C.byref(self.filter_program.struct),
                                                                         int(self.num_build_channels), C.byref(h)))
        return HashBuilderOperator(self.ctx, h, self.bridge)

    def duplicate(self):
        raise RuntimeError("Parallel hash build can not be duplicated")   # HashBuilderOperator.java:131-134


class LookupJoinOperatorFactory(OperatorFactory):
    def __init__(self, ctx, bridge, join_type, output_single_match, probe_join_channels, probe_output_channels):
        super().__init__()
        self.ctx, self.bridge, self.join_type, self.output_single_match = ctx, bridge, join_type, output_single_match
        self.probe_join_channels, self.probe_output_channels = list(probe_join_channels), list(probe_output_channels)

    def _create(self):
        if not self.bridge.is_built():
            # PageJoiner.process blocks on lookupSourceFuture (PageJoiner.java:102-105); here the driver must build first
            raise RuntimeError("lookup source is not built yet")
        kc, oc = _i32(self.probe_join_channels), _i32(self.probe_output_channels)
        spec = abi.JoinProbeSpec(self.join_type, int(self.output_single_match), len(self.probe_join_channels), C.cast(kc, C.POINTER(C.c_int32)),
                                 len(self.probe_output_channels), C.cast(oc, C.POINTER(C.c_int32)))
        h = C.c_void_p()
        self.ctx.check(self.ctx.lib.tgpu_join_probe_create(self.ctx.h, C.byref(spec), self.bridge.lookup_source.h, C.byref(h)))
        return Operator(self.ctx, h)

    def duplicate(self):
        return LookupJoinOperatorFactory(self.ctx, self.bridge, self.join_type, self.output_single_match, self.probe_join_channels,
                                         self.probe_output_channels)


class LookupOuterOperatorFactory(OperatorFactory):
    """M/operator/join/LookupOuterOperator.java:38-95.  `probe_output_types`: tgpu types of the probe output channels."""

    def __init__(self, ctx, bridge, probe_output_types):
        super().__init__()
        self.ctx, self.bridge, self.probe_output_types = ctx, bridge, list(probe_output_types)

    def _create(self):
        if not self.bridge.is_built():
            raise RuntimeError("lookup source is not built yet")
        t = _i32(self.probe_output_types)
        h = C.c_void_p()
        self.ctx.check(self.ctx.lib.tgpu_join_outer_create(self.ctx.h, self.bridge.lookup_source.h, C.cast(t, C.POINTER(C.c_int32)), len(self.probe_output_types),
                                                            C.byref(h)))
        return Operator(self.ctx, h)


class SetBuilderOperatorFactory(OperatorFactory):
    """M/operator/SetBuilderOperator.java: the ChannelSet of a semi-join is a lookup source over one channel without outputs."""

    def __init__(self, ctx, bridge, set_channel, expected_positions=0):
        super().__init__()
        self.inner = HashBuilderOperatorFactory(ctx, bridge, [set_channel], [], expected_positions)

    def _create(self):
        return self.inner.create_operator()


class HashSemiJoinOperatorFactory(OperatorFactory):
    """M/operator/HashSemiJoinOperator.java:43-100"""

    def __init__(self, ctx, bridge, probe_join_channel):
        super().__init__()
        self.ctx, self.bridge, self.probe_join_channel = ctx, bridge, probe_join_channel

    def _create(self):
        if not self.bridge.is_built():
            raise RuntimeError("channel set is not built yet")
        h = C.c_void_p()
        self.ctx.check(self.ctx.lib.tgpu_semi_join_create(self.ctx.h, self.bridge.lookup_source.h, self.probe_join_channel, C.byref(h)))
        return Operator(self.ctx, h)


# ---- partitioned output -----------------------------------------------------------------------------
class ColumnDomain:
    """One column's Domain of a dynamic filter's TupleDomain (S/predicate/Domain.java): nullAllowed + a value set.
    Constructors mirror the reference's factories: all / none / only_null / single_value / multiple_values / range (end exclusive,
    like Range.range(type, lo, true, hi, false) in the reference's tests)."""

    def __init__(self, channel, kind, null_allowed=False, lo=0, hi=0, values=None):
        self.channel, self.kind, self.null_allowed, self.lo, self.hi, self.values = channel, kind, null_allowed, lo, hi, values

    @staticmethod
    def all(channel):
        return ColumnDomain(channel, abi.DOMAIN_ALL, True)

    @staticmethod
    def none(channel):
        return ColumnDomain(channel, abi.DOMAIN_NONE, False)

    @staticmethod
    def only_null(channel):
        return ColumnDomain(channel, abi.DOMAIN_NONE, True)

    @staticmethod
    def single_value(channel, value, null_allowed=False):
        return ColumnDomain(channel, abi.DOMAIN_DISCRETE, null_allowed, values=[value])

    @staticmethod
    def multiple_values(channel, values, null_allowed=False):
        return ColumnDomain(channel, abi.DOMAIN_DISCRETE, null_allowed, values=list(values))

    @staticmethod
    def range(channel, lo, hi_exclusive, null_allowed=False):
        """[lo, hi_exclusive) over an integer channel (the bound becomes hi_exclusive - 1); DOUBLE channels take double_range"""
        return ColumnDomain(channel, abi.DOMAIN_RANGE, null_allowed, lo=lo, hi=hi_exclusive - 1)

    @staticmethod
    def double_range(channel, lo, hi, null_allowed=False):
        """[lo, hi] over a DOUBLE channel, both bounds inclusive floats (passed as their raw IEEE bits; compared by value)"""
        lo_bits, hi_bits = np.array([lo, hi], dtype=np.float64).view(np.int64).tolist()
        return ColumnDomain(channel, abi.DOMAIN_RANGE, null_allowed, lo=lo_bits, hi=hi_bits)


class DynamicFilterOperator(Operator):
    def update(self, domains):
        arr, keep = _domains(domains)
        self.ctx.check(self.ctx.lib.tgpu_dynamic_filter_update(self.h, C.cast(arr, C.c_void_p), len(domains)))

    def is_effective(self, index):
        v = C.c_int32()
        self.ctx.check(self.ctx.lib.tgpu_dynamic_filter_is_effective(self.h, index, C.byref(v)))
        return bool(v.value)


def _domains(domains):
    arr = (abi.Domain * max(1, len(domains)))()
    keep = []
    for i, d in enumerate(domains):
        arr[i].channel, arr[i].null_allowed, arr[i].kind = d.channel, int(d.null_allowed), d.kind
        arr[i].min, arr[i].max = d.lo, d.hi
        if d.values is not None:
            vals = (C.c_int64 * len(d.values))(*d.values)
            keep.append(vals)
            arr[i].num_values = len(d.values)
            arr[i].values = C.cast(vals, C.POINTER(C.c_int64))
    return arr, keep


class DynamicFilterOperatorFactory(OperatorFactory):
    """DynamicPageFilter (M/sql/gen/columnar/DynamicPageFilter.java:47-211) as an operator in front of the probe: drops the rows the
    build side's key domain rules out.  `domains`: ColumnDomains in evaluation order; none = TupleDomain.all()."""

    def __init__(self, ctx, domains, selectivity_threshold=1.0):
        super().__init__()
        self.ctx, self.domains, self.threshold = ctx, list(domains), selectivity_threshold

    def _create(self):
        arr, keep = _domains(self.domains)
        h = C.c_void_p()
        self.ctx.check(self.ctx.lib.tgpu_dynamic_filter_create(self.ctx.h, C.cast(arr, C.c_void_p), len(self.domains), self.threshold, C.byref(h)))
        return DynamicFilterOperator(self.ctx, h)

    def duplicate(self):
        return DynamicFilterOperatorFactory(self.ctx, self.domains, self.threshold)


class PartitionedOutputOperator(Operator):
    def get_output_with_partition(self):
        """(partition, Page) or None — the OutputBuffer.enqueue(partition, pages) call of PagePartitioner.java:484-487"""
        page = self.get_output()
        if page is None:
            return None
        p = C.c_int32()
        self.ctx.check(self.ctx.lib.tgpu_partition_last_output_partition(self.h, C.byref(p)))
        return p.value, page

    def get_partitions(self, page):
        ap = _as_abi_page(page)
        out = np.empty(page.position_count, dtype=np.int32)
        self.ctx.check(self.ctx.lib.tgpu_partition_get_partitions(self.h, ap.ref(), C.c_void_p(out.ctypes.data)))
        return out


class PartitionedOutputOperatorFactory(OperatorFactory):
    """PartitionedOutputFactory.createOutputOperator (M/operator/output/PartitionedOutputOperator.java:69-118).
    `partition_constants`: one entry per partition channel, None or a one-position Block - read where the channel is negative
    (PagePartitioner.java:78-101).  `partition_function`: abi.PARTITION_HASH_BUCKET, or abi.PARTITION_LOCAL for the
    LocalPartitionGenerator of the local exchange (M/operator/exchange/LocalPartitionGenerator.java:45-77)."""

    def __init__(self, ctx, partition_channels, bucket_count, bucket_to_partition=None, null_channel=-1, replicates_any_row=False,
                 partition_constants=None, partition_function=abi.PARTITION_HASH_BUCKET):
        super().__init__()
        self.ctx, self.partition_channels, self.bucket_count = ctx, list(partition_channels), bucket_count
        self.bucket_to_partition, self.null_channel, self.replicates_any_row = bucket_to_partition, null_channel, replicates_any_row
        self.partition_constants, self.partition_function = partition_constants, partition_function

    def _create(self):
        kc = _i32(self.partition_channels)
        b2p = _i32(list(self.bucket_to_partition)) if self.bucket_to_partition is not None else None
        constants = None
        if self.partition_constants is not None:
            blocks = [b if b is not None else Block.bigint(np.zeros(1, dtype=np.int64)) for b in self.partition_constants]
            constants = AbiPage(Page(*blocks))      # alive until the create call returns: the library keeps only the hashes
        spec = abi.PartitionSpec(len(self.partition_channels), C.cast(kc, C.POINTER(C.c_int32)), self.bucket_count,
                                 C.cast(b2p, C.POINTER(C.c_int32)) if b2p is not None else None, self.null_channel, int(self.replicates_any_row),
                                 self.partition_function, C.cast(constants.columns, C.c_void_p) if constants is not None else None)
        h = C.c_void_p()
        self.ctx.check(self.ctx.lib.tgpu_partition_create(self.ctx.h, C.byref(spec), C.byref(h)))
        return PartitionedOutputOperator(self.ctx, h)

    def duplicate(self):
        return PartitionedOutputOperatorFactory(self.ctx, self.partition_channels, self.bucket_count, self.bucket_to_partition, self.null_channel,
                                                self.replicates_any_row, self.partition_constants, self.partition_function)


class LocalPartitionGenerator:
    """M/operator/exchange/LocalPartitionGenerator.java:23-77 over the library's partitioner: getPartitions of a page's hash channels."""

    def __init__(self, ctx, hash_channels, partition_count):
        if partition_count < 1 or partition_count & (partition_count - 1):
            raise ValueError("partitionCount must be a power of 2")                 # LocalPartitionGenerator.java:33
        self.partition_count = partition_count
        self._op = PartitionedOutputOperatorFactory(ctx, hash_channels, partition_count, partition_function=abi.PARTITION_LOCAL).create_operator()

    def get_partitions(self, page):
        return self._op.get_partitions(page)

    def close(self):
        self._op.close()


def drive(operator, pages):
    """The relevant slice of Driver.processInternal (M/operator/Driver.java:391-424) for one operator:
    feed pages while needsInput, drain getOutput, then finish and drain.  Returns the output pages."""
    out = []
    for p in pages:
        while not operator.needs_input():
            o = operator.get_output()
            if o is not None:
                out.append(o)
        operator.add_input(p)
        while True:
            o = operator.get_output()
            if o is None:
                break
            out.append(o)
    operator.finish()
    while not operator.is_finished():
        o = operator.get_output()
        if o is not None:
            out.append(o)
        elif operator.is_finished():
            break
    return out
