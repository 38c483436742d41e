/*
 * vexb200.h -- C ABI of libvexb200.so, the Hopper (sm_90a) compute back end
 * that sits behind the vex:: C++ front end in include/vexcl/.
 *
 * This is the drop-in boundary (SURVEY.md section 8b).  Every entry point
 * replaces one thing the reference's hot path does through its
 * `vex::backend` layer (reference paths are relative to /root/reference):
 *
 *   lifecycle / props   <- backend::queue_list, backend::device
 *                          (vexcl/backend/cuda/context.hpp:96-155, :385-413)
 *   streams / events    <- backend::command_queue, backend::event
 *                          (vexcl/backend/cuda/context.hpp:205-260, event.hpp:54-123)
 *   memory              <- backend::device_vector<T> ctor/read/write
 *                          (vexcl/backend/cuda/device_vector.hpp:66-210)
 *   vexb_eval           <- detail::assign_expression launch loop body
 *                          (vexcl/operations.hpp:1818-1897)
 *   vexb_reduce*        <- Reductor::operator() device stage + host fold
 *                          (vexcl/reductor.hpp:302-439)
 *   vexb_partition      <- partitioning_scheme<>::get (vexcl/vector.hpp:131-167)
 *   vexb_halo_plan_*    <- SpMat::setup_exchange (vexcl/spmat.hpp:291-378)
 *   vexb_csr_create /
 *   vexb_spmv           <- SpMatCSR / SpMatHELL ctor + mul_local/mul_remote
 *                          (vexcl/spmat/csr.inl:45-209, hybrid_ell.inl:53-330)
 *   vexb_bsr_create /
 *   vexb_bspmv          <- sparse::matrix<block value> ctor + product with the
 *                          value types of rhs_of / spmv_ops_impl
 *                          (vexcl/sparse/distributed.hpp:17-21, spmv_ops.hpp)
 *   vexb_zsr_create /
 *   vexb_zspmv          <- sparse::matrix<std::complex<T>> ctor + product with
 *                          the spmv_ops_impl of examples/complex_spmv.cpp
 *   vexb_usr_create /
 *   vexb_usr_spmv       <- sparse::matrix<user value type> ctor + product
 *                          generated from its spmv_ops_impl snippets
 *                          (sparse/spmv_ops.hpp, sparse/csr.hpp:109-126)
 *   vexb_dspmat_*       <- SpMat ctor + SpMat::apply (vexcl/spmat.hpp:71-185)
 *   vexb_ccsr_*         <- SpMatCCSR ctor + its generated product function
 *                          (vexcl/spmat/ccsr.hpp:70-78, :176-201)
 *   vexb_comm_*         <- the host-staged D2H/H2D halo and the host fold of
 *                          reduction partials (spmat.hpp:149-176,
 *                          reductor.hpp:412-436), moved to NCCL over NVLink.
 *
 * Conventions: plain pointers and sizes only; every function returns 0
 * (VEXB_OK) on success and a vexb_status code otherwise and never throws;
 * vexb_last_error() returns a thread-local "file:line: message" string for
 * the last failure on the calling thread.  All `stream` arguments are
 * cudaStream_t passed as void* (NULL = the legacy default stream).  Device
 * pointers are owned by the caller unless stated otherwise.  The library is
 * thread-compatible: concurrent calls that touch different streams/handles
 * are legal, there is no shared argument stack (contrast
 * vexcl/backend/cuda/kernel.hpp:44-241).
 *
 * There is NO CPU fallback: compute entry points fail with VEXB_ERR_CUDA when
 * no CUDA device is usable.
 */
#ifndef VEXB200_H
#define VEXB200_H

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define VEXB_ABI_VERSION 1

typedef enum {
    VEXB_OK = 0,
    VEXB_ERR_CUDA = 1,        /* a CUDA runtime call failed               */
    VEXB_ERR_INVALID = 2,     /* bad argument / precondition violated     */
    VEXB_ERR_NCCL = 3,        /* NCCL missing or an NCCL call failed      */
    VEXB_ERR_UNSUPPORTED = 4, /* valid request the back end cannot serve  */
    VEXB_ERR_NOMEM = 5,
    VEXB_ERR_PEER = 6         /* a peer GPU did not arrive in a fused combine / peer-memory halo */
} vexb_status;

/* Scalar element types (subset of vexcl/types.hpp:202-260). */
typedef enum {
    VEXB_F64 = 0, VEXB_F32 = 1, VEXB_I32 = 2, VEXB_U32 = 3, VEXB_I64 = 4, VEXB_U64 = 5
} vexb_dtype;

/* Assignment operators, same set and order as vexcl/operations.hpp:70-80. */
typedef enum {
    VEXB_SET = 0, VEXB_ADD = 1, VEXB_SUB = 2, VEXB_MUL = 3, VEXB_DIV = 4, VEXB_MOD = 5,
    VEXB_AND = 6, VEXB_OR = 7, VEXB_XOR = 8, VEXB_LSH = 9, VEXB_RSH = 10
} vexb_assign;

/* Reduction kinds (vexcl/reductor.hpp:47-128, :132-280). */
typedef enum {
    VEXB_SUM = 0, VEXB_SUM_KAHAN = 1, VEXB_MAX = 2, VEXB_MIN = 3,
    VEXB_MINMAX = 4 /* result[0]=min, result[1]=max, as MIN_MAX (reductor.hpp:262-280) */
} vexb_reduce_op;

/* ------------------------------------------------------------------------
 * Expression IR.  The front end lowers a vex:: expression tree to a postfix
 * program over a table of terminals; this replaces the source text the
 * reference emits in vexcl/operations.hpp:1209-1353.
 * ---------------------------------------------------------------------- */
#define VEXB_MAX_TERMS 16
#define VEXB_MAX_CODE  64
#define VEXB_MAX_STACK 12
#define VEXB_MAX_TEMPS 8   /* temporary slots of one program (VEXB_OP_TDEF / VEXB_OP_TREF) */

typedef enum {
    VEXB_TERM_VEC = 0,    /* v.ptr: device array of `dtype`, element i of this device slice */
    VEXB_TERM_SCALAR = 1, /* by-value scalar of `dtype` (operations.hpp:168-175)            */
    VEXB_TERM_INDEX = 2,  /* element_index: index_offset + i + v.i64 (element_index.hpp:40-111), type u64 */
    VEXB_TERM_DSCALAR = 3,/* v.ptr: ONE device-resident value of `dtype`, broadcast to every element.  Lets the
                             result of vexb_reduce feed the next expression without a host round trip. */
    VEXB_TERM_SPMV = 4,   /* v.ptr: a vexb_spmat (host handle; CSR or hybrid ELL, plain strip -- or, in vexb_eval only,
                             sliced ELL: see vexb_dspmat_sweep_strip); pad[0]: slot of the
                             VEXB_TERM_VEC holding x.  Element i evaluates to row i of A*x (products added in storage
                             order, as vexb_spmv does): the sparse product as a *terminal* of the consumer's kernel --
                             `y = x + A*x` is one launch, y is written once and A*x never goes to memory
                             (vexcl/sparse/product.hpp:45-130, sparse/csr.hpp:102-132, sparse/ell.hpp:207-265,
                             spmat/inline_spmv.hpp:68-76).  Expressions with such terminals run on the NVRTC side path
                             (the row loop is generated into the kernel, specialised to the strip's format and width),
                             reductions of them included (vexb_reduce_all / vexb_reduce_multi). */
    VEXB_TERM_CCSR = 5,   /* v.ptr: a vexb_ccsr (host handle); pad[0]: slot of the VEXB_TERM_VEC holding x; pad[1]: the
                             matrix's idx width on the device (vexb_ccsr_info.idx_bytes: 1, 2 or 4); dtype: the matrix's
                             value type, which is also x's.  Element i evaluates to
                                 s = 0;  s = s + val[j] * x[i + col[j]]  for j over the unique row idx[i], in storage order,
                             every product and sum rounded on its own: the bits of vexb_ccsr_spmv(alpha = 1, append = 0) at
                             row i -- the reference's ccsr_product terminal (spmat/ccsr.hpp:88-270), `sin(A*x)`,
                             `x * (A*x)`, `sum(x * (A*x))` in one launch.  Served like VEXB_TERM_SPMV by the NVRTC kernels of
                             vexb_eval, vexb_reduce_all and vexb_reduce_multi (one kernel per value type and idx width, not per
                             matrix: the row loop reads the unique-row table through a small device descriptor that the
                             handle allocates, with a blocking copy, at its first use as a terminal); vexb_eval_multi reports
                             it as not handled.  Checked before any launch (VEXB_ERR_INVALID otherwise): the handle lives on
                             `dev`, dtype is its value type, the call covers the whole matrix (index_offset 0, n = nrows),
                             pad[0] names a vector terminal of that type, pad[1] agrees with the handle.  vexb_eval returns
                             VEXB_ERR_UNSUPPORTED when x is the assignment's target (threads would write x[i] while others
                             read x[i + col[j]]): evaluate the product into a temporary first. */
    VEXB_TERM_PTR = 6     /* v.ptr: the device address of element 0 of an array of `dtype` (vex::raw_pointer,
                             vexcl/vector_pointer.hpp); pad[0..5]: the array's element count, little-endian.  It gives the
                             expression no size.  An element is read by VEXB_OP_LOAD, and a LOAD outside [0, count) reads 0
                             without touching memory: every branch of a SELECT is evaluated, so `i > 0 ? p[i - 1] : 0` must
                             not fault at i = 0, as the reference's lazy `?:` does not.  A VEXB_OP_TERM on it
                             pushes the pointer itself, with type VEXB_PTR(dtype), which is legal only as the argument of a
                             VEXB_OP_CALL whose function declared that parameter VEXB_PTR(dtype).  Pointers travel in the
                             terminal table as vectors do, so one compiled kernel serves every pointer of one request shape.
                             NULL is refused outside the source printers.  vexb_eval and vexb_eval_multi return
                             VEXB_ERR_UNSUPPORTED, before any launch, when a pointer addresses a target slice (threads would read
                             elements that others overwrite): the front ends then redirect it to a device copy of the vector.
                             vexb_eval_multi reports no "not handled" fall-back in that case, since component by component
                             would race too.  Pointers are not taken by stencil operators or as a sparse product's x. */
} vexb_term_kind;

/* The type of a pointer to `dtype` elements: the value a VEXB_OP_TERM on a VEXB_TERM_PTR pushes, and a parameter type of
 * vexb_function_register(_ex) (never a return type).  A function registered with VEXB_F64 and one with VEXB_PTR(VEXB_F64)
 * for the same parameter are two functions. */
#define VEXB_PTR(dtype) ((dtype) | 0x10)

typedef struct {
    uint8_t kind;   /* vexb_term_kind */
    uint8_t dtype;  /* vexb_dtype     */
    uint8_t pad[6];
    union { const void *ptr; double f64; float f32; int32_t i32; uint32_t u32; int64_t i64; uint64_t u64; } v;
} vexb_term;

/* Opcodes.  `type` of an instruction is the vexb_dtype the node evaluates in
 * (operands of binary ops must already have that type: the front end inserts
 * VEXB_OP_CVT following the usual arithmetic conversions).  Comparisons and
 * logical ops take operands of `type` and produce I32 0/1. */
typedef enum {
    VEXB_OP_TERM = 0,  /* push term[arg] converted to nothing: its own dtype            */
    VEXB_OP_CVT,       /* convert top from dtype `arg` to `type`                         */
    /* unary */
    VEXB_OP_NEG, VEXB_OP_LNOT,
    /* binary arithmetic / bitwise */
    VEXB_OP_ADD, VEXB_OP_SUB, VEXB_OP_MUL, VEXB_OP_DIV, VEXB_OP_MOD,
    VEXB_OP_BAND, VEXB_OP_BOR, VEXB_OP_BXOR, VEXB_OP_SHL, VEXB_OP_SHR,
    /* comparisons / logical (result I32) */
    VEXB_OP_LT, VEXB_OP_GT, VEXB_OP_LE, VEXB_OP_GE, VEXB_OP_EQ, VEXB_OP_NE,
    VEXB_OP_LAND, VEXB_OP_LOR,
    /* ternary: stack [cond(I32) a b] -> cond ? a : b  (if_else, operations.hpp:1277-1301) */
    VEXB_OP_SELECT,
    /* builtin functions (vexcl/function.hpp:287-...), floating types only unless noted */
    VEXB_OP_SIN, VEXB_OP_COS, VEXB_OP_TAN, VEXB_OP_ASIN, VEXB_OP_ACOS, VEXB_OP_ATAN,
    VEXB_OP_SINH, VEXB_OP_COSH, VEXB_OP_TANH, VEXB_OP_EXP, VEXB_OP_EXP2, VEXB_OP_LOG,
    VEXB_OP_LOG2, VEXB_OP_LOG10, VEXB_OP_SQRT, VEXB_OP_RSQRT, VEXB_OP_CBRT, VEXB_OP_FABS /* also ints: abs */,
    VEXB_OP_FLOOR, VEXB_OP_CEIL, VEXB_OP_ROUND, VEXB_OP_TRUNC,
    VEXB_OP_POW, VEXB_OP_ATAN2, VEXB_OP_FMOD, VEXB_OP_HYPOT,
    VEXB_OP_FMIN /* also ints: min */, VEXB_OP_FMAX /* also ints: max */,
    VEXB_OP_FMA,      /* ternary: a*b+c with one rounding (builtin fma)                 */
    VEXB_OP_CALL,     /* user function (VEX_FUNCTION): arg = id from vexb_function_register; pops its
                         declared number of arguments (already converted to the declared types), pushes
                         `type` = its return type.  Expressions with calls run on the NVRTC side path. */
    /* Temporaries (vex::make_temp, vexcl/temporary.hpp): a subexpression evaluated once per element into a local
     * variable that every use reads.  TDEF pops one value of `type` into temporary slot `arg` (< VEXB_MAX_TEMPS); it is
     * legal only at stack depth 1 and leaves the stack empty, so every definition comes before the main expression (a
     * program is: definitions in post-order, dependencies first, then the expression).  TREF pushes temporary `arg` with
     * the type of its TDEF.  A temporary is evaluated for every element, whether or not a branch of a SELECT reads it,
     * and the program has the bits of the same program with the definition written out at each TREF.  Refused with
     * VEXB_ERR_INVALID by every entry point, before any launch or NVRTC run: a slot >= VEXB_MAX_TEMPS, a second TDEF of
     * one slot, a TREF before its TDEF, a TREF whose type differs from its TDEF's, a TDEF whose type differs from the
     * value on top of the stack, a TDEF at a depth other than 1.  vexb_eval and the reductions serve such programs with
     * the interpreter or the generated kernel, never a hand-written sweep.  In vexb_eval_multi each component's slots
     * are its own; a temporary that two components define by the same instructions over equal terminals (same kind,
     * dtype and pointer or value) is computed once per element by the generated kernel and handed to both. */
    VEXB_OP_TDEF,
    VEXB_OP_TREF,
    /* Subscript and dereference through a raw pointer (the reference grammar's `a[b]` and `*p`, operations.hpp:493-494):
     * `arg` is the slot of a VEXB_TERM_PTR terminal and `type` is its dtype; pops one VEXB_I64 index and pushes ptr[index],
     * or 0 when the index is outside [0, count) of the terminal.
     * The front ends fold C pointer arithmetic into the index: each offset is widened on its own (signed types
     * sign-extended, unsigned zero-extended, U64 reinterpreted), then the offsets are added in I64, so *(p + a), *(p - a),
     * p[a], (p + a)[b], a + p and *p are all one LOAD.  Refused with VEXB_ERR_INVALID by every entry point, before any
     * launch or NVRTC run: an `arg` that is not a pointer terminal, an index that is not I64, a `type` other than the
     * pointer's dtype, and a pointer value anywhere but a matching call parameter (arithmetic, CVT, TDEF, SELECT, the
     * result).  vexb_eval and the reductions serve such programs with the interpreter or the generated kernel, never a
     * hand-written sweep.  Loads take the read-only path in generated kernels unless the kernel passes a pointer to a
     * user function, whose body may write through it. */
    VEXB_OP_LOAD,
    VEXB_OP_COUNT_
} vexb_opcode;

typedef struct {
    uint8_t  op;    /* vexb_opcode */
    uint8_t  type;  /* vexb_dtype  */
    uint16_t arg;   /* TERM / LOAD: term slot; CVT: source dtype; CALL: function id; TDEF / TREF: temporary slot */
} vexb_instr;

typedef struct {
    int32_t    n_terms;
    int32_t    n_code;
    vexb_term  term[VEXB_MAX_TERMS];
    vexb_instr code[VEXB_MAX_CODE];
} vexb_expr;

/* ------------------------------------------------------------------------
 * Lifecycle, device properties
 * ---------------------------------------------------------------------- */
typedef struct {
    char     name[256];
    int32_t  cc_major, cc_minor;
    int32_t  sm_count;
    int32_t  max_threads_per_block;
    int32_t  warp_size;
    int32_t  pad;
    size_t   smem_per_block_optin;
    size_t   total_mem;
    size_t   l2_bytes;
} vexb_devprops;

int         vexb_abi_version(void);
const char *vexb_last_error(void);
int vexb_init(void);                       /* idempotent; fails loudly when no CUDA device */
int vexb_shutdown(void);
int vexb_device_count(int *n);
int vexb_device_props(int dev, vexb_devprops *p);
/* Tunables for experiments ("sweep.blocks_per_sm", "spmv.tile_nnz", ...). */
int vexb_set_param(const char *name, long value);
int vexb_get_param(const char *name, long *value);
/* Count of kernels this library has launched from the calling process. */
int vexb_launch_count(uint64_t *n);

/* ------------------------------------------------------------------------
 * Streams and events
 * ---------------------------------------------------------------------- */
int vexb_stream_create(int dev, void **stream);
int vexb_stream_destroy(int dev, void *stream);
int vexb_stream_sync(int dev, void *stream);
int vexb_device_sync(int dev);
int vexb_event_create(int dev, void **event);
int vexb_event_destroy(int dev, void *event);
int vexb_event_record(int dev, void *event, void *stream);
int vexb_event_sync(int dev, void *event);
int vexb_stream_wait_event(int dev, void *stream, void *event);
int vexb_event_elapsed_ms(void *start, void *stop, float *ms);

/* ------------------------------------------------------------------------
 * Memory
 * ---------------------------------------------------------------------- */
int vexb_malloc(int dev, size_t bytes, void **p);
int vexb_free(int dev, void *p);
int vexb_host_alloc(size_t bytes, void **p);   /* pinned host memory */
int vexb_host_free(void *p);
int vexb_h2d(int dev, void *dst, const void *src, size_t bytes, void *stream, int blocking);
int vexb_d2h(int dev, void *dst, const void *src, size_t bytes, void *stream, int blocking);
int vexb_d2d(int dev, void *dst, const void *src, size_t bytes, void *stream);
int vexb_memset(int dev, void *dst, int byte, size_t bytes, void *stream);

/* ------------------------------------------------------------------------
 * Partitioning (host only; no GPU needed)
 * vexcl/vector.hpp:131-167 with util.hpp:91-93 (alignup 16).
 * weights == NULL means equal weights (vector.hpp:79-81).
 * part must hold nparts+1 entries.
 * ---------------------------------------------------------------------- */
int vexb_partition(size_t n, int nparts, const double *weights, size_t *part);

/* ------------------------------------------------------------------------
 * Elementwise: lhs[i] OP= expr(i), i in [0,n) of one device slice.
 * Replaces the per-device kernel launch of assign_expression
 * (operations.hpp:1886-1895).  Asynchronous on `stream`.
 * ---------------------------------------------------------------------- */
int vexb_eval(int dev, void *stream, void *lhs, int lhs_dtype, int assign_op,
              const vexb_expr *expr, size_t n, size_t index_offset);
/* User-defined device functions (VEX_FUNCTION, vexcl/function.hpp:225): `body` is C source that refers to its
 * arguments as prm1, prm2, ... (the reference's convention) and returns a value of `ret_dtype`.  An argument type may
 * be VEXB_PTR(dtype): the parameter is then `T *prmK`, and the call passes a VEXB_TERM_PTR terminal.
 * Such functions cannot be pre-compiled: an expression that calls one is turned into CUDA source
 * (the sweep skeleton with the expression inlined), compiled once with NVRTC for sm_90a, cached, and launched
 * through the driver API.  Setting the tunable "eval.jit" = 1 sends every non-sweep expression down the same
 * path instead of the interpreter.  Registering the same definition twice returns the same id. */
int vexb_function_register(const char *name, int ret_dtype, int nargs, const int *arg_dtypes,
                           const char *body, int *id);
/* The same with dependencies and a preamble (VEX_FUNCTION_D / _SD / _DS, VEX_FUNCTION_V1_WITH_PREAMBLE,
 * vexcl/function.hpp:70-203); vexb_function_register is this with ndeps = 0 and no preamble.
 *   deps[0..ndeps) (ndeps <= 64): ids of functions registered before, which `body` calls by their plain names.  A
 *     program that calls this function holds the closure of the dependency lists, post-order as written (a dependency
 *     before its dependents), each function of it once and under its plain name `name`; the called function itself
 *     is emitted as name_<id>, and under its plain name as well when it is also a dependency.  Two distinct functions
 *     with one plain name in a program's dependencies: VEXB_ERR_INVALID, before NVRTC runs.
 *   preamble (NULL or ""): file-scope text emitted once per program, before the function's first definition.  A
 *     program with a preamble is compiled with NVRTC --device-as-default-execution-space, so helpers in it may be
 *     written without __device__.
 * The same (name, ret_dtype, arg_dtypes, body, deps, preamble) returns the same id. */
int vexb_function_register_ex(const char *name, int ret_dtype, int nargs, const int *arg_dtypes, const char *body,
                              int ndeps, const int *deps, const char *preamble, int *id);
/* Program headers (vex::push_program_header, backend/common.hpp:120-206): a stack per device ordinal, host state only
 * (no device is touched).  A push replaces the effective header (the top), a pop restores the previous one; popping an
 * empty stack is VEXB_ERR_INVALID.  The effective header of `dev` goes at the very top of every program compiled for dev
 * that carries user text -- vexb_eval, vexb_eval_multi, vexb_reduce_all and vexb_reduce_multi kernels that call a user
 * function, vexb_stencil_operator_apply and vexb_usr_spmv -- and into those kernels' cache keys; a background
 * compilation uses the header in effect when it was requested.  _get: the effective header ("" when none), two-call
 * pattern on *len. */
int vexb_program_header_push(int dev, const char *text);
int vexb_program_header_pop(int dev);
int vexb_program_header_get(int dev, char *buf, size_t *len);
/* Generated source and NVRTC build log of the kernel vexb_eval would JIT for this request (for inspection
 * and for tests on machines without a GPU: NVRTC needs no device).  Two-call pattern on *len. */
int vexb_jit_source(int lhs_dtype, int assign_op, const vexb_expr *expr, char *buf, size_t *len, int compile);
/* The same for the one kernel vexb_eval_multi generates for ncomp (2..8) components. */
int vexb_jit_source_multi(int lhs_dtype, int assign_op, int ncomp, const vexb_expr *const *exprs, char *buf, size_t *len, int compile);
/* The same for the kernel that reduces an expression with user functions or inlined sparse products in `dtype`: the one
 * vexb_reduce_all generates when nops == 1 (ops[0]: any vexb_reduce_op), the one vexb_reduce_multi generates when
 * nops > 1 (SUM / SUM_KAHAN / MAX / MIN).  The skeleton follows the tunables in force, as at a launch. */
int vexb_jit_source_reduce(int dtype, int nops, const int *ops, const vexb_expr *expr, char *buf, size_t *len, int compile);
/* The three above as device `dev` would compile them now: its program header first when the program calls a user
 * function.  dev = -1 is the header-less text of the functions above.  No device is touched. */
int vexb_jit_source_dev(int dev, int lhs_dtype, int assign_op, const vexb_expr *expr, char *buf, size_t *len, int compile);
int vexb_jit_source_multi_dev(int dev, int lhs_dtype, int assign_op, int ncomp, const vexb_expr *const *exprs, char *buf,
                              size_t *len, int compile);
int vexb_jit_source_reduce_dev(int dev, int dtype, int nops, const int *ops, const vexb_expr *expr, char *buf, size_t *len,
                               int compile);
/* Expressions without a hand-written sweep are served by the pre-compiled interpreter while NVRTC builds a kernel
 * specialised to the expression on a background thread (started at the first use of a new expression shape; tunable
 * "eval.jit": 0 = interpreter only, 1 = compile synchronously, 2 = this, the default).  *pending = 1 while any such
 * compilation is still running: benchmarks and tests wait on it to time / check the specialised kernel. */
int vexb_jit_pending(int *pending);
/* Compile the kernel of a request shape before its first use (background != 0: on a background thread, as the first
 * vexb_eval of a new shape does in the default mode).  Needs NVRTC, no device.  A process may exit while background
 * compilations run: the thread that started them waits for the one in flight and cancels the rest on its way out. */
int vexb_jit_precompile(int lhs_dtype, int assign_op, const vexb_expr *expr, int background);
/* All components of a multi-expression assignment in one launch (assign_multiexpression, operations.hpp:2081-2185):
 * lhs[k][i] OP= exprs[k](i), k < ncomp <= 8, all of one type; every right-hand side of element i is evaluated before
 * any left-hand side of element i is written.  *handled = 0 when the request is not served here (NVRTC missing or
 * still compiling in the background, sparse-product terminals): evaluate component by component then. */
int vexb_eval_multi(int dev, void *stream, int ncomp, void *const *lhs, int lhs_dtype, int assign_op,
                    const vexb_expr *const *exprs, size_t n, size_t index_offset, int *handled);
/* Which kernel vexb_eval would take for this request: writes a short
 * name ("sweep:muladd", "interp", "jit", ...) to buf. */
int vexb_eval_path(int lhs_dtype, int assign_op, const vexb_expr *expr, char *buf, size_t buflen);

/* ------------------------------------------------------------------------
 * Reduction of an expression over one device slice to ONE device-resident
 * value (two for VEXB_MINMAX) of type `dtype`, written to d_result.
 * d_workspace: at least vexb_reduce_workspace_bytes() bytes of device memory
 * private to the (device, stream) in use; it must be zero-initialised once
 * (vexb_memset) before first use and is left reusable after each call.
 * Replaces reductor.hpp:327-410; the host fold :412-436 is replaced by
 * vexb_reduce_fetch (single device) or vexb_comm_allreduce (+ fetch).
 * Expressions that call user functions (VEXB_OP_CALL) or inline sparse products (VEXB_TERM_SPMV) are reduced by ONE
 * kernel NVRTC generates for the request (compiled at its first use, then cached): the row loop or the call feeds the
 * fold directly, and the result has the bits of evaluating the expression into a vector of its own type and reducing
 * that vector with the same tunables.  VEXB_ERR_UNSUPPORTED when NVRTC cannot be loaded: reduce such a temporary then.
 * Expressions that load through raw pointers (VEXB_OP_LOAD) are reduced by such a kernel too, unless "eval.jit" is 0;
 * then, and when NVRTC cannot be loaded, by the interpreter.
 * ---------------------------------------------------------------------- */
typedef struct vexb_peer vexb_peer;   /* a group of GPUs that write each other's memory; see "Peer memory" below */
int vexb_reduce_workspace_bytes(int dev, size_t *bytes);
int vexb_reduce(int dev, void *stream, const vexb_expr *expr, int dtype, size_t n,
                size_t index_offset, int op, void *d_result, void *d_workspace);
/* Several reductions of the SAME expression in one pass over memory: vex::CombineReductors<R...> (reductor.hpp:132-280).
 * ops: nops <= VEXB_MAX_COMBINED of VEXB_SUM / VEXB_SUM_KAHAN / VEXB_MAX / VEXB_MIN; d_result receives nops values of
 * `dtype` in that order; d_workspace must hold nops * vexb_reduce_workspace_bytes() zero-initialised bytes.  With a
 * peer group every value is combined across the GPUs inside the kernel, as in vexb_reduce_all. */
#define VEXB_MAX_COMBINED 16
int vexb_reduce_multi(int dev, void *stream, const vexb_expr *expr, int dtype, size_t n, size_t index_offset,
                      int nops, const int *ops, void *d_result, void *d_workspace, vexb_peer *peer);
/* Fill d_result with the identity of `op` (reductor.hpp:55,87,111): used for empty slices. */
int vexb_reduce_identity(int dev, void *stream, int dtype, int op, void *d_result);
/* D2H of `count` values + stream sync. */
int vexb_reduce_fetch(int dev, void *stream, const void *d_result, int dtype, int count, void *host_out);

/* ------------------------------------------------------------------------
 * Communication (NCCL over NVLink).  NCCL is dlopen()ed on first use.
 *   single process, n devices : vexb_comm_create_all
 *   one process per device    : rank 0 calls vexb_comm_unique_id, the 128-byte
 *                               id is broadcast by the host program, every
 *                               rank calls vexb_comm_create_rank
 * ---------------------------------------------------------------------- */
typedef struct vexb_comm vexb_comm;
#define VEXB_UNIQUE_ID_BYTES 128
int vexb_comm_unique_id(void *id128);
int vexb_comm_create_rank(int dev, int nranks, int rank, const void *id128, vexb_comm **comm);
int vexb_comm_create_all(int ndev, const int *devs, vexb_comm **comms /* ndev out */);
int vexb_comm_destroy(vexb_comm *comm);
int vexb_comm_rank(const vexb_comm *comm, int *rank, int *nranks, int *dev);
/* In-place all-reduce of `count` values on each local device.  op: VEXB_SUM / VEXB_MAX / VEXB_MIN. */
int vexb_comm_allreduce(int nlocal, vexb_comm *const *comms, void *const *bufs, void *const *streams,
                        int count, int dtype, int op);
int vexb_comm_barrier(int nlocal, vexb_comm *const *comms, void *const *streams);

/* ------------------------------------------------------------------------
 * CUDA graphs: record everything enqueued on `stream` (and on streams that
 * fork from / join it through events, e.g. the halo side stream and its NCCL
 * calls) between begin and end, then replay it with one launch.  Replaces the
 * per-kernel host launch loop of the reference for launch-bound inner loops
 * (a CG iteration at 8 GPUs).  Only asynchronous entry points may be called
 * while capturing (no blocking copies, no vexb_reduce_fetch).
 * ---------------------------------------------------------------------- */
typedef struct vexb_graph vexb_graph;
int vexb_graph_begin(int dev, void *stream);
int vexb_graph_end(int dev, void *stream, vexb_graph **graph);
int vexb_graph_launch(vexb_graph *graph, void *stream);
int vexb_graph_destroy(vexb_graph *graph);

/* ------------------------------------------------------------------------
 * Peer memory: a group of ranks (one per GPU) whose kernels write into each
 * other's device memory over NVLink.  Used to fuse the combine of
 * Reductor across GPUs into the reduction kernel itself (vexb_reduce_all):
 * the last block of every rank pushes its value into all peers' mailboxes
 * and folds what it received, in rank order -- one kernel, no NCCL call, no
 * host (replaces reductor.hpp:412-436).
 *   one process per GPU : vexb_peer_create (returns a 64-byte CUDA IPC handle),
 *                         the launcher all-gathers the handles (rank order),
 *                         vexb_peer_connect maps the other ranks' mailboxes;
 *   one process, n GPUs : vexb_peer_create_all (peer access, distinct devices).
 * A rank that never shows up makes the waiting kernel give up after ~20 s:
 * it stores NaN / all-ones instead of a partial fold and raises a sticky fault
 * (vexb_peer_error, vexb_peer_fault) instead of hanging.
 * ---------------------------------------------------------------------- */
#define VEXB_IPC_HANDLE_BYTES 64
int vexb_peer_create(int dev, int rank, int nranks, vexb_peer **peer, void *handle64);
int vexb_peer_connect(vexb_peer *peer, const void *handles /* nranks * 64 bytes, rank order */);
int vexb_peer_create_all(int ndev, const int *devs, vexb_peer **peers /* ndev out */);
int vexb_peer_destroy(vexb_peer *peer);
int vexb_peer_error(vexb_peer *peer, unsigned long long *epoch_of_timeout /* 0 = none */);
/* Process-wide sticky fault: non-zero once any kernel of this process (fused reduction combine, peer-memory halo)
 * gave up waiting for a peer.  Such a kernel never folds or multiplies stale data: the values that needed the peer
 * are written as NaN (floating types) or all-ones (integers).  vexb_reduce_fetch returns VEXB_ERR_PEER while the
 * fault is set; the front ends turn that into an exception.  clear != 0 resets it (after the group was rebuilt). */
int vexb_peer_fault(unsigned long long *epoch, int clear);
/* In-place all-reduce of one value (two for VEXB_MINMAX) per rank. */
int vexb_peer_allreduce(vexb_peer *peer, void *stream, void *d_buf, int dtype, int op);
/* vexb_reduce + the combine across the peer group in the same kernel; every rank ends with the
 * same bits in d_result.  peer == NULL (or a group of one) is plain vexb_reduce. */
int vexb_reduce_all(int dev, void *stream, const vexb_expr *expr, int dtype, size_t n,
                    size_t index_offset, int op, void *d_result, void *d_workspace, vexb_peer *peer);

/* ------------------------------------------------------------------------
 * Halo plan (host only; no GPU needed): who sends which x entries to whom.
 * Input: column partition and, for every part d, the sorted unique list of
 * global column ids outside [col_part[d], col_part[d+1]) referenced by the
 * rows of part d (the `ghost_cols[d]` sets of spmat.hpp:300-316),
 * concatenated, with ghost_off[d]..ghost_off[d+1] delimiting part d.
 * ---------------------------------------------------------------------- */
typedef struct vexb_halo_plan vexb_halo_plan;
/* Ghost columns of one row strip: two-call pattern (out == NULL returns the count). */
int vexb_strip_ghost_cols(size_t nrows, const void *ptr, int ptr_bytes, const void *col, int col_bytes,
                          size_t col_begin, size_t col_end, int64_t *out, size_t *count);
int vexb_halo_plan_create(int nparts, const size_t *col_part, const int64_t *ghost_cols,
                          const size_t *ghost_off, vexb_halo_plan **plan);
int vexb_halo_plan_destroy(vexb_halo_plan *plan);
/* Reference-equivalent tables (spmat.hpp:319-371), for parity checks:
 * cols_to_send: global sorted union (n_send_total entries) with the owner's
 * col_part start subtracted; cidx: nparts+1 offsets into it. */
int vexb_halo_plan_ref_sizes(const vexb_halo_plan *plan, size_t *n_send_total);
int vexb_halo_plan_ref_tables(const vexb_halo_plan *plan, int64_t *cols_to_send, size_t *cidx);
int vexb_halo_plan_ref_recv(const vexb_halo_plan *plan, int part, int64_t *cols_to_recv /* n_ghost(part) */);
/* Pairwise form used by the exchange: for `part`, send_counts[p] values go to
 * peer p (send_cols lists the local x indices, grouped by ascending p);
 * recv_counts[p] values arrive from peer p and land contiguously, in
 * ascending p order, in the ghost buffer (which is ordered like the sorted
 * ghost list, exactly the renumbering of csr.inl:92-96). */
int vexb_halo_plan_counts(const vexb_halo_plan *plan, int part, size_t *send_counts, size_t *recv_counts);
int vexb_halo_plan_send_cols(const vexb_halo_plan *plan, int part, int64_t *send_cols);

/* ------------------------------------------------------------------------
 * Sparse strips (one device).  Input: host CSR with column ids already local
 * to the strip's x (ptr[0] may be non-zero; it is subtracted).  Index width
 * on the device is 32-bit whenever that is lossless.
 * ---------------------------------------------------------------------- */
typedef struct vexb_spmat vexb_spmat;
typedef enum {
    VEXB_FMT_AUTO = 0,  /* CSR row-block stream kernel unless ELL is clearly better */
    VEXB_FMT_CSR = 1,   /* row-block CSR, tiles staged through shared memory by TMA bulk copies */
    VEXB_FMT_HELL = 2,  /* hybrid ELL + CSR tail, width by hybrid_ell.inl:66-114 */
    VEXB_FMT_PATTERNS = 3,/* the strip's unique rows (column offsets from the diagonal + values) and one pattern id per
                             row: the reference's CCSR (spmat/ccsr.hpp) found automatically.  Used when the strip has at
                             most "spmv.max_patterns" (256) distinct rows and no row map; otherwise as VEXB_FMT_AUTO.
                             Opt-in in round 1 (not yet run on a GPU). */
    VEXB_FMT_SELL = 4     /* sliced ELL (SELL-32-sigma): slices of 32 rows stored column-major at the width of their longest
                             row, rows sorted by length inside windows of "spmv.sell_sigma" (1024) rows so that a slice
                             holds rows of similar length.  One warp per slice, one lane per row, coalesced loads, no
                             shared memory, products added in storage order (same bits as the reference loop).  What
                             VEXB_FMT_AUTO picks for rows too irregular for hybrid ELL. */
} vexb_spfmt;
/* Flag ORed into `fmt` of vexb_csr_create / vexb_dspmat_create, double values only: store each value as (float)v (round
 * to nearest even; a finite value that would round to +-inf is rejected with VEXB_ERR_INVALID).  x, y, every product
 * double(v_f) * x_j and every sum stay double, in the order of the double strip: y has the bits of the double strip built
 * from the rounded values, with the same layout (format, width, encoding, classes, tiles).  Only the per-entry value
 * arrays shrink (sliced ELL, hybrid ELL and its CSR tail, CSR); row-class and row-pattern strips keep their small tables
 * in double.  CSR strips run "spmv.kernel" 3 and 4 only (VEXB_ERR_UNSUPPORTED for the others).  Readers without a
 * float-valued kernel refuse such strips: vexb_spmv_multi multiplies one vector at a time, vexb_dspmat_inline_strip gives
 * NULL, vexb_dspmat_halo_connect* and vexb_dspmat_apply_dot return VEXB_ERR_UNSUPPORTED. */
#define VEXB_FMT_VALUES_F32 0x100
/* Host-only: the row patterns VEXB_FMT_PATTERNS would use.  *n_patterns = number of distinct rows; idx (optional,
 * nrows entries) = pattern of each row.  Returns VEXB_ERR_UNSUPPORTED when there are more than max_patterns. */
int vexb_csr_row_patterns(size_t nrows, const void *ptr, int ptr_bytes, const void *col, int col_bytes,
                          const void *val, int val_dtype, size_t max_patterns, size_t *n_patterns, int32_t *idx);

/* Host-only: the sliced-ELL layout VEXB_FMT_SELL would use.  perm (optional, 32 * n_slices entries): the row each slice
 * lane multiplies, -1 = none; slice_ptr (optional, n_slices + 1): first slot of each slice.  sigma = sorting window. */
int vexb_csr_sell_layout(size_t nrows, const void *ptr, int ptr_bytes, long sigma, size_t *n_slices, size_t *n_slots,
                         int32_t *perm, int32_t *slice_ptr);

int vexb_csr_create(int dev, void *stream, size_t nrows, size_t ncols,
                    const void *ptr, int ptr_bytes, const void *col, int col_bytes,
                    const void *val, int val_dtype, int fmt, vexb_spmat **out);
int vexb_spmat_destroy(vexb_spmat *A);
typedef struct {
    size_t  nrows, ncols, nnz;
    int32_t fmt;          /* VEXB_FMT_CSR, VEXB_FMT_HELL, VEXB_FMT_PATTERNS or VEXB_FMT_SELL */
    int32_t val_dtype;
    size_t  ell_width, ell_pitch, csr_tail_nnz;   /* HELL only */
    size_t  n_tiles, tile_nnz;                    /* CSR: tiles, nnz per tile; PATTERNS: unique rows, entries in their table */
    size_t  device_bytes;                         /* bytes of matrix data resident in HBM */
    int32_t ell_col_bytes;                        /* HELL: bytes per ELL slot of the column encoding: 4 = 32-bit columns,
                                                     2 = 16-bit offsets ("spmv.col16"), 0 = no column array, one slot mask
                                                     byte per row ("spmv.ell_diag"; width 0 also reports 0) */
    int32_t ell_classes;                          /* HELL: number of row classes ("spmv.ell_classes": one class byte per row,
                                                     slot masks and values in a table of at most 256 classes); 0 = values
                                                     stored per slot */
    int32_t val_bytes;                            /* bytes per stored value of the per-entry value arrays: 8 (double),
                                                     4 (float, or double values with VEXB_FMT_VALUES_F32); 0 for row-class
                                                     and row-pattern strips, whose tables hold the values */
} vexb_spmat_info;
int vexb_spmat_get_info(const vexb_spmat *A, vexb_spmat_info *info);
/* Copy the HELL arrays back (parity with hybrid_ell.inl:132-193); any pointer may be NULL.  Values come back in the
 * strip's value type: double for VEXB_FMT_VALUES_F32 strips (the rounded values). */
int vexb_spmat_hell_download(const vexb_spmat *A, int32_t *ell_col, void *ell_val,
                             int64_t *csr_ptr, int32_t *csr_col, void *csr_val);
/* y (=|+=) alpha * A x     (csr.inl:188-209: append ? "+=" : "=") */
int vexb_spmv(int dev, void *stream, const vexb_spmat *A, const void *x, void *y, double alpha, int append);

/* ------------------------------------------------------------------------
 * Block sparse strips (one device): B x B blocks as values, B = 2, 3 or 4 --
 * vex::sparse::{csr, ell, matrix}<std::array<std::array<T,B>,B>>, the
 * reference's custom value types (sparse/distributed.hpp:17-21 rhs_of,
 * tests/sparse_matrices.cpp:239-282).  Stored as sliced ELL over block rows
 * (the layout of VEXB_FMT_SELL, "spmv.sell_sigma"), one 32-bit block column
 * per slot and the B*B values of a slot planar, so that a warp's value loads
 * are 32 consecutive elements.
 *   y_i (=|+=) alpha * sum over the blocks j of block row i, in storage order,
 *   of A_j x_col(j); row r of a block is t = a_r0 x_0 + a_r1 x_1 + ... added
 *   left to right, then s_r = s_r + t, every product and sum rounded on its own.
 * create() validates every argument before it touches a device.
 * ---------------------------------------------------------------------- */
typedef struct vexb_bspmat vexb_bspmat;
typedef struct {
    size_t  nrows, ncols, nnzb;      /* block rows, block columns, stored blocks */
    int32_t block, val_dtype;        /* B; VEXB_F64 or VEXB_F32 */
    size_t  n_slices, n_slots;       /* sliced-ELL slices of 32 block rows, slots over all slices (as vexb_csr_sell_layout) */
    size_t  device_bytes;            /* n_slots * (B*B*sizeof(T) + 4) + perm + slice_ptr */
} vexb_bspmat_info;
/* nrows/ncols/ptr/col count BLOCK rows/columns; val: nnzb blocks of B*B values, row-major inside a block;
 * x: ncols*B values, y: nrows*B values (block i = elements [i*B, i*B+B)). */
int vexb_bsr_create(int dev, void *stream, size_t nrows, size_t ncols, int block, const void *ptr, int ptr_bytes,
                    const void *col, int col_bytes, const void *val, int val_dtype, vexb_bspmat **out);
int vexb_bspmat_destroy(vexb_bspmat *A);
int vexb_bspmat_get_info(const vexb_bspmat *A, vexb_bspmat_info *info);
/* y (=|+=) alpha * A x; with no stored block, y = A*x zeroes y and y += A*x leaves it as it is (as vexb_spmv). */
int vexb_bspmv(int dev, void *stream, const vexb_bspmat *A, const void *x, void *y, double alpha, int append);

/* ------------------------------------------------------------------------
 * Complex sparse strips (one device): std::complex<T> values, T = double or
 * float -- vex::sparse::{csr, ell, matrix}<std::complex<T>>, the reference's
 * examples/complex_spmv.cpp (its spmv_ops_impl<std::complex<T>, ...>).
 * Stored as the block strips above with 2 planar components (re, im) per slot
 * instead of B*B.  For each stored entry a + bi of row i, in storage order:
 *   s_re = s_re + (a xr - b xi),   s_im = s_im + (a xi + b xr),
 * every product and sum rounded on its own; y_i (=|+=) alpha * s per
 * component (alpha real).  The same bits as vexb_bspmv on the 2 x 2 blocks
 * [[a, -b], [b, a]].  create() validates every argument before it touches a
 * device.
 * ---------------------------------------------------------------------- */
typedef struct vexb_zspmat vexb_zspmat;
typedef struct {
    size_t  nrows, ncols, nnz;       /* rows, columns, stored complex entries */
    int32_t val_dtype;               /* VEXB_F64 (complex<double>) or VEXB_F32 (complex<float>) */
    size_t  n_slices, n_slots;       /* sliced-ELL slices of 32 rows, slots over all slices (as vexb_csr_sell_layout) */
    size_t  device_bytes;            /* n_slots * (2*sizeof(T) + 4) + perm + slice_ptr */
} vexb_zspmat_info;
/* val: nnz interleaved (re, im) pairs of T, the bytes of std::complex<T>[nnz]; val_dtype names T.
 * x: 2*ncols T and y: 2*nrows T, the bytes of std::complex<T>[]; x must be aligned to 2*sizeof(T). */
int vexb_zsr_create(int dev, void *stream, size_t nrows, size_t ncols, const void *ptr, int ptr_bytes,
                    const void *col, int col_bytes, const void *val, int val_dtype, vexb_zspmat **out);
int vexb_zspmat_destroy(vexb_zspmat *A);
int vexb_zspmat_get_info(const vexb_zspmat *A, vexb_zspmat_info *info);
/* y (=|+=) alpha * A x, alpha real; with no stored entry, y = A*x zeroes y and y += A*x leaves it as it is. */
int vexb_zspmv(int dev, void *stream, const vexb_zspmat *A, const void *x, void *y, double alpha, int append);

/* ------------------------------------------------------------------------
 * Sparse strips of user value types (one device): vex::sparse::{csr, ell,
 * matrix}<V> for a type V the user declares with vex::is_cl_native,
 * vex::type_name_impl, vex::sparse::rhs_of and vex::sparse::spmv_ops_impl
 * (the reference's sparse/spmv_ops.hpp).  The library does not know the
 * components of V: each value is val_bytes opaque bytes, stored as the
 * complex strips above with one component of val_bytes per slot (lane l of
 * slot k in slice s holds value slice_ptr[s] + 32k + l; padding is zero).
 * The product kernel is generated from the snippets of vexb_usr_ops and
 * compiled by NVRTC for sm_90a (--fmad=false) at its first use on a device,
 * then cached.  For each row, in storage order:
 *   decl;  append_product(sum, v, xv) for every stored value v, xv = x[col];
 *   then y_r = sum (append = 0)  or  t = y_r; append(t, sum); y_r = t.
 * There is no alpha: spmv_ops_impl has no hook for scaling or negation.
 * create() validates every argument before it touches a device.
 * ---------------------------------------------------------------------- */
typedef struct vexb_usrmat vexb_usrmat;
typedef struct {
    size_t  nrows, ncols, nnz;       /* rows, columns, stored values */
    int32_t val_bytes;               /* sizeof(V) */
    size_t  n_slices, n_slots;       /* sliced-ELL slices of 32 rows, slots over all slices (as vexb_csr_sell_layout) */
    size_t  device_bytes;            /* n_slots * (val_bytes + 4) + perm + slice_ptr */
} vexb_usrmat_info;
/* The device side of spmv_ops_impl<V, X>.  Snippets use the fixed names sum (the accumulator, declared by decl),
 * v (const V, the stored value), xv (const X, x at its column) and t (X, the old y_r).  The generated source holds
 * static_assert(sizeof(V) == val_bytes && sizeof(X) == rhs_bytes), so a host/device size mismatch fails in NVRTC. */
typedef struct {
    const char *val_type;            /* device type name of V, e.g. "double4" */
    const char *rhs_type;            /* device type name of X, the element of x and y, e.g. "double2" */
    size_t      rhs_bytes;           /* sizeof(X) on the host, 1..64 */
    const char *decl;                /* spmv_ops_impl<V, X>::decl_accum_var(src, "sum") */
    const char *product;             /* spmv_ops_impl<V, X>::append_product(src, "sum", "v", "xv") */
    const char *append;              /* spmv_ops_impl<V, X>::append(src, "t", "sum") */
} vexb_usr_ops;
/* val: nnz values of val_bytes bytes each (val_bytes a multiple of 4 in 4..64), the bytes of V[nnz]. */
int vexb_usr_create(int dev, void *stream, size_t nrows, size_t ncols, const void *ptr, int ptr_bytes,
                    const void *col, int col_bytes, const void *val, int val_bytes, vexb_usrmat **out);
int vexb_usrmat_destroy(vexb_usrmat *A);
int vexb_usrmat_get_info(const vexb_usrmat *A, vexb_usrmat_info *info);
/* y (=|+=) A x with x: ncols X and y: nrows X, both aligned to the natural alignment of an X of rhs_bytes (the largest
 * power of two up to 16 that divides it).  With no stored value, y = A*x zeroes y and y += A*x leaves it as it is.  An
 * NVRTC failure returns VEXB_ERR_INVALID with the compiler's log in vexb_last_error(). */
int vexb_usr_spmv(int dev, void *stream, const vexb_usrmat *A, const vexb_usr_ops *ops, const void *x, void *y, int append);
/* Source of the kernel vexb_usr_spmv generates for these ops (compile != 0: also compiled by NVRTC for sm_90a, no device
 * needed).  *len in: capacity, out: bytes needed. */
int vexb_jit_source_usr(const vexb_usr_ops *ops, int val_bytes, char *buf, size_t *len, int compile);

/* ------------------------------------------------------------------------
 * Compressed CSR for stencil-like matrices: vex::SpMatCCSR
 * (vexcl/spmat/ccsr.hpp:54-86 ctor, :176-201 kernel).  Single device.
 *   y[i] (=|+=) alpha * sum_{j = row[idx[i]] .. row[idx[i]+1]} val[j] * x[i + col[j]]
 * idx: n entries naming one of the m unique rows; row: m+1 offsets; col: SIGNED
 * offsets from the diagonal.  Unlike the reference, create() rejects a matrix
 * whose rows reach outside [0, n).
 * ---------------------------------------------------------------------- */
typedef struct vexb_ccsr vexb_ccsr;
typedef struct {
    size_t  nrows, unique_rows, nnz;
    int32_t idx_bytes;       /* width idx was re-encoded to on the device (1, 2 or 4) */
    int32_t table_in_smem;   /* unique-row table staged in shared memory by the kernel */
    size_t  device_bytes;
} vexb_ccsr_info;
int vexb_ccsr_create(int dev, void *stream, size_t n, size_t m, const void *idx, int idx_bytes,
                     const void *row, int row_bytes, const void *col, int col_bytes,
                     const void *val, int val_dtype, vexb_ccsr **out);
int vexb_ccsr_destroy(vexb_ccsr *A);
int vexb_ccsr_get_info(const vexb_ccsr *A, vexb_ccsr_info *info);
int vexb_ccsr_spmv(int dev, void *stream, const vexb_ccsr *A, const void *x, void *y, double alpha, int append);
/* Source of the matrix-specialised product kernel (tunable "ccsr.jit"; the unique rows become code, compiled by
 * NVRTC at first use -- the counterpart of the reference's generated "<prm>_spmv" function, ccsr.hpp:176-201).
 * Host-only: m unique rows, row[m+1] offsets, col/val entries; idx_bytes = device width of idx (1, 2 or 4).
 * compile != 0 also runs NVRTC for sm_90a (no device needed).  *len in: capacity, out: bytes needed. */
int vexb_ccsr_jit_source(size_t m, const int32_t *row, const int32_t *col, const void *val, int val_dtype,
                         int idx_bytes, char *buf, size_t *len, int compile);

/* ------------------------------------------------------------------------
 * Stencil convolution: vex::stencil<T> (vexcl/stencil.hpp:168-330), one device
 * slice per call:
 *   y[i] (=|+=) alpha * sum_{k<width} s[k] * X(i + k - center)
 * X = the slice x[0..n) extended by `left` (the `center` elements before it)
 * and `right` (the width-1-center elements after it); a NULL side clamps to the
 * slice's first / last element (the ends of the whole vector).  s, x, left,
 * right, y are device pointers of `dtype` (VEXB_F64 or VEXB_F32).
 * vexb_copy_peer moves halo pieces between devices (replaces the D2H/H2D
 * staging of stencil_base::exchange_halos, stencil.hpp:86-150).
 * ---------------------------------------------------------------------- */
int vexb_stencil_apply(int dev, void *stream, int dtype, const void *s, int width, int center,
                       const void *x, size_t n, const void *left, const void *right,
                       void *y, double alpha, int append);
int vexb_copy_peer(int dst_dev, void *dst, int src_dev, const void *src, size_t bytes, void *stream);
/* User-defined stencil operators: vex::StencilOperator / VEX_STENCIL_OPERATOR (stencil.hpp:510-680).
 *   y[i] (=|+=) alpha * f(X),  X[k] = the element k places from i (k in [-center, width-1-center]); `body` is the C
 * source of f with X a pointer into the staged window, e.g. "return sin(X[1] - X[0]) + sin(X[0] - X[-1]);".
 * register() is host-only and returns the same id for the same definition; the kernel is compiled by NVRTC at the first
 * apply() on a device (needs libnvrtc; there is no pre-compiled alternative).  source() returns the generated kernel
 * (compile != 0: also runs NVRTC for sm_90a, no device needed).  Run on the GPU by tests/cpp/test_stencil.cpp. */
int vexb_stencil_operator_register(int dtype, int width, int center, const char *body, int *id);
int vexb_stencil_operator_source(int id, char *buf, size_t *len, int compile);
int vexb_stencil_operator_apply(int dev, void *stream, int id, const void *x, size_t n, const void *left,
                                const void *right, void *y, double alpha, int append);

/* ------------------------------------------------------------------------
 * Distributed SpMat part: the slice of a vex::SpMat owned by one device
 * (spmat.hpp:71-106 ctor body for one d, :120-185 apply).
 * `col` holds GLOBAL column ids for the strip's rows, indexed by ptr values
 * relative to ptr[0].
 * ---------------------------------------------------------------------- */
typedef struct vexb_dspmat vexb_dspmat;
int vexb_dspmat_create(int dev, void *stream, int part, const vexb_halo_plan *plan,
                       size_t nrows, const void *ptr, int ptr_bytes, const void *col, int col_bytes,
                       const void *val, int val_dtype, int fmt, vexb_dspmat **out);
int vexb_dspmat_destroy(vexb_dspmat *A);
typedef struct {
    size_t nrows, ncols_local, n_ghost, n_send, loc_nnz, rem_nnz;
    vexb_spmat_info loc, rem;
} vexb_dspmat_info;
int vexb_dspmat_get_info(const vexb_dspmat *A, vexb_dspmat_info *info);
/* Split tables back on the host for parity with csr.inl:70-112 (any pointer may be NULL); VEXB_FMT_VALUES_F32 parts give
 * the rounded values, as double. */
int vexb_dspmat_download_split(const vexb_dspmat *A, int64_t *loc_ptr, int64_t *loc_col, void *loc_val,
                               int64_t *rem_ptr, int64_t *rem_col, void *rem_val);
/* The part's strip for use as a VEXB_TERM_SPMV terminal: set when the part has no ghost columns and its rows are
 * stored plainly in CSR or hybrid ELL (then row i of the strip is element i of the part's slice); NULL otherwise. */
int vexb_dspmat_inline_strip(const vexb_dspmat *A, const vexb_spmat **strip);
/* The part's strip for use as a VEXB_TERM_SPMV terminal of an ASSIGNMENT (vexb_eval): set when the part has no ghost
 * columns and its rows are stored plainly in sliced ELL with values of the vector type, and the tunables
 * "spmv.sell_inline" (default 1) and "spmv.no_inline" (default 0) allow it; NULL otherwise.  The generated kernel then
 * sweeps in the strip's storage order -- one thread per stored lane, every operand and the target at that lane's row --
 * so the column and value loads stay coalesced as in the plain product.  One distinct sliced-ELL strip per expression,
 * any number of times (`A*x + A*z`); a second one is VEXB_ERR_UNSUPPORTED.  vexb_eval_multi and the reductions
 * (vexb_reduce_all, vexb_reduce_multi) do not take such strips. */
int vexb_dspmat_sweep_strip(const vexb_dspmat *A, const vexb_spmat **strip);
void *vexb_dspmat_send_buffer(const vexb_dspmat *A);  /* device, n_send values  */
void *vexb_dspmat_ghost_buffer(const vexb_dspmat *A); /* device, n_ghost values */
/* Steps of SpMat::apply, all asynchronous on `stream`: */
int vexb_dspmat_pack(const vexb_dspmat *A, void *stream, const void *x);                       /* spmat.hpp:127-135 */
int vexb_dspmat_mul_local(const vexb_dspmat *A, void *stream, const void *x, void *y, double alpha, int append); /* :142-146 */
int vexb_dspmat_mul_remote(const vexb_dspmat *A, void *stream, void *y, double alpha);         /* :178-183 */
/* Halo exchange for the local parts (grouped ncclSend/ncclRecv): send buffers -> peers' ghost buffers.
 * Replaces spmat.hpp:149-176. */
int vexb_halo_exchange(int nlocal, vexb_comm *const *comms, vexb_dspmat *const *parts, void *const *streams);
/* Peer-memory halo (csrc/distapply.cu): when every part is connected, vexb_dspmat_apply is ONE kernel per GPU -- it
 * stores the x values its neighbours need straight into their ghost buffers over NVLink, multiplies the interior rows,
 * waits (in the kernel) for its own ghosts and finishes the boundary rows; no NCCL call, no copy, no extra launch, CUDA-
 * graph replayable.  Replaces spmat.hpp:127-183 in one launch.  Up to 16 parts on distinct devices.
 *   one process per GPU : vexb_dspmat_halo_handle (64-byte CUDA IPC handle of this part's ghost box), all-gather the
 *                         handles in part order, vexb_dspmat_halo_connect;
 *   one process, n GPUs : vexb_dspmat_halo_connect_local (peer access).
 * Every part of the matrix must then call apply the same number of times (as with NCCL).  A neighbour that never
 * arrives makes the kernel give up after ~20 s, store NaN in the rows it could not finish and raise vexb_peer_fault. */
int vexb_dspmat_halo_handle(vexb_dspmat *A, void *handle64);
int vexb_dspmat_halo_connect(vexb_dspmat *A, const void *handles /* nparts * 64 bytes, part order */);
int vexb_dspmat_halo_connect_local(int nlocal, vexb_dspmat *const *parts);
int vexb_dspmat_halo_connected(const vexb_dspmat *A, int *connected);
int vexb_dspmat_halo_disconnect(vexb_dspmat *A);   /* back to NCCL / copies (e.g. when another rank failed to connect) */
/* Whole apply for the local parts: pack -> (side stream: exchange) || mul_local -> mul_remote.
 * x[k], y[k] are the device slices of part k.  comms may be NULL when there are no ghosts. */
int vexb_dspmat_apply(int nlocal, vexb_comm *const *comms, vexb_dspmat *const *parts, void *const *streams,
                      const void *const *x, void *const *y, double alpha, int append);

/* Several right-hand sides in one pass over the matrix: vex::SpMat * vex::multivector<T,N> (multivector.hpp;
 * the reference multiplies component by component, operations.hpp:876-880).  Hybrid-ELL and sliced-ELL strips take groups
 * of up to 4 vectors per launch (columns and values loaded once, same per-component bits as vexb_spmv); anything else falls back to
 * one product per vector.  vexb_dspmat_apply_multi: x[k * nrhs + r] / y[k * nrhs + r] = slice of component r on part k;
 * parts with a halo multiply component by component. */
int vexb_spmv_multi(int dev, void *stream, const vexb_spmat *A, int nrhs, const void *const *x, void *const *y,
                    double alpha, int append);
int vexb_dspmat_apply_multi(int nlocal, vexb_comm *const *comms, vexb_dspmat *const *parts, void *const *streams,
                            int nrhs, const void *const *x, void *const *y, double alpha, int append);

/* The product and a dot product with its result without re-reading the vectors: y (=|+=) alpha*A*x, and
 * d_result[k][0] = sum over all parts of dot_with . y (same bits on every GPU).  The product kernel leaves one partial
 * per block; a one-block second launch folds them and combines across the peer group.  With dot_with = x this is q = A*p, (p, q) of a CG iteration.  Needs the peer-memory halo on every part
 * (or a single part) and a hybrid-ELL or sliced-ELL (VEXB_FMT_SELL) interior strip with at least one entry and values
 * of the vector type; returns VEXB_ERR_UNSUPPORTED otherwise (CSR or row-pattern interiors, VEXB_FMT_VALUES_F32,
 * dspmat.no_peer_halo, dspmat.no_fused_dot: compose apply + reduce). */
int vexb_dspmat_apply_dot(int nlocal, vexb_dspmat *const *parts, void *const *streams, const void *const *x,
                          void *const *y, double alpha, int append, const void *const *dot_with,
                          void *const *d_result, vexb_peer *const *peers);

/* The vector half of a conjugate-gradient iteration (BASELINE configs[4]) in two sweeps, scalars device-resident:
 *   vexb_cg_update_r  : alpha = *d_rho / *d_pq;  r -= alpha q;  *d_rho_new = (r, r)   (folded like vexb_reduce, combined
 *                       over `peer` in the same kernel; peer == NULL: this slice only)             24 bytes per row
 *   vexb_cg_update_xp : alpha as above, beta = *d_rho_new / *d_rho;  x += alpha p;  p = r + beta p  40 bytes per row
 * Same unfused per-element arithmetic as the vexb_eval / vexb_reduce composition (viennacl.hpp:36-64 composes CG from
 * those); d_workspace as for vexb_reduce.  Vectors must be 32-byte aligned (vexb_malloc's are). */
int vexb_cg_update_r(int dev, void *stream, int dtype, size_t n, void *r, const void *q,
                     const void *d_rho, const void *d_pq, void *d_rho_new, void *d_workspace, vexb_peer *peer);
int vexb_cg_update_xp(int dev, void *stream, int dtype, size_t n, void *x, void *p, const void *r,
                      const void *d_rho, const void *d_pq, const void *d_rho_new);

/* ------------------------------------------------------------------------
 * Sort (vex::sort, vex::sort_by_key with vex::less / less_equal / greater / greater_equal, vexcl/sort.hpp).
 * vexb_sort sorts n keys of `key_dtype` in place on one device slice, ascending (descending = 0) or descending, and
 * moves the n values of `val_dtype` with them (vals = NULL and val_dtype = -1: keys only).  Stable in both directions.
 * Floating keys: -0.0 equals +0.0, every NaN equals every other NaN and is greater than +inf; keys keep their bits.
 * Asynchronous on `stream`; n < 2 launches nothing.  At most 2^31 - 1 elements.  d_workspace: device memory of at
 * least vexb_sort_workspace_bytes(n, key_dtype, val_dtype) bytes (0 for n < 2, when it may be NULL).  Arguments are
 * checked before anything touches the device (VEXB_ERR_INVALID).  Shape of the launches: csrc/sort.cu.
 * vexb_sort_merge (host only) merges nparts sorted host runs, run p at [part[p] - part[0], part[p+1] - part[0]) of
 * keys (and vals), into keys_out (and vals_out) in the same order, stably: equal keys keep their run order, then their
 * order within the run.
 * ---------------------------------------------------------------------- */
int vexb_sort_workspace_bytes(size_t n, int key_dtype, int val_dtype, size_t *bytes);
int vexb_sort(int dev, void *stream, void *keys, int key_dtype, void *vals, int val_dtype, size_t n, int descending,
              void *d_workspace, size_t workspace_bytes);
int vexb_sort_merge(int nparts, const size_t *part, const void *keys, int key_dtype, const void *vals, int val_dtype,
                    int descending, void *keys_out, void *vals_out);

/* ------------------------------------------------------------------------
 * Scans (vex::inclusive_scan, vex::exclusive_scan, vexcl/scan.hpp), scans by key (vex::inclusive_scan_by_key,
 * vex::exclusive_scan_by_key, vexcl/scan_by_key.hpp) and vex::reduce_by_key (vexcl/reduce_by_key.hpp) of one device
 * slice, with `+` on the values and `==` on the keys.  Integer sums wrap; every float add is rounded on its own, in an
 * order that depends on n only (csrc/scan.cu).  A run is a maximal range of keys equal under ==: -0.0 and +0.0 share
 * one, every NaN key is a run of its own.
 * vexb_scan: out[i] = in[0] + ... + in[i] (inclusive; h_init is not read) or, exclusive, out[0] = *h_init with its own
 * bits and out[i] = *h_init + in[0] + ... + in[i-1].  in == out scans in place.
 * vexb_scan_by_key: the same within every run of keys; an exclusive scan starts every run at *h_init.  ivals == ovals
 * scans in place; keys must not be ovals.
 * vexb_reduce_by_key_count runs the first two of the three launches and returns the number of runs in *nruns (one
 * device-to-host read; it waits for the stream); vexb_reduce_by_key_write, with the same arguments and workspace, then
 * writes the last key of run j to okeys[j] and the sum of its values to ovals[j].  The outputs must not alias the
 * inputs or each other.
 * h_init: one element of the value dtype on the host; NULL reads as zero.  Asynchronous on `stream` (apart from
 * vexb_reduce_by_key_count); n = 0 launches nothing.  At most 2^31 - 1 elements.  d_workspace: device memory of at least
 * vexb_scan_workspace_bytes(n, val_dtype) bytes (0 for n = 0, when it may be NULL).  Arguments are checked before
 * anything touches the device (VEXB_ERR_INVALID).
 * ---------------------------------------------------------------------- */
int vexb_scan_workspace_bytes(size_t n, int val_dtype, size_t *bytes);
int vexb_scan(int dev, void *stream, const void *in, void *out, int dtype, size_t n, int exclusive, const void *h_init,
              void *d_workspace, size_t workspace_bytes);
int vexb_scan_by_key(int dev, void *stream, const void *keys, int key_dtype, const void *ivals, void *ovals, int val_dtype,
                     size_t n, int exclusive, const void *h_init, void *d_workspace, size_t workspace_bytes);
int vexb_reduce_by_key_count(int dev, void *stream, const void *ikeys, int key_dtype, const void *ivals, int val_dtype,
                             size_t n, void *d_workspace, size_t workspace_bytes, size_t *nruns);
int vexb_reduce_by_key_write(int dev, void *stream, const void *ikeys, int key_dtype, const void *ivals, int val_dtype,
                             size_t n, void *okeys, void *ovals, void *d_workspace, size_t workspace_bytes);

#ifdef __cplusplus
}
#endif
#endif /* VEXB200_H */
