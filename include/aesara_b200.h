/* aesara_b200.h — C ABI of libaesara_b200.so, the H100 (sm_90a) device runtime
 * behind Aesara's Linker/Op plugin surface.
 *
 * Conventions (they mirror the reference's native thunk ABI,
 * aesara/link/c/basic.py:1668-1709 and lazylinker_c.c:501-520: "0 = success,
 * non-zero = failure id"):
 *   - every function returns 0 on success, a non-zero ab_status otherwise;
 *     ab_last_error() returns the message of the last failure on this thread;
 *   - no exceptions cross the ABI, no torch / Python types in any signature;
 *   - the caller owns all descriptors and device buffers it passes in; the
 *     library owns only what it hands out as opaque handles (ab_module);
 *   - every launch is asynchronous on the caller-supplied stream (a CUDA
 *     stream handle cast to void*, NULL = default stream);
 *   - strides are in ELEMENTS (not bytes); a broadcast dimension has stride 0
 *     (the run-time broadcast rule of aesara/tensor/elemwise_cgen.py:72-76).
 */
#ifndef AESARA_B200_H
#define AESARA_B200_H

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define AB_MAX_DIMS 8      /* after collapsing; callers may pass up to 32 raw dims */
#define AB_MAX_RAW_DIMS 32
#define AB_MAX_OPERANDS 40 /* inputs + outputs of one fused Elemwise */

typedef enum {
  AB_OK = 0,
  AB_ERR_CUDA = 1,        /* a CUDA runtime/driver call failed */
  AB_ERR_NVRTC = 2,       /* JIT compilation failed (log in ab_last_error) */
  AB_ERR_INVALID = 3,     /* bad argument (maps to ValueError/TypeError) */
  AB_ERR_SHAPE = 4,       /* shape mismatch (maps to the reference's ValueError texts) */
  AB_ERR_UNSUPPORTED = 5, /* valid request the device path does not implement */
  AB_ERR_NO_DEVICE = 6,   /* no usable GPU */
  AB_ERR_LINALG = 7       /* matrix not positive definite / singular (maps to LinAlgError) */
} ab_status;

/* dtype codes — the dtype set of aesara/tensor/type.py:39-54 minus complex */
typedef enum {
  AB_BOOL = 0, AB_I8 = 1, AB_I16 = 2, AB_I32 = 3, AB_I64 = 4,
  AB_U8 = 5, AB_U16 = 6, AB_U32 = 7, AB_U64 = 8,
  AB_F16 = 9, AB_F32 = 10, AB_F64 = 11, AB_BF16 = 12
} ab_dtype;

typedef struct ab_module ab_module; /* a loaded JIT module (one fused Composite / one reduction) */

typedef struct {
  int sm_count;
  int cc_major, cc_minor;
  size_t total_mem;
  size_t l2_bytes;
  int max_smem_per_block_optin;
  char name[128];
} ab_device_info;

/* ---- runtime ----------------------------------------------------------- */
/* Select the device and create the context.  Idempotent.  Replaces nothing in
 * the reference (it has no device); called once from B200Linker.make_all. */
int ab_init(int device_ordinal);
int ab_get_device_info(int device_ordinal, ab_device_info* out);
const char* ab_last_error(void);
const char* ab_version(void);
int ab_stream_synchronize(void* stream);
int ab_device_synchronize(void);

/* Stream-ordered device memory for hosts that do not bring their own
 * allocator (the Python host uses torch's caching allocator instead). */
int ab_malloc(void** dptr, size_t bytes, void* stream);
int ab_free(void* dptr, void* stream);
int ab_memcpy_h2d(void* dst, const void* src, size_t bytes, void* stream);
int ab_memcpy_d2h(void* dst, const void* src, size_t bytes, void* stream);
int ab_memset(void* dst, int value, size_t bytes, void* stream);

/* CUDA-event timing on the launching stream (replaces the call_times/call_counts
 * host timers of aesara/link/vm.py:389-406 — host timers are meaningless for
 * asynchronous launches). */
int ab_event_create(void** ev);
int ab_event_record(void* ev, void* stream);
int ab_event_elapsed_ms(void* start, void* stop, float* ms);
int ab_event_destroy(void* ev);

/* ---- JIT: generated kernel per fused Elemwise{Composite} / CAReduce ------ */
/* Compile CUDA C++ to an sm_90a cubin with NVRTC.  Needs no GPU.  Replaces
 * GCC_compiler.compile_str (aesara/link/c/cmodule.py:2482).  *cubin is
 * malloc()ed; release with ab_buffer_free. */
int ab_nvrtc_compile(const char* src, const char* name, const char* const* extra_opts,
                     int n_extra_opts, void** cubin, size_t* cubin_size);
/* Version of the NVRTC that ab_nvrtc_compile uses: the libnvrtc.so.12 the process loaded
 * first (a process that has imported torch uses torch's bundled one).  Part of the key of
 * the cubin cache, since two NVRTC versions make different code from the same source. */
int ab_nvrtc_version(int* major, int* minor);
void ab_buffer_free(void* p);
/* Load a cubin on the current device (replaces dlimport of the compiled module,
 * aesara/link/c/cmodule.py:ModuleCache). */
int ab_module_load(const void* cubin, size_t cubin_size, ab_module** out);
int ab_module_unload(ab_module* m);
/* Launch a kernel of a loaded module by name with a 1-D grid (generated kernels whose
 * parameter list is not one of the fixed Elemwise / CAReduce skeletons, e.g. the fused
 * Gemv -> Elemwise -> Gemv^T row kernel).  args[i] points at the i-th kernel parameter. */
int ab_kernel_launch(ab_module* m, const char* name, unsigned grid_x, unsigned block_x,
                     size_t smem_bytes, void** args, void* stream);

/* ---- Elemwise (aesara/tensor/elemwise.py:304, C thunk _c_all :835-1168) ---
 * Launch the fused scalar expression compiled in `m` over an ndim-dimensional
 * index space.  operand k (inputs first, then outputs) is ptrs[k] with
 * strides[k*ndim + d] (elements; 0 = broadcast).  The launcher squeezes and
 * merges dimensions, then picks the vectorised flat / row / generic kernel.
 * In-place outputs simply alias an input pointer.  `vec`/`unroll` are the
 * AB_VEC / AB_UNROLL the module was generated with. */
int ab_elemwise_launch(ab_module* m, int n_in, int n_out, int ndim, const int64_t* shape,
                       void* const* ptrs, const int64_t* strides, const int32_t* itemsizes,
                       int vec, int unroll, void* stream);
/* Number of ab_elemwise_launch calls since load that ran kernel flavour `which`:
 * 0 flat_vec, 1 flat, 2 rows_vec, 3 rows, 4 nd, 5 tile (0 for any other value). */
uint64_t ab_elemwise_path_count(int which);

/* ---- CAReduce (aesara/tensor/elemwise.py:1221, C loop elemwise_cgen.py:502) -
 * Reduce `in` over the axes flagged in reduce_mask into a C-contiguous `out`
 * of the remaining dims.  The module fixes (scalar op, in/acc/out dtype).
 * `workspace` must hold ab_careduce_workspace_bytes() bytes. */
int ab_careduce_workspace_bytes(int ndim, const int64_t* shape, const int32_t* reduce_mask,
                                int acc_itemsize, size_t* bytes);
int ab_careduce_launch(ab_module* m, int ndim, const int64_t* shape, const int64_t* in_strides,
                       const int32_t* reduce_mask, const void* in, void* out, void* workspace,
                       size_t workspace_bytes, int in_itemsize, int acc_itemsize,
                       int out_itemsize, void* stream);

/* ---- BLAS family ------------------------------------------------------------
 * Gemv  (aesara/tensor/blas.py:231, blas_c.py:369-577):  y <- beta*y + alpha*A@x
 *   A is [m,n] with element strides (a_rs, a_cs); when beta == 0, y is not read.
 * Ger   (aesara/tensor/blas.py:330, blas_c.py:45-357):    A <- A + alpha*x*y^T
 * Gemm / Dot22 (aesara/tensor/blas.py:872 / :1659, C template :518-869):
 *   C[m,n] <- beta*C + alpha * A[m,k] @ B[k,n]; arbitrary 2-D element strides
 *   (the eight stride cases of blas.py:765-776 plus copies for the rest);
 *   wgmma tensor-core tiles fed by TMA.  `precision`:
 *     0 = fp32-faithful (3xTF32 split, rtol 1e-5 vs sgemm),
 *     1 = single TF32 pass, 2 = BF16 operands / FP32 accumulate (policy mode).
 *   dtype is AB_F32 or AB_F64 (the only dtypes the reference Gemm accepts,
 *   blas.py:613-629); f64 runs on the FP64 pipe. */
int ab_gemv(int dtype, int64_t m, int64_t n, double alpha, const void* A, int64_t a_rs,
            int64_t a_cs, const void* x, int64_t x_s, double beta, void* y, int64_t y_s,
            void* workspace, size_t workspace_bytes, void* stream);
int ab_gemv_workspace_bytes(int dtype, int64_t m, int64_t n, int64_t a_rs, int64_t a_cs,
                            size_t* bytes);
int ab_ger(int dtype, int64_t m, int64_t n, double alpha, const void* x, int64_t x_s,
           const void* y, int64_t y_s, void* A, int64_t a_rs, int64_t a_cs, void* stream);
int ab_gemm(int dtype, int precision, int64_t m, int64_t n, int64_t k, double alpha,
            const void* A, int64_t a_rs, int64_t a_cs, const void* B, int64_t b_rs,
            int64_t b_cs, double beta, void* C, int64_t c_rs, int64_t c_cs, void* workspace,
            size_t workspace_bytes, void* stream);
int ab_gemm_workspace_bytes(int dtype, int precision, int64_t m, int64_t n, int64_t k,
                            int64_t a_rs, int64_t a_cs, int64_t b_rs, int64_t b_cs,
                            size_t* bytes);

/* Packed tensor-core operands.  ab_gemm converts its operands on every call
 * (hi/lo TF32 split, bf16, or a K-/MN-major copy).  A caller that multiplies the
 * same matrix several times (X and X^T, h and h^T in an MLP backward pass) packs
 * it once: logical operand [rows, k] (rows = M for A, N for B; element strides
 * s_r, s_k) -> ab_gemm_operand, then ab_gemm_packed.  A transposed view of the
 * same memory yields the same planes with mn_major flipped, so one pack serves
 * both products (the operand is handed to wgmma as MN-major). */
typedef struct {
  const void* plane0;   /* hi / only plane */
  const void* plane1;   /* lo plane of the 3xTF32 split, else NULL */
  int64_t rows, k, pitch;
  int32_t mn_major;     /* 0: planes are [rows,pitch] K-contiguous; 1: [k,pitch] rows-contiguous */
  int32_t precision;
} ab_gemm_operand;
int ab_gemm_pack_bytes(int precision, int64_t rows, int64_t k, int64_t s_r, int64_t s_k,
                       size_t* bytes);
int ab_gemm_pack(int precision, const void* src, int64_t rows, int64_t k, int64_t s_r,
                 int64_t s_k, void* dst, size_t dst_bytes, ab_gemm_operand* out, void* stream);
/* The same with the planes forced K-major whatever the strides (a row-contiguous view, i.e.
 * the transpose of a row-major matrix, is turned while it is packed): for small matrices
 * (weights) that a product reads with the contraction along their rows. */
int ab_gemm_pack_kmajor_bytes(int precision, int64_t rows, int64_t k, int64_t s_r, int64_t s_k,
                              size_t* bytes);
int ab_gemm_pack_kmajor(int precision, const void* src, int64_t rows, int64_t k, int64_t s_r,
                        int64_t s_k, void* dst, size_t dst_bytes, ab_gemm_operand* out,
                        void* stream);
/* C <- beta*Cin + alpha*A@B.  Cin == NULL means in place (Cin = C); a separate Cin is
 * the Gemm{no_inplace} case (blas.py:1065-1093) without the copy of z.  `workspace` is
 * optional scratch for split-K (ab_gemm_packed_workspace_bytes; 0 bytes = not wanted):
 * problems with few output tiles and a long K are cut along K so that every SM has work,
 * and the partial products are summed into C by a second kernel. */
int ab_gemm_packed(int precision, int64_t m, int64_t n, int64_t k, double alpha,
                   const ab_gemm_operand* A, const ab_gemm_operand* B, double beta,
                   const void* Cin, int64_t cin_rs, int64_t cin_cs, void* C, int64_t c_rs,
                   int64_t c_cs, void* workspace, size_t workspace_bytes, void* stream);
int ab_gemm_packed_workspace_bytes(int precision, int64_t m, int64_t n, int64_t k, size_t* bytes);

/* Gemm/Dot22 followed by the Elemwise (and Sum) nodes that consume it, in one kernel:
 * `module` is the NVRTC build of the tensor-core GEMM kernels with the scalar program of those nodes
 * as the epilogue (aesara_b200/codegen/gemm_epilogue.py).  Per element the program maps
 * v = beta*Cin + alpha*A@B and the operands e_i = ptr[i][row*rs[i] + col*cs[i]] (stride 0
 * broadcasts) to n_outputs values.  Value 0 is stored to C (C may be NULL: not stored),
 * value k >= 1 to out_f32[k] ([m, out_rs[k]] rows, unit column stride; NULL: not stored).
 * `shadow_bf16[k]` (optional) receives the bf16 copy of value k as a [m, shadow_pitch[k]]
 * plane: the packed operand of the next product (replaces ab_gemm_pack for that matrix).
 * `shadow_t_bf16` (optional; modules generated with a transposed-plane value) receives the
 * TRANSPOSED bf16 copy of that value, an [n, shadow_t_pitch] plane (pitch >= m, % 8 == 0): the
 * K-major operand of a product that contracts over the rows of the value (X.T @ value,
 * value.T @ Y -- the weight gradients of tensor/blas.py:1650 Dot22 in a backward pass).
 * Reductions the module was generated with (tensor/elemwise.py:1221 CAReduce{add}, float64
 * accumulators like the reference): column sums of one value as partials per 32-row block,
 * colsum_ws[row_blocks][n]; the sum of all elements of one value as partials
 * fullsum_ws[row_blocks][fullsum_cols] (ab_gemm_fused_layout gives the extents).  The
 * caller adds the partials (a deterministic second pass). */
typedef struct {
  ab_module* module;
  int32_t n_operands;
  const void* ptr[4];
  int64_t rs[4], cs[4];
  int32_t n_outputs;
  void* out_f32[3];
  int64_t out_rs[3];
  void* shadow_bf16[3];
  int64_t shadow_pitch[3];
  void* colsum_ws;
  void* fullsum_ws;
  void* shadow_t_bf16;
  int64_t shadow_t_pitch;
} ab_gemm_epilogue;
int ab_gemm_fused_layout(int64_t m, int64_t n, int64_t* row_blocks, int64_t* fullsum_cols);
int ab_gemm_packed_fused(int precision, int64_t m, int64_t n, int64_t k, double alpha,
                         const ab_gemm_operand* A, const ab_gemm_operand* B, double beta,
                         const void* Cin, int64_t cin_rs, int64_t cin_cs, void* C, int64_t c_rs,
                         int64_t c_cs, const ab_gemm_epilogue* ep, void* stream);
int ab_gemm_tensorcore_eligible(int64_t m, int64_t n, int64_t k);
/* How many clusters of `ctas` CTAs of the ahead-of-time tensor-core GEMM kernel of `precision`
 * can be resident at once on the current device (cudaOccupancyMaxActiveClusters, full shared
 * memory): GPCs whose SM count is not a multiple of `ctas` leave SMs idle. */
int ab_gemm_max_clusters(int precision, int ctas, int* clusters);

/* ---- row ops (SURVEY §8f N1) ---------------------------------------------------
 * The operand is a C-contiguous [outer, r, inner] view; the op runs along r.
 * ab_softmax mode 0: Softmax (aesara/tensor/special.py:239), 1: LogSoftmax (:508),
 * 2: SoftmaxGrad (:13; in = dy, in2 = sm).  float32 / float64.
 * ab_max_and_argmax (aesara/tensor/math.py:126): per row of [outer, r] the maximum
 * (out_max, may be NULL) and the int64 index of its first occurrence (out_argmax, may
 * be NULL); NaN wins, like np.max / np.argmax. */
int ab_softmax(int dtype, int mode, int64_t outer, int64_t r, int64_t inner, const void* in,
               const void* in2, void* out, void* stream);
int ab_max_and_argmax(int dtype, int64_t outer, int64_t r, const void* in, void* out_max,
                      void* out_argmax, void* stream);

/* ---- integer-array indexing (SURVEY §8f N3) ---------------------------------------
 * ab_take_rows: AdvancedSubtensor1 (aesara/tensor/subtensor.py:1925): out[r,:] = x[idx[r],:]
 *   over x viewed as [n_rows, inner] (inner contiguous, rows x_row_stride elements apart);
 *   negative indices wrap.  ab_scatter_rows: AdvancedIncSubtensor1 (:2128) and
 *   AdvancedIncSubtensor (:2700), by mode:
 *     AB_SCATTER_ADD       x[idx[r],:] += y[r,:] for every r (duplicates accumulate, np.add.at);
 *     AB_SCATTER_SET       x[d,:] = y[r,:] with r the LAST occurrence of d in idx (x[idx] = y);
 *     AB_SCATTER_ADD_LAST  x[d,:] += y[r,:], r the last occurrence (out[idx] += y, the
 *                          reference's ignore_duplicates).
 *   The last-occurrence modes need ab_scatter_rows_workspace_bytes (an int64 per row) of
 *   workspace; AB_SCATTER_ADD needs none.
 * check != 0: synchronise and return AB_ERR_SHAPE if an index was out of range
 * (the reference's IndexError). */
typedef enum { AB_SCATTER_ADD = 0, AB_SCATTER_SET = 1, AB_SCATTER_ADD_LAST = 2 } ab_scatter_mode;
int ab_take_rows(int itemsize, int idx_dtype, const void* x, int64_t x_row_stride, int64_t n_rows,
                 int64_t inner, const void* idx, int64_t idx_stride, int64_t n_idx, void* out,
                 int check, void* stream);
int ab_scatter_rows_workspace_bytes(int mode, int64_t n_rows, size_t* bytes);
int ab_scatter_rows(int dtype, int idx_dtype, int mode, void* x, int64_t x_row_stride,
                    int64_t n_rows, int64_t inner, const void* idx, int64_t idx_stride,
                    int64_t n_idx, const void* y, int64_t y_row_stride, int64_t y_col_stride,
                    void* workspace, size_t workspace_bytes, int check, void* stream);

/* AdvancedSubtensor / AdvancedIncSubtensor with one integer vector per leading dimension
 * (x[i, j], aesara/tensor/subtensor.py:2577/2727): ab_ravel_index folds the k int64 index
 * vectors (element strides idx_stride, 0 broadcasts a length-1 vector) over dims[0..k) into
 * one flat int64 row index, wrapping negative values; the gather / scatter is then
 * ab_take_rows / ab_scatter_rows over x viewed as [prod(dims), inner]. */
int ab_ravel_index(int k, const void* const* idx, const int64_t* idx_stride, const int64_t* dims,
                   int64_t n, void* out, int check, void* stream);
/* ARange (aesara/tensor/basic.py:3011): out[i] = start + i*step in dtype (floats use
 * start/step, integers start_i/step_i). */
int ab_arange(int dtype, double start, double step, int64_t start_i, int64_t step_i, int64_t n,
              void* out, void* stream);

/* CumOp (aesara/tensor/extra_ops.py:253): running sum (mul = 0) / product (mul = 1) along the
 * middle axis of x viewed as C-contiguous [outer, len, inner]; out has the dtype of x. */
int ab_cumulative(int dtype, int mul, const void* x, void* out, int64_t outer, int64_t len,
                  int64_t inner, void* stream);

/* ---- random draws (aesara/tensor/random/basic.py UniformRV, NormalRV, BernoulliRV) ----------
 * Fill the C-contiguous `out` of `shape` with draws of the Philox4x32-10 stream under `key`
 * (the stream is defined in csrc/ab_random.cu and README "Random draws"):
 *   AB_RNG_UNIFORM   params (low, high),  dtype AB_F32 / AB_F64, parameters of that dtype;
 *   AB_RNG_NORMAL    params (loc, scale), dtype AB_F32 / AB_F64, parameters of that dtype;
 *   AB_RNG_BERNOULLI params (p),          dtype AB_I64, p float64.
 * params[k] is read at element strides param_strides[k*ndim + d] (0 = broadcast).
 * check != 0: synchronise and return AB_ERR_INVALID if a parameter was invalid (scale < 0,
 * p outside [0, 1] or NaN: the reference's ValueError); with check == 0 nothing is checked. */
typedef enum { AB_RNG_UNIFORM = 0, AB_RNG_NORMAL = 1, AB_RNG_BERNOULLI = 2 } ab_rng_dist;
int ab_random(int dist, int dtype, uint64_t key, int ndim, const int64_t* shape, int n_params,
              const void* const* params, const int64_t* param_strides, void* out, int check,
              void* stream);

/* ---- dense linear algebra (aesara/tensor/slinalg.py Cholesky, SolveTriangular, CholeskySolve,
 * Solve(assume_a="pos")); float32 (AB_F32) and float64 (AB_F64).  Blocked in csrc/ab_linalg.cu,
 * with the rank-k updates on the GEMMs (float32: always the 3xTF32 product).
 * Errors go to a device status word the caller owns (8 bytes): ab_linalg_status_reset before the
 * calls of one node, ab_linalg_status_check after them (one synchronisation) returns
 *   AB_ERR_INVALID  a non-finite value in a checked operand (the reference's ValueError),
 *   AB_ERR_LINALG   a pivot that is not > 0 (not positive definite, NaN pivots included) or a
 *                   zero on the diagonal of a non-unit triangular system (LinAlgError),
 *   AB_ERR_UNSUPPORTED while the stream is being captured into a CUDA graph (nothing is read).
 * The message names the flat index of the non-finite value, the leading minor or the diagonal.
 * ab_cholesky: out (C-contiguous n x n) <- the lower (lower != 0) or upper factor of the symmetric
 *   matrix built from that triangle of a (element strides a_rs, a_cs; the other triangle is not
 *   read, and is exactly 0 in out).  nan_on_error: a failed factorisation leaves out all NaN.
 *   check_finite: scan all of a (both triangles) first.
 * ab_trsm: x (C-contiguous n x nrhs; a vector when nrhs == 1) <- op(A)^-1 b, op(A) = A (trans 0)
 *   or A^T (trans != 0), A triangular by `lower`, unit_diagonal: its diagonal is taken as 1 and not
 *   read.  b may be x itself (in place).  check_finite scans a and b; check_singular tests the
 *   diagonal of a for zeros.
 * Workspace: ab_*_workspace_bytes (the tensor-core GEMM's operand planes; 0 for float64).
 * ab_linalg_update_count(tc): rank-k updates run so far on the tensor cores (tc != 0) or on the
 *   CUDA-core kernel (tc == 0). */
int ab_linalg_status_reset(void* status, void* stream);
int ab_linalg_status_check(const void* status, void* stream);
uint64_t ab_linalg_update_count(int tensor_core);
int ab_cholesky_workspace_bytes(int dtype, int64_t n, size_t* bytes);
int ab_cholesky(int dtype, int64_t n, const void* a, int64_t a_rs, int64_t a_cs, int lower,
                int nan_on_error, int check_finite, void* out, void* status, void* workspace,
                size_t workspace_bytes, void* stream);
int ab_trsm_workspace_bytes(int dtype, int64_t n, int64_t nrhs, size_t* bytes);
int ab_trsm(int dtype, int64_t n, int64_t nrhs, const void* a, int64_t a_rs, int64_t a_cs,
            int lower, int trans, int unit_diagonal, const void* b, int64_t b_rs, int64_t b_cs,
            void* x, int check_finite, int check_singular, void* status, void* workspace,
            size_t workspace_bytes, void* stream);

/* ---- Scan fast path: LSTM-cell recurrence as one persistent kernel -----------------
 * (aesara/scan/op.py:637; inner graph of SURVEY App. A.4).  For t in [0,T):
 *   pre = x[t] + h_{t-1} @ U;  c_t = sigmoid(pre_f)*c_{t-1} + sigmoid(pre_i)*tanh(pre_g);
 *   h_t = sigmoid(pre_o)*tanh(c_t)      (gate column order i, f, o, g; 3xTF32 wgmma tiles)
 * hbuf / cbuf are the Scan's circular output buffers [sh|sc, B, H] (contiguous); the row
 * before pos_h / pos_c holds the initial state; step t writes row (pos + t) % s.
 * x is [T, B, 4H] with element strides (x_ts, x_rs, 1); U is [H, 4H] with strides
 * (u_rs, u_cs).  One cooperative launch; there is no barrier between steps: a step-t+1
 * tile waits only for the step-t tiles of its own 256-row block (per-row-block counters). */
int ab_lstm_scan_supported(int64_t t, int64_t b, int64_t h);
int ab_lstm_scan_workspace_bytes(int64_t b, int64_t h, size_t* bytes);
int ab_lstm_scan(int64_t T, int64_t B, int64_t H, const void* x, int64_t x_ts, int64_t x_rs,
                 const void* U, int64_t u_rs, int64_t u_cs, void* hbuf, int64_t sh, int64_t pos_h,
                 void* cbuf, int64_t sc, int64_t pos_c, void* workspace, size_t workspace_bytes,
                 void* stream);

/* The same persistent kernel for the whole family "one Gemm(x_t, 1, s_hs, U, 1) + Elemwise
 * nodes on its column slices" (aesara/scan/op.py:1673-2160 runs such an inner function step
 * by step): pre = x[t] + s_hs[t-1] @ U is [B, gates*H]; the cell maps the `gates` column
 * blocks of pre and the `states` previous states to the new states.  `module` is the NVRTC
 * build of csrc/ab_scan_cell_kernel.cuh with the cell generated from the inner graph's scalar
 * expressions (aesara_b200/codegen/scan_cell.py).  state_bufs[k] is the Scan's output ring
 * [state_lens[k], B, H] of state k (row state_pos[k] - 1 holds the initial value); x is
 * [T, B, gates*H] with strides (x_ts, x_rs, 1); U is [H, gates*H] with strides (u_rs, u_cs). */
int ab_cell_scan_supported(int gates, int states, int64_t t, int64_t b, int64_t h);
int ab_cell_scan_workspace_bytes(int gates, int64_t b, int64_t h, size_t* bytes);
int ab_cell_scan(ab_module* module, int gates, int states, int hs, int64_t T, int64_t B, int64_t H,
                 const void* x, int64_t x_ts, int64_t x_rs, const void* U, int64_t u_rs, int64_t u_cs,
                 void* const* state_bufs, const int64_t* state_lens, const int64_t* state_pos,
                 void* workspace, size_t workspace_bytes, void* stream);

/* number of kernels this library has launched since load (bench.py reports it) */
uint64_t ab_launch_count(void);

#ifdef __cplusplus
}
#endif
#endif /* AESARA_B200_H */
