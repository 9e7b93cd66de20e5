/* quanto_b200 -- C ABI of the H100-native quantized-linear hot path.
 *
 * This is the drop-in boundary for the CUDA side of huggingface/optimum-quanto's quantized linear forward
 * (reference commit e33f8202).  Every entry point takes raw DEVICE pointers and sizes, enqueues work on the
 * caller's stream, never allocates, never synchronises, and returns an int status (0 = ok), the convention of the
 * reference's marlin binding (optimum/quanto/library/extensions/cuda/marlin/marlin_cuda.cpp:25-26,65-74:
 * ERR_PROB_SHAPE = 1, ERR_KERN_SHAPE = 2).  The caller (the torch.library "CUDA" impls, see INTEGRATION.md)
 * validates dtype / contiguity / device, allocates outputs with torch.empty and passes
 * torch.cuda.current_stream().cuda_stream.
 *
 * Replaces the pybind11 module `quanto_cuda` (optimum/quanto/library/extensions/cuda/pybind_module.cpp:30-37)
 * whose functions exchange torch::Tensor by value and allocate their own outputs.
 */
#ifndef QUANTO_B200_H
#define QUANTO_B200_H

#include <stdint.h>

#if defined(__GNUC__)
#define QB200_API __attribute__((visibility("default")))
#else
#define QB200_API
#endif

#ifdef __cplusplus
extern "C" {
#endif

/* status codes */
#define QB200_OK 0
#define QB200_ERR_ARG 1         /* bad problem description (shape, dtype, alignment)  ~ ERR_PROB_SHAPE */
#define QB200_ERR_UNSUPPORTED 2 /* no kernel for this configuration                  ~ ERR_KERN_SHAPE */
#define QB200_ERR_CUDA 3        /* a CUDA runtime / driver call failed (see qb200_last_error) */
#define QB200_ERR_ARCH 4        /* device is not sm_90 */

/* element types */
#define QB200_F32 0
#define QB200_F16 1
#define QB200_BF16 2
#define QB200_I8 3
#define QB200_U8 4
#define QB200_E4M3 5 /* torch.float8_e4m3fn */
#define QB200_E5M2 6 /* torch.float8_e5m2   */
#define QB200_E4M3FNUZ 7 /* torch.float8_e4m3fnuz (weights of qbytes_mm, target of quantize_symmetric) */

/* Library version (round * 100 + revision). */
QB200_API int qb200_version(void);

/* 1 if `device` can run the kernels (compute capability 10.x), 0 if not, negative on CUDA error. */
QB200_API int qb200_device_supported(int device);

/* Human-readable description of the last non-zero status returned on the calling thread. */
QB200_API const char* qb200_last_error(void);

/* quanto::unpack(Tensor self, int bits) -> Tensor
 * reference: optimum/quanto/library/unpack.py:18-54 (schema, python impl),
 *            optimum/quanto/library/extensions/cuda/unpack.cu:85-97 (CUDA entry `unpack`, pybind_module.cpp:36).
 * in: n_bytes packed uint8; out: n_bytes * (8/bits) uint8, plane p at out + p*n_bytes. bits in {2, 4}. */
QB200_API int qb200_unpack(const uint8_t* in, uint8_t* out, int64_t n_bytes, int bits, void* stream);

/* quanto::quantize_symmetric(Tensor base, ScalarType dtype, int? axis, Tensor scale) -> Tensor
 * reference: optimum/quanto/library/quantize.py:22-55 (python only; no native kernel upstream).
 * base is contiguous, viewed as [outer, inner].  axis_mode: 0 per-tensor (scale has 1 element),
 * 1 = axis 0 (scale[outer]), 2 = axis -1 (scale[inner]).  in_dtype in {F32,F16,BF16} (scale has the same dtype);
 * out_dtype in {I8, E4M3, E5M2, E4M3FNUZ}.  Bit-exact with the reference (quotient rounded to in_dtype before rint). */
QB200_API int qb200_quantize_symmetric(const void* base, const void* scale, void* out, int64_t outer, int64_t inner,
                             int axis_mode, int in_dtype, int out_dtype, void* stream);

/* QBitsTensor.dequantize() for axis-0 weights in canonical storage, one launch.
 * reference: optimum/quanto/tensor/qbits.py:27-49 (unpack, scale*data, -= shift, ungroup).
 * packed: uint8 [ceil(N*K/group / (8/bits)), group]; scale/shift: [N*K/group] in `dtype` (shift: uint8 zero-point
 * when shift_is_int); out: [N, K] `dtype`.  Bit-exact. */
QB200_API int qb200_dequantize_qbits(const uint8_t* packed, const void* scale, const void* shift, void* out, int64_t n,
                           int64_t k, int group, int bits, int dtype, int shift_is_int, void* stream);

/* Fused packed-int4 / int2 linear: out[M,N] = A[M,K] @ dequant(packed, scale, shift)[N,K]^T (+ bias).  The `udqmm`
 * role: replaces quanto::gemm_f16i4_awq / gemm_f16i4_marlin (optimum/quanto/library/extensions/cuda/__init__.py:82-121,
 * 170-202) and the dequantize-then-matmul path (optimum/quanto/tensor/weights/qbits.py:276-281,
 * optimum/quanto/tensor/function.py:42-47).  Weights stay in quanto's canonical axis-0 packing (no repacking):
 * packed uint8 [ceil(N*K/group / (8/bits)), group], scale / shift [N*K/group] (shift: `dtype`, or uint8 zero-points when
 * shift_is_int), group divides K (per-axis quantisation: group = K).  dtype in {F32, F16, BF16} (A, scale, shift, bias,
 * out); bits in {2, 4}.
 * Kernel selection: 4-bit, F16 / BF16, N even, K % 16 == 0, group 32 or a multiple of 64 and 16-byte aligned buffers run
 * on the TMA / tensor-core kernels (M <= 16: TMA-ring gemvs; M <= 8 shapes they decline: stream-K gemv; otherwise the
 * persistent wgmma GEMM); every
 * other valid problem runs on a shape-agnostic CUDA-core kernel with the same operands and rounding order -- there is
 * no library / eager fallback behind this entry point.
 *
 * `workspace` (device memory, may be NULL): scratch for the small-M stream-K gemv, at least
 * qb200_qbits_mm_workspace_bytes(m, n, k) bytes, ZERO-INITIALISED ONCE by the caller (the kernel leaves its ticket
 * counters zero on exit) and not shared between streams that run concurrently.  Like the caller-provided zeroed
 * `workspace` of the reference's marlin binding (optimum/quanto/tensor/weights/marlin/int4/qbits.py:101).  Without
 * it, 8 < M <= 128 calls use the general kernel (same results, lower bandwidth). */
QB200_API int qb200_qbits_mm(const void* a, const uint8_t* packed, const void* scale, const void* shift, const void* bias,
                   void* out, int64_t m, int64_t n, int64_t k, int group, int bits, int dtype, int shift_is_int,
                   void* workspace, int64_t workspace_bytes, void* stream);

/* Column-parallel form of qb200_qbits_mm with the all-gather of the output AND the rank synchronisation fused into the
 * kernel (SURVEY 8e; the reference has no distributed code -- optimum/quanto/nn/qlinear.py:49-50 is the single-device
 * call this shards).  This rank holds the [n_local, K] slice `rank` of the weight (itself a canonical packed tensor, see
 * quanto_b200/parallel.py::shard_weight).
 *   out_peers  : HOST array of `world` DEVICE pointers, the full [M, n_local * world] output buffer of every rank,
 *                peer-mapped into this process (symmetric memory over NVLink).  Every output tile is stored into columns
 *                [rank * n_local, (rank + 1) * n_local) of all of them from the kernel's epilogue (staged in shared
 *                memory, full rows handed to the TMA store unit), so there is no collective launch and no re-read.
 *   flag_peers : HOST array of `world` DEVICE pointers to every rank's flag array (world + 2 uint32, peer-mapped,
 *                zero-initialised once).  The kernels synchronise the ranks through them (csrc/gather.cuh): a kernel
 *                publishes "my slab has landed everywhere" when its last CTA finishes; no host-issued barrier is needed.
 *   wait_flags : QB200_GATHER_WAIT_INPUT  -- `a` is itself the gathered output of the previous gathered call: the role
 *                                            that reads it waits (in-kernel) until every rank has published that call;
 *                QB200_GATHER_WAIT_OUTPUT -- the kernel completes only when every rank's slab has landed in THIS rank's
 *                                            buffer (for consumers that are not gathered kernels: copies, ATen ops).
 * All ranks must issue the same sequence of gathered calls.  A buffer may be reused once two other gathered calls have
 * been issued since its last reader was enqueued.  Needs (n_local / 2) % 64 == 0.  `workspace`: as for qb200_qbits_mm
 * (qb200_qbits_mm_workspace_bytes(m, n_local, k)); without it 8 < M <= 128 runs on the general kernel. */
#define QB200_GATHER_WAIT_INPUT 1
#define QB200_GATHER_WAIT_OUTPUT 2
QB200_API int qb200_qbits_mm_gather(const void* a, const uint8_t* packed, const void* scale, const void* shift,
                                    const void* bias, void* const* out_peers, void* const* flag_peers, int world,
                                    int rank, int wait_flags, int64_t m, int64_t n_local, int64_t k, int group,
                                    int dtype, int shift_is_int, void* workspace, int64_t workspace_bytes, void* stream);

/* Bytes of workspace the small-M path of qb200_qbits_mm wants for this problem (0 = the path is not used). */
QB200_API int64_t qb200_qbits_mm_workspace_bytes(int64_t m, int64_t n, int64_t k);

/* Host-only query (no GPU needed; tests): how the decode ring kernel (M <= 16) would cut K for this problem on `grid` CTAs.
 * Returns 1 and fills out5 = {64-byte slabs per warp and stage, passes over K, ring stages, token groups of 8, dynamic
 * shared memory bytes}, or 0 when that kernel does not take the problem.  The first two decide the order in which every
 * output's sum is formed; they depend on (M, K, group, zeropoint) only -- never on N -- which is what makes a column shard
 * bit-identical to the same rows of the full matrix. */
QB200_API int qb200_qbits_ring_plan(int64_t m, int64_t n, int64_t k, int group, int zeropoint, int grid, int* out5);

/* quanto::qbytes_mm(Tensor A, Tensor B, Tensor scales) -> Tensor   (+ optional fused bias)
 * reference: optimum/quanto/library/qbytes_mm.py:22 (schema), :25-33 (python), :36-50 (int), :73-88 (CUDA dispatch).
 * A [M,K] a_dtype in {I8,E4M3,E5M2,E4M3FNUZ,F16,BF16,F32}; W [N,K] w_dtype in {I8,E4M3,E5M2,E4M3FNUZ}; scales [N] and out [M,N] in
 * out_dtype in {F32,F16,BF16}.  int8 x int8 is exact (int32 accumulate, fp32 scale, one rounding). */
QB200_API int qb200_qbytes_mm(const void* a, const void* w, const void* scales, const void* bias, void* out, int64_t m,
                    int64_t n, int64_t k, int a_dtype, int w_dtype, int out_dtype, void* stream);

/* qbytes_mm with the output quantisation of the quantized linear fused into the epilogue (SURVEY.md 8f rank 2):
 * WeightQBytesLinearFunction (optimum/quanto/tensor/weights/qbytes.py:68-82: qbytes_mm(...) + bias) followed by the
 * QModuleMixin.quantize_output hook (optimum/quanto/nn/qmodule.py:300-302 -> quanto::quantize_symmetric, per tensor) as
 * ONE launch: out_q[m, n] = quantize_symmetric(rnd(rnd(acc * scales[n]) + bias[n]), out_scale) -- the [M, N] result is
 * never written in 16 bits and read back.  Bit-exact with that composition.
 * A, W both int8 or both float8 (the kernels quantized activations reach); scales [N], bias [N] or NULL and out_scale
 * (ONE element, device memory) in scale_dtype in {F32, F16, BF16}; out_q [M, N] bytes of q_dtype in {I8, E4M3, E5M2}.
 * Returns QB200_ERR_UNSUPPORTED when the tensor-core kernels do not take the problem (K % 16 != 0, unaligned buffers,
 * mixed operand types): the caller then composes qb200_qbytes_mm + qb200_quantize_symmetric. */
QB200_API int qb200_qbytes_mm_quantized(const void* a, const void* w, const void* scales, const void* bias, void* out_q,
                                        const void* out_scale, int64_t m, int64_t n, int64_t k, int a_dtype, int w_dtype,
                                        int scale_dtype, int q_dtype, void* stream);

/* ---- quantized attention: per-tensor int8 / float8 activations kept quantized (the reference's ActivationQBytesTensor
 * op table, optimum/quanto/tensor/activations/qbytes_ops.py) ------------------------------------------------------ */

/* aten.bmm of two qint8 activations (qbytes_ops.py:175-186):
 *   out[b] = rnd_dt( f32(A[b] @ B[b]) * f32(rnd_dt(scale_a * scale_b)) )
 * with the sum an exact int32 sum (bit-identical to the reference's fp32 bmm whenever K <= 1024).
 * A: int8 [batch, m, k], rows dense, batch b at a + b * a_batch_stride (0 = one A for every batch).
 * B: int8, element (k, n) of batch b at b + b * b_batch_stride + (b_layout == 0 ? n * k + k : k * n + n): layout 0 is
 * K-contiguous (a transposed key), layout 1 N-contiguous (a value, or a key after matmul's reshape); stride 0 = one B
 * for every batch (an expanded operand, read in place).
 * scale_a, scale_b: ONE element each (device memory) of scale_dtype in {F32, F16, BF16}; out: dense [batch, m, n] of
 * scale_dtype.
 * K % 16 == 0 with A 16-byte aligned runs on the tensor cores (wgmma, family 1); an N-contiguous B is first copied
 * K-major by one byte-transpose pass into `workspace` (family 4), which must hold
 * qb200_qbytes_bmm_workspace_bytes(...) bytes, 16-byte aligned, owned by the call until the stream reaches its end.
 * Every other problem runs on a CUDA-core kernel with the same exact sum and roundings (family 2). */
QB200_API int qb200_qbytes_bmm(const void* a, const void* b, const void* scale_a, const void* scale_b, void* out,
                               void* workspace, int64_t workspace_bytes, int64_t batch, int64_t m, int64_t n, int64_t k,
                               int64_t a_batch_stride, int64_t b_batch_stride, int b_layout, int scale_dtype,
                               void* stream);

/* Bytes of workspace qb200_qbytes_bmm needs for this B (0 when B is read in place). */
QB200_API int64_t qb200_qbytes_bmm_workspace_bytes(int64_t batch, int64_t n, int64_t k, int64_t b_batch_stride,
                                                   int b_layout);

/* aten._softmax over the last dim of a per-tensor quantized activation, re-quantized (qbytes_ops.py:208-215), in one
 * launch: x, out: [rows, cols] codes of q_dtype in {I8, E4M3, E5M2, E4M3FNUZ}; scale (the input's) and out_scale
 * (1 / qmax rounded to the scale dtype, as torch.tensor(1 / qmax, dtype=...) gives it): ONE element each of
 * scale_dtype in {F32, F16, BF16}, device memory.  Per row: x = rnd_dt(scale * payload), y = rnd_dt(softmax(x)) with
 * fp32 max / exp / sum, out = quantize_symmetric(y, q_dtype, out_scale).  Any row length; rows of up to 32768 codes are
 * read from memory once. */
QB200_API int qb200_qbytes_softmax(const void* x, const void* scale, const void* out_scale, void* out, int64_t rows,
                                   int64_t cols, int q_dtype, int scale_dtype, void* stream);

/* ---- quantized layer norm (the reference's QLayerNorm, optimum/quanto/nn/qlayernorm.py:27-53) -------------------- */

/* F.layer_norm over rows of h elements (qlayernorm.py:52-53), optionally from and to 8-bit codes, in one launch
 * (family 6).  Replaces F.layer_norm after qfallback's dequantize of an ActivationQBytesTensor input
 * (tensor/qbytes.py:23-31) followed by the quantize_output hook (nn/qmodule.py:296-302 -> library/quantize.py:51-55):
 *   x   = x[r, i] in `dtype`, or rnd_dt(in_scale * payload) when in_dtype is a code dtype
 *   y   = rnd_dt(weight[i] * (x - mean) / sqrt(var + eps) + bias[i])   fp32 mean, then the biased variance about it;
 *                                                                        1 / sqrt correctly rounded
 *   out = y in `dtype` (out_dtype == dtype), or quantize_symmetric(y, out_dtype, out_scale): the quotient y / out_scale
 *         rounded to `dtype`, then rint / clamp / cast as qb200_quantize_symmetric.
 * x: dense [rows, h] of in_dtype, in `dtype` in {F32, F16, BF16} or codes in {I8, E4M3, E5M2, E4M3FNUZ}; in_scale: ONE
 * element of `dtype` (codes in only).  weight, bias: [h] in `dtype`, each may be NULL.  out: dense [rows, h] of
 * out_dtype (`dtype` or a code dtype).  out_scale: ONE element of out_scale_dtype in {F32, dtype}, read on the device
 * (codes out only; F32 with a 16-bit dtype divides by the fp32 value, as ATen's CPU division by a 0-dim fp32 tensor
 * does).  Any h >= 1; rows of up to 16384 elements are read from memory once. */
QB200_API int qb200_layer_norm(const void* x, const void* in_scale, const void* weight, const void* bias,
                               const void* out_scale, void* out, int64_t rows, int64_t h, double eps, int in_dtype,
                               int dtype, int out_dtype, int out_scale_dtype, void* stream);

/* ---- quantized 2-D convolution (the reference's QConv2d, optimum/quanto/nn/qconv2d.py) -------------------------- */

/* out = F.conv2d(x, dequantize(W), bias, stride, padding, dilation) with groups == 1, as an implicit GEMM on the tensor
 * cores (family 5): M = batch * Ho * Wo output pixels, N = cout, K = cin * kh * kw with k = c * kh * kw + r * kw + s.
 * The weight [cout, cin, kh, kw] quantized along axis 0 is the linear weight [N, K] of qb200_qbits_mm (canonical packing,
 * scale / shift [N * K / group]) and is dequantised in-kernel with the same arithmetic.  x: [batch, cin, h, w] and
 * out: [batch, cout, Ho, Wo], both NCHW-contiguous in `dtype` (BF16 / F16), Ho = (h + 2 pad_h - dil_h (kh - 1) - 1) /
 * stride_h + 1 (likewise Wo); zero padding.  bias: [cout] in `dtype` or NULL; out = rnd(conv + bias) with the bias
 * added to the fp32 sum, the one rounding of the reference's QConv2d on the CPU (ATen's cuDNN path rounds the conv,
 * then the bias add).  Nothing is allocated.
 * QB200_ERR_ARG: bad shape or geometry, group not dividing K.  QB200_ERR_UNSUPPORTED: dtype F32, bits != 4, odd cout,
 * K % 16 != 0, group neither a multiple of 32 nor K, M / N / K over int32, packed not 16-byte aligned, x / out / bias not
 * aligned to their elements. */
QB200_API int qb200_qbits_conv2d(const void* x, const uint8_t* packed, const void* scale, const void* shift,
                                 const void* bias, void* out, int64_t batch, int64_t cin, int64_t h, int64_t w,
                                 int64_t cout, int64_t kh, int64_t kw, int stride_h, int stride_w, int pad_h, int pad_w,
                                 int dil_h, int dil_w, int group, int bits, int dtype, int shift_is_int, void* stream);

/* The same for a weight-only 8-bit weight: W [cout, cin * kh * kw] of w_dtype in {I8, E4M3, E5M2, E4M3FNUZ} and
 * scales [cout] in `dtype`; the weight operand is rnd(scale * W), as for qb200_qbytes_mm.  Same errors, with W
 * (instead of packed) required 16-byte aligned. */
QB200_API int qb200_qbytes_conv2d(const void* x, const void* w, const void* scales, const void* bias, void* out,
                                  int64_t batch, int64_t cin, int64_t h, int64_t w_, int64_t cout, int64_t kh, int64_t kw,
                                  int stride_h, int stride_w, int pad_h, int pad_w, int dil_h, int dil_w, int w_dtype,
                                  int dtype, void* stream);

/* ---- input gradient of the quantized linear (the backward's dX = gO @ W) ---------------------------------------- */

/* grad_in[M, K] = grad_out[M, N] @ dequant(packed, scale, shift)[N, K] in one launch, reading the packed weights.
 * Replaces the reference's backward composition QuantizedLinearFunction.backward (optimum/quanto/tensor/function.py:
 * 49-63: torch.matmul(gO, other)) -> qfallback (optimum/quanto/tensor/qtensor.py: other.dequantize(), a dense [N, K] copy
 * of the weight) -> QBitsDequantizer (optimum/quanto/tensor/qbits.py:27-49) -> a dense GEMM.
 * The weight operand is bit-identical to qb200_dequantize_qbits; fp32 accumulation, one rounding to `dtype`, no bias.
 * packed: canonical 4-bit storage, uint8 [N*K/group / 2, group] (as for qb200_qbits_mm with bits = 4); scale / shift
 * [N*K/group] in `dtype` (shift: uint8 zero-points when shift_is_int); grad_out [M, N], grad_in [M, K] in `dtype`.
 * QB200_ERR_ARG: bad shape, group not dividing K, dtype not F32 / F16 / BF16.
 * QB200_ERR_UNSUPPORTED (the caller composes dequantize + GEMM instead): dtype F32; N % 16 != 0 (odd N included);
 * K % 16 != 0; group neither 32 nor a multiple of 64; grad_out, packed or grad_in not 16-byte aligned.  2-bit weights
 * have no kernel: do not pass them here. */
QB200_API int qb200_qbits_mm_grad_input(const void* grad_out, const uint8_t* packed, const void* scale, const void* shift,
                                        void* grad_in, int64_t m, int64_t n, int64_t k, int group, int dtype,
                                        int shift_is_int, void* stream);

/* grad_in[M, K] = grad_out[M, N] @ (scales[n] * W[n, k])[N, K] in one launch: the input gradient of the 8-bit linear.
 * Replaces the same backward composition with QBytesDequantizer (optimum/quanto/tensor/qbytes.py:23-31: scale * data in
 * the scale dtype, one rounding) as the dequantisation; the weight operand is bit-identical to it.
 * W [N, K] of w_dtype in {I8, E4M3, E5M2, E4M3FNUZ}; scales [N] (one per out-feature), grad_out [M, N], grad_in [M, K]
 * in `dtype`.  QB200_ERR_UNSUPPORTED: dtype F32; N % 8 != 0; K % 16 != 0; grad_out, W or grad_in not 16-byte aligned.
 * A per-tensor scale has no kernel: expand it to [N] or compose. */
QB200_API int qb200_qbytes_mm_grad_input(const void* grad_out, const void* w, const void* scales, void* grad_in,
                                         int64_t m, int64_t n, int64_t k, int w_dtype, int dtype, void* stream);

/* ---- weight freeze / calibration: the step before the hot path (SURVEY.md 8f rank 1-2) ------------------------- */

/* quanto::quantize_affine(Tensor base, int bits, int axis, int? group_size, Tensor scale, Tensor shift) -> Tensor
 * reference: optimum/quanto/library/quantize.py:58-78 (python only upstream: group, add/div, round, clamp, cast =
 * 4-5 ATen launches).  `base` is the already GROUPED weight viewed as [outer, inner] in `dtype` (axis 0 grouping is a
 * pure reshape, optimum/quanto/tensor/grouped.py:17-30).  axis_mode: 0 = one scale/shift, 1 = per row (scale[outer]),
 * 2 = per column (scale[inner]).  shift: `dtype`, or zero-point bytes: shift_is_int 1 = uint8 values, 2 = int8 values
 * (the reference adds the tensor's VALUE, so int8 zero-points may be negative).  out: uint8 [outer, inner],
 * values in [0, 2^bits - 1].  Bit-exact with the reference's CPU arithmetic. */
QB200_API int qb200_quantize_affine(const void* base, const void* scale, const void* shift, uint8_t* out, int64_t outer,
                                    int64_t inner, int axis_mode, int bits, int dtype, int shift_is_int, void* stream);

/* pack_weights(intweights, bits) -- optimum/quanto/tensor/packed.py:24-69 (a python loop of shift/or launches).
 * in: uint8 [rows, cols]; out: uint8 [ceil(rows / (8/bits)), cols]; plane p of out row r = in row r + p*R.
 * The inverse of qb200_unpack followed by the [:rows] slice.  bits in {2, 4}. */
QB200_API int qb200_pack(const uint8_t* in, uint8_t* out, int64_t rows, int64_t cols, int bits, void* stream);

/* freeze() of an axis-0 int4/int2 weight in ONE launch: MaxOptimizer (optimum/quanto/tensor/optimizers/
 * max_optimizer.py:26-37 + affine_optimizer.py:52-63) + quanto::quantize_affine + pack_weights, i.e. what
 * QModuleMixin.qweight / freeze (optimum/quanto/nn/qmodule.py:245-266, 304-307) run as ~12 launches.
 * base: [n, k] `dtype` row-major, 16-byte aligned; group divides k, group % 8 == 0, group <= 256 (else
 * QB200_ERR_UNSUPPORTED: compose ATen amin/amax + qb200_quantize_affine + qb200_pack).  rows = n*k/group.
 * packed: uint8 [ceil(rows/(8/bits)), group]; scale: [rows] `dtype`; shift: [rows] `dtype`, or uint8 zero-points when
 * `zeropoint`.  Bit-exact with the reference's CPU arithmetic (true division by 2^bits-1; torch's CUDA kernels
 * multiply by the reciprocal there, which can differ in the last bit). */
QB200_API int qb200_quantize_qbits_max(const void* base, uint8_t* packed, void* scale, void* shift, int64_t n, int64_t k,
                                       int group, int bits, int dtype, int zeropoint, void* stream);

/* max |base| over the whole tensor (the reduction of absmax_scale, optimum/quanto/calibrate.py:37-61: abs + max, two
 * ATen passes), written to out[0] in `dtype`.  `scratch`: 8 bytes of device memory, 4-byte aligned, zeroed on the stream
 * by this call (running maximum + CTA ticket; the last CTA publishes the result). */
QB200_API int qb200_absmax(const void* base, void* out, void* scratch, int64_t numel, int dtype, void* stream);

/* One calibration step of a per-tensor activation scale, in place and without a host synchronisation: absmax_scale
 * (optimum/quanto/calibrate.py:37-61) and the momentum update of Calibration (calibrate.py:31-34) as ONE launch.
 *   new    = rnd(max|base| / qmax)                  true division, rounded to `dtype`
 *   *scale = (*scale == 1) ? new : rnd(rnd(*scale * m) + rnd(new * om)),  m = (float)momentum, om = (float)(1 - momentum)
 * Every rnd rounds to `dtype`, as the reference's ATen ops do; a NaN in base gives a NaN scale.  base: `numel` >= 1
 * elements of `dtype` (f32 / f16 / bf16), any alignment (16-byte aligned bases take vector loads); scale: one element
 * of `dtype`; `scratch`: 8 bytes of device memory, 4-byte aligned, zeroed on the stream by this call.  QB200_ERR_ARG
 * for an empty tensor, a non-float dtype, qmax <= 0 or a misaligned scratch buffer. */
QB200_API int qb200_absmax_update(const void* base, void* scale, void* scratch, int64_t numel, int dtype, double qmax,
                                  double momentum, void* stream);

/* freeze() of an axis-0 8-bit weight in ONE launch: AbsmaxOptimizer (optimum/quanto/tensor/optimizers/
 * absmax_optimizer.py:29-36: scale[n] = max|W[n,:]| / qmax, qmax = 127 / 448 / 57344) + quanto::quantize_symmetric
 * (optimum/quanto/library/quantize.py:51-55).  base [n, k] `dtype`; out [n, k] out_dtype in {I8, E4M3, E5M2};
 * scale [n] `dtype`.  Bit-exact with the reference's CPU arithmetic. */
QB200_API int qb200_quantize_qbytes_absmax(const void* base, void* out, void* scale, int64_t n, int64_t k, int dtype,
                                           int out_dtype, void* stream);

/* freeze() of an axis-0 int4/int2 weight with the HQQ optimizer in TWO launches and no host synchronisation:
 * HqqOptimizer (optimum/quanto/tensor/optimizers/hqq_optimizer.py:28-34 shrink_lp_op, :60-87 optimize, after
 * max_optimizer.py:26-37) + affine_optimizer.py:52-63 (zeropoint) + quanto::quantize_affine + pack_weights.
 * Outputs as qb200_quantize_qbits_max.  `errors`: float32 [iters + 2], the dt-rounded tensor-wide mean errors of the
 * all-accepted trajectory (start error, then one per iteration), then the number of accepted iterations.
 * `workspace`: qb200_quantize_qbits_hqq_workspace_bytes(n, k, group, iters) bytes of device memory, 256-byte aligned,
 * owned by the call until the stream reaches its end.  bf16 / fp16 only, group % 8 == 0, group <= 256, iters <= 64,
 * lp_norm > 0 (not 4, where torch's pow is a cube); else QB200_ERR_UNSUPPORTED.  Bit-exact with the reference's CPU
 * arithmetic for the scale, shift and packed codes; the stop index follows from the dt-rounded means. */
QB200_API int qb200_quantize_qbits_hqq(const void* base, uint8_t* packed, void* scale, void* shift, float* errors,
                                       void* workspace, int64_t n, int64_t k, int group, int bits, int dtype,
                                       int zeropoint, double lp_norm, double beta, double kappa, int iters, void* stream);

/* Bytes of workspace qb200_quantize_qbits_hqq needs (0 for an invalid shape). */
QB200_API int64_t qb200_quantize_qbits_hqq_workspace_bytes(int64_t n, int64_t k, int group, int iters);

/* shrink_lp_op(x, beta, lp_norm) (optimum/quanto/tensor/optimizers/hqq_optimizer.py:28-34) elementwise on `numel`
 * bf16 / fp16 values: the device shrink qb200_quantize_qbits_hqq uses, exposed so that it can be checked on every input.
 * Same configurations as qb200_quantize_qbits_hqq. */
QB200_API int qb200_hqq_shrink(const void* x, void* out, int64_t numel, double beta, double lp_norm, int dtype,
                               void* stream);

/* Which kernel family the last qb200_qbytes_mm / qb200_qbytes_bmm / qb200_qbits_mm / *_grad_input / qb200_layer_norm call on this thread dispatched to:
 * 0 none, 1 wgmma (TMA + warpgroup MMA), 2 CUDA-core (shape-agnostic), 3 warp-MMA gemv (int4, M <= 32: TMA ring or register streaming),
 * 4 byte-transpose pass + wgmma (qb200_qbytes_bmm with a B that is not K-contiguous), 5 implicit-GEMM convolution
 * (qb200_qbits_conv2d / qb200_qbytes_conv2d), 6 layer norm (qb200_layer_norm: one warp per row up to 1024 elements, one
 * CTA per row above).
 * For tests and bench accounting. */
QB200_API int qb200_last_kernel_family(void);

/* Test hook: choose among kernels that all compute the same result, so that a test-suite can execute every shipped
 * instantiation (value 0 = automatic choice, the default).  Process-wide.
 *   key 0  wgmma tile rows                 : 64 (one consumer warpgroup) | 128 (two)
 *   key 1  int8 x int8 tile N              : 128 | 256
 *   key 2  int4 route                      : 1 wgmma kernel, 3 warp-MMA gemv (M <= 32), 4 TMA-ring gemv (M <= 8),
 *                                            8 second-generation TMA-ring gemv (M <= 16)
 *   key 3  qbytes route                    : 2 CUDA-core kernel
 *   key 4  ring-gemv producer              : 1 one issuing thread, 2 one lane per packed row, 3 32 lanes
 *   key 5  programmatic dependent launch   : 1 off
 *   key 6  ring-gemv shape (M <= 2)        : 2 two CTAs per SM (opt-in experiment; default one CTA per SM)
 *   key 7  int4 wgmma epilogue             : 1 ordinary stores (default: TMA stores from a shared-memory tile when the
 *                                            output is one dense [M, N] buffer with N % 16 == 0)
 *   key 8  qbytes_bmm route                : 2 CUDA-core kernel, 3 byte-transpose pass + wgmma for either B layout
 *                                            (default: wgmma reading a K-contiguous B in place)
 *   key 9  conv2d tile rows                : 64 | 128 output pixels per tile */
QB200_API int qb200_test_override(int key, int value);

/* Developer aids.  They act only in a library built with `make KNOCKOUTS=1` (qb200_developer_build() == 1); in the
 * release library the setters are no-ops and qb200_debug_flags() is always 0.
 *   qb200_debug_set_trace : device buffer of >= 4*5*64 int64 for clock64 stamps of the pipeline roles
 *   qb200_debug_set_flags : timing knock-outs, results are WRONG while set: 1 skip dequant arithmetic, 2 skip the MMA,
 *                           4 constant scales, 8 skip activations / stream only, 16 no segment end,
 *                           256 no output rows,
 *                           512 extra trace stamps */
QB200_API void qb200_debug_set_trace(void* device_buffer);
QB200_API void qb200_debug_set_flags(int flags);
QB200_API int qb200_debug_flags(void);
QB200_API int qb200_developer_build(void);

#ifdef __cplusplus
}
#endif

#endif /* QUANTO_B200_H */
