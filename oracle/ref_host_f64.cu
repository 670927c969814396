// TEST INFRASTRUCTURE (oracle/_ref): host side of the reference's float64 DCNv2 build (_ext.dcn_v2_double) on the GPU.
//
// The reference's float64 kernels are compiled UNMODIFIED, from where they lie under /root/reference
//   src/lib/models/networks/DCNv2/src/cuda/dcn_v2_im2col_cuda_double.cu
//   src/lib/models/networks/DCNv2/src/cuda/dcn_v2_psroi_pooling_cuda_double.cu
// (recipe: oracle/build_ref_f64.py) and linked with this file into oracle/_ref/libdcnv2_ref_f64.so, a library of
// its own because the float and double files export the same extern "C" launcher names.  The reference's host
// wrapper (src/dcn_v2_cuda_double.c) is written against the THC API that no longer exists, so its per-sample loop
// is re-stated here with plain cuBLAS calls, keeping the order of the launches, the GEMM shapes/transposes and the
// accumulation (beta) of
//   forward : dcn_v2_cuda_double.c:66-105   (bias via ones x bias DGEMM, im2col, Y += W.col)
//   backward: dcn_v2_cuda_double.c:177-247  (col = W^T.dY, col2im_coord, col2im, im2col, dW += , dB += by DGEMV)
//   pooling : dcn_v2_cuda_double.c:266-357
// THCudaBlas_Dgemm(ta, tb, m, n, k, ...) is cublasDgemm with the same column-major arguments.
// Plain C ABI, raw device pointers; `columns`/`ones` scratch is caller-allocated as in the
// reference (dcn_v2_func.py:30-33).  Returns 0 or a non-zero cuBLAS/CUDA status.
#include <cublas_v2.h>
#include <cuda_runtime.h>
#include "dcn_v2_im2col_cuda_double.h"
#include "dcn_v2_psroi_pooling_cuda_double.h"

namespace {
cublasHandle_t g_handle = nullptr;
int handle_for(cudaStream_t s) {
    if (!g_handle) {
        if (cublasCreate(&g_handle) != CUBLAS_STATUS_SUCCESS) return 1;
        cublasSetMathMode(g_handle, CUBLAS_PEDANTIC_MATH);
    }
    return cublasSetStream(g_handle, s) == CUBLAS_STATUS_SUCCESS ? 0 : 2;
}
inline cublasOperation_t op(char c) { return c == 't' ? CUBLAS_OP_T : CUBLAS_OP_N; }
int dgemm(char ta, char tb, long m, long n, long k, double alpha, const double* a, long lda,
          const double* b, long ldb, double beta, double* c, long ldc) {
    return cublasDgemm(g_handle, op(ta), op(tb), (int)m, (int)n, (int)k, &alpha, a, (int)lda, b, (int)ldb,
                       &beta, c, (int)ldc) == CUBLAS_STATUS_SUCCESS ? 0 : 3;
}
}  // namespace

extern "C" {

int ref_dcn_v2_forward_f64(const double* input, const double* weight, const double* bias, const double* ones,
                       const double* offset, const double* mask, double* output, double* columns,
                       int batch, int channels, int height, int width, int channels_out,
                       int kernel_h, int kernel_w, int stride_h, int stride_w, int pad_h, int pad_w,
                       int dilation_h, int dilation_w, int deformable_group, void* stream) {
    cudaStream_t s = (cudaStream_t)stream;
    if (int e = handle_for(s)) return e;
    const int height_out = (height + 2 * pad_h - (dilation_h * (kernel_h - 1) + 1)) / stride_h + 1;
    const int width_out = (width + 2 * pad_w - (dilation_w * (kernel_w - 1) + 1)) / stride_w + 1;
    const long in_n = (long)channels * height * width;
    const long off_n = (long)deformable_group * 2 * kernel_h * kernel_w * height_out * width_out;
    const long mask_n = off_n / 2;
    const long out_n = (long)channels_out * height_out * width_out;
    for (int b = 0; b < batch; b++) {
        double* output_n = output + b * out_n;
        {   // bias first: (N x 1)(1 x M)
            long m_ = channels_out, n_ = (long)height_out * width_out, k_ = 1;
            if (int e = dgemm('t', 'n', n_, m_, k_, 1.0, ones, k_, bias, k_, 0.0, output_n, n_)) return e;
        }
        modulated_deformable_im2col_cuda(s, input + b * in_n, offset + b * off_n, mask + b * mask_n, 1, channels,
                                         height, width, height_out, width_out, kernel_h, kernel_w, pad_h, pad_w,
                                         stride_h, stride_w, dilation_h, dilation_w, deformable_group, columns);
        long m = channels_out, n = (long)height_out * width_out, k = (long)channels * kernel_h * kernel_w;
        if (int e = dgemm('n', 'n', n, m, k, 1.0, columns, n, weight, k, 1.0, output_n, n)) return e;
    }
    return cudaGetLastError() == cudaSuccess ? 0 : 4;
}

int ref_dcn_v2_backward_f64(const double* input, const double* weight, const double* ones, const double* offset,
                        const double* mask, double* columns, double* grad_input, double* grad_weight,
                        double* grad_bias, double* grad_offset, double* grad_mask, const double* grad_output,
                        int batch, int channels, int height, int width, int channels_out,
                        int kernel_h, int kernel_w, int stride_h, int stride_w, int pad_h, int pad_w,
                        int dilation_h, int dilation_w, int deformable_group, void* stream) {
    cudaStream_t s = (cudaStream_t)stream;
    if (int e = handle_for(s)) return e;
    const int height_out = (height + 2 * pad_h - (dilation_h * (kernel_h - 1) + 1)) / stride_h + 1;
    const int width_out = (width + 2 * pad_w - (dilation_w * (kernel_w - 1) + 1)) / stride_w + 1;
    const long in_n = (long)channels * height * width;
    const long off_n = (long)deformable_group * 2 * kernel_h * kernel_w * height_out * width_out;
    const long mask_n = off_n / 2;
    const long out_n = (long)channels_out * height_out * width_out;
    for (int b = 0; b < batch; b++) {
        const double* grad_output_n = grad_output + b * out_n;
        long m = (long)channels * kernel_h * kernel_w, n = (long)height_out * width_out, k = channels_out;
        if (int e = dgemm('n', 't', n, m, k, 1.0, grad_output_n, n, weight, m, 0.0, columns, n)) return e;
        modulated_deformable_col2im_coord_cuda(s, columns, input + b * in_n, offset + b * off_n, mask + b * mask_n, 1,
                                               channels, height, width, height_out, width_out, kernel_h, kernel_w,
                                               pad_h, pad_w, stride_h, stride_w, dilation_h, dilation_w,
                                               deformable_group, grad_offset + b * off_n, grad_mask + b * mask_n);
        modulated_deformable_col2im_cuda(s, columns, offset + b * off_n, mask + b * mask_n, 1, channels, height,
                                         width, height_out, width_out, kernel_h, kernel_w, pad_h, pad_w, stride_h,
                                         stride_w, dilation_h, dilation_w, deformable_group, grad_input + b * in_n);
        modulated_deformable_im2col_cuda(s, input + b * in_n, offset + b * off_n, mask + b * mask_n, 1, channels,
                                         height, width, height_out, width_out, kernel_h, kernel_w, pad_h, pad_w,
                                         stride_h, stride_w, dilation_h, dilation_w, deformable_group, columns);
        long m_ = channels_out, n_ = (long)channels * kernel_h * kernel_w, k_ = (long)height_out * width_out;
        if (int e = dgemm('t', 'n', n_, m_, k_, 1.0, columns, k_, grad_output_n, k_, 1.0, grad_weight, n_)) return e;
        const double one = 1.0;
        if (cublasDgemv(g_handle, CUBLAS_OP_T, (int)k_, (int)m_, &one, grad_output_n, (int)k_, ones, 1, &one,
                        grad_bias, 1) != CUBLAS_STATUS_SUCCESS) return 5;
    }
    return cudaGetLastError() == cudaSuccess ? 0 : 4;
}

int ref_psroi_forward_f64(const double* input, const double* bbox, const double* trans, double* out, double* top_count,
                      int batch, int channels, int height, int width, int num_bbox, int channels_trans,
                      int no_trans, double spatial_scale, int output_dim, int group_size, int pooled_size,
                      int part_size, int sample_per_part, double trans_std, void* stream) {
    DeformablePSROIPoolForward((cudaStream_t)stream, input, bbox, trans, out, top_count, batch, channels, height,
                               width, num_bbox, channels_trans, no_trans, spatial_scale, output_dim, group_size,
                               pooled_size, part_size, sample_per_part, trans_std);
    return cudaGetLastError() == cudaSuccess ? 0 : 4;
}

int ref_psroi_backward_f64(const double* out_grad, const double* input, const double* bbox, const double* trans,
                       const double* top_count, double* input_grad, double* trans_grad, int batch, int channels,
                       int height, int width, int num_bbox, int channels_trans, int no_trans, double spatial_scale,
                       int output_dim, int group_size, int pooled_size, int part_size, int sample_per_part,
                       double trans_std, void* stream) {
    DeformablePSROIPoolBackwardAcc((cudaStream_t)stream, out_grad, input, bbox, trans, top_count, input_grad,
                                   trans_grad, batch, channels, height, width, num_bbox, channels_trans, no_trans,
                                   spatial_scale, output_dim, group_size, pooled_size, part_size, sample_per_part,
                                   trans_std);
    return cudaGetLastError() == cudaSuccess ? 0 : 4;
}

}  // extern "C"
