// conflux_b200/csrc/update.cu -- the trailing update of the factorisations (kernels.h TrailingUpdate): which kernel runs,
// and how its operands are split and its window launched.
#include <algorithm>

#include "kernels.h"

namespace cflx {

int TrailingUpdate::create(int rows, int cols, int K, bool int8) {
    this->rows = rows;
    this->cols = cols;
    this->K = K;
    if (int8) CFLX_TRY(ozaki_workspace_create(&oz, rows, cols, K));
    this->int8 = int8;
    return CFLX_OK;
}
int TrailingUpdate::with_tf32(int terms, const std::function<int()>& fn) {
    if (!tf.maps) CFLX_TRY(tf32_workspace_create(&tf, rows, cols, std::max(K, 1)));
    this->terms = terms;
    const int rc = fn();
    this->terms = 0;
    return rc;
}
int TrailingUpdate::split_a(const double* AT, int64_t ld, int n, cudaStream_t s) {
    if (terms) return tf32_split_a(&tf, terms, AT, ld, n, s);
    return int8 ? ozaki_split_a(&oz, AT, ld, n, s) : CFLX_OK;
}
int TrailingUpdate::split_b(const double* B, int64_t ld, int col0, int n, cudaStream_t s) {
    if (terms) return tf32_split_b(&tf, terms, B, ld, col0, n, s);
    return int8 ? ozaki_split_b(&oz, B, ld, col0, n, s) : CFLX_OK;
}
int TrailingUpdate::apply(const GemmArgs& g, int row0, int col0, int leave_sms, cudaStream_t s) {
    if (terms)
        return launch_tf32_gemm(&tf, terms, g.M, g.N, row0, col0, g.D, g.ldd, leave_sms > 0 ? tf.sms - leave_sms : 0, s);
    if (int8) return launch_ozaki_gemm(&oz, g.M, g.N, row0, col0, g.D, g.ldd, leave_sms > 0 ? oz.sms - leave_sms : 0, s);
    return launch_gemm_tn(g, s);
}

}  // namespace cflx
