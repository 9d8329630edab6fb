// C-ABI dispatcher for the correlation-volume build (see include/macvo_b200.h).
#include "common.cuh"

int macvo_corr_build_simt(const float* f1, const float* f2, float* corr, int batch, int dim, int n, cudaStream_t st);
size_t macvo_corr_tc_workspace_bytes(int batch, int dim, int n, int passes);
int macvo_corr_build_tc(const float* f1, const float* f2, float* corr, int batch, int dim, int n, int passes, int kmajor,
                        void* workspace, size_t workspace_bytes, cudaStream_t st);

extern "C" const char* macvo_b200_version(void) { return "macvo_b200 0.1.0 sm_90a"; }

extern "C" size_t macvo_corr_workspace_bytes(int batch, int dim, int n, int mode) {
    if (batch <= 0 || dim <= 0 || n <= 0) return 0;
    mode &= ~MACVO_CORR_KMAJOR_INPUT;
    if (mode == MACVO_CORR_TC_3XF16) return macvo_corr_tc_workspace_bytes(batch, dim, n, 3);
    if (mode == MACVO_CORR_TC_1XF16) return macvo_corr_tc_workspace_bytes(batch, dim, n, 1);
    return 0;
}

extern "C" int macvo_corr_build(const float* fmap1, const float* fmap2, float* corr, int batch, int dim, int n,
                                int mode, void* workspace, size_t workspace_bytes, void* stream) {
    if (!fmap1 || !fmap2 || !corr || batch <= 0 || dim <= 0 || n <= 0) return MACVO_E_ARG;
    cudaStream_t st = as_stream(stream);
    const int kmajor = (mode & MACVO_CORR_KMAJOR_INPUT) != 0;
    switch (mode & ~MACVO_CORR_KMAJOR_INPUT) {
        case MACVO_CORR_SIMT: return kmajor ? MACVO_E_UNSUPPORTED : macvo_corr_build_simt(fmap1, fmap2, corr, batch, dim, n, st);
        case MACVO_CORR_TC_3XF16: return macvo_corr_build_tc(fmap1, fmap2, corr, batch, dim, n, 3, kmajor, workspace, workspace_bytes, st);
        case MACVO_CORR_TC_1XF16: return macvo_corr_build_tc(fmap1, fmap2, corr, batch, dim, n, 1, kmajor, workspace, workspace_bytes, st);
        case MACVO_CORR_TC_TF32: return kmajor ? macvo_corr_build_tc(fmap1, fmap2, corr, batch, dim, n, 2, 1, nullptr, 0, st)
                                               : MACVO_E_UNSUPPORTED;       // reads the fp32 K-major features in place
        default: return MACVO_E_ARG;
    }
}
