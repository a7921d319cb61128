// C entry point of libmelgan_b200_simt_test.so: the first-generation fp32 SIMT generator (mg_gen_simt.cu), kept as an
// independent second implementation that tests cross-check the wgmma product path against.  TEST INFRASTRUCTURE: nothing
// in the product library or the package links or loads this; only tests/test_simt_crosscheck_gpu.py does.
#include "../mg_common.cuh"

using namespace mg;

extern "C" {

const char *mg_simt_last_error_string(void) { return error_buffer(); }

// packed: the blob written by the PRODUCT library's mg_gen_pack (the SIMT kernels read its fp32 region);
// workspace: mg_gen_workspace_bytes(B, T) bytes.  Asynchronous on `stream`.
int mg_simt_gen_forward(const void *packed, const float *mel, float *audio, int B, int T, void *workspace, void *stream) {
    if (!packed || !mel || !audio || !workspace || B < 1 || T < 1)
        return set_error(MG_ERR_INVALID_ARGUMENT, "mg_simt_gen_forward: bad argument");
    return launch_generator_simt((const float *)packed, mel, audio, B, T, (float *)workspace, (cudaStream_t)stream, nullptr);
}

}  // extern "C"
