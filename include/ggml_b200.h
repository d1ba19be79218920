/*
 * include/ggml_b200.h — the drop-in boundary: a ggml backend ("B200") that exposes the sm_90a kernels of
 * libprima_b200.so through the reference's own plugin interface, the C structs of function pointers in
 * ggml/src/ggml-backend-impl.h:15-220 (ggml_backend_reg_i / _device_i / _i / _buffer_type_i / _buffer_i).
 *
 * It replaces ggml_backend_cuda_reg() (ggml/src/ggml-cuda.cu:3302) for the decode hot path.  src/llama.cpp discovers GPUs
 * purely through the registry (src/llama.cpp:20443-20456, 21118-21127), so registering this reg before
 * llama_load_model_from_file makes the ggml scheduler place the ops listed under supports_op on the GPU and everything else
 * on the CPU backend — no change to llama.cpp, ggml-backend.cpp or the tests (tests/test-backend-ops.cpp enumerates the
 * registry, :3765-3861).
 *
 * The plugin is compiled against the HOST's ggml headers (prima.cpp_b200/ggml_backend/Makefile, -I<reference>/ggml/include
 * -I<reference>/ggml/src) and resolves ggml_* symbols from the host's libggml at load time, like any ggml backend.
 */
#ifndef GGML_B200_H
#define GGML_B200_H

#ifdef __cplusplus
extern "C" {
#endif

struct ggml_backend_reg;      /* ggml/src/ggml-backend-impl.h:209-216 */
struct ggml_backend;          /* ggml/src/ggml-backend-impl.h:128-133 */
struct ggml_backend_buffer_type;

/* the registry entry; replaces ggml_backend_cuda_reg (ggml-cuda.cu:3302-3340) */
__attribute__((visibility("default"))) struct ggml_backend_reg * ggml_backend_b200_reg(void);
/* convenience constructors mirroring ggml_backend_cuda_init / ggml_backend_cuda_buffer_type (ggml-cuda.h) */
__attribute__((visibility("default"))) struct ggml_backend * ggml_backend_b200_init(int device);
__attribute__((visibility("default"))) struct ggml_backend_buffer_type * ggml_backend_b200_buffer_type(int device);
__attribute__((visibility("default"))) int ggml_backend_is_b200(struct ggml_backend * backend);
/* number of graph nodes this backend has executed on the GPU since load (tests: proves the native path ran) */
__attribute__((visibility("default"))) unsigned long long ggml_backend_b200_nodes_computed(void);
/* number of fused launches graph_compute has issued (mat-vec groups with folded norm / silu / bias / residual, attention chains) */
__attribute__((visibility("default"))) unsigned long long ggml_backend_b200_fused_steps(void);
/* graph_compute calls served by replaying a captured CUDA graph (same topology and tensor addresses as an earlier call) */
__attribute__((visibility("default"))) unsigned long long ggml_backend_b200_graph_replays(void);

/* Loading the shared object registers the backend automatically (a constructor calls ggml_backend_register,
 * ggml-backend-impl.h:220) unless the environment variable GGML_B200_NO_AUTOREG is set. */

#ifdef __cplusplus
}
#endif
#endif
