// oracle/sampling_stubs.cpp — the few libllama / ggml symbols the reference's src/llama-sampling.cpp (and the grammar / vocab
// units it pulls in) link against, so its sampler chain can run on its own as a CPU oracle (oracle/_ref/libsampling_ref.so).
// The chain is driven through llama_sampler_apply on a caller-built llama_token_data_array; the logits / model accessors below
// are only reached by llama_sampler_sample, which the tests never call.
#include <cstdarg>
#include <cstdio>
#include <cstdlib>

#include "ggml.h"
#include "llama.h"

extern "C" {
void ggml_abort(const char * file, int line, const char * fmt, ...) {
    fprintf(stderr, "%s:%d: ", file, line);
    va_list ap;
    va_start(ap, fmt);
    vfprintf(stderr, fmt, ap);
    va_end(ap);
    fputc('\n', stderr);
    abort();
}
int64_t ggml_time_us(void) { return 0; }
struct llama_sampler_chain_params llama_sampler_chain_default_params(void) { return {/* .no_perf = */ true}; }
float * llama_get_logits_ith(struct llama_context *, int32_t) { return nullptr; }
const struct llama_model * llama_get_model(const struct llama_context *) { return nullptr; }
int32_t llama_n_vocab(const struct llama_model *) { return 0; }
}

void llama_log_internal(ggml_log_level, const char *, ...) {}
