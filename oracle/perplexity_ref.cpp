// oracle/perplexity_ref.cpp — llama-perplexity's log-probability writer and KL-divergence functions as a CPU oracle (test infrastructure
// only; never linked by the product).
//
// The reference's examples/perplexity/perplexity.cpp is included UNMODIFIED from where it lies under $(REF); its main() becomes an unused
// static function, so nothing of libllama / common is linked (Makefile.perplexity: -Wl,--no-undefined).  The wrappers below export both
// log_softmax overloads that llama-perplexity's --kl-divergence-base / --kl-divergence modes call, and both process_logits drivers with no
// worker threads (the serial order of the reference's sums).
#define main static ref_perplexity_main
#include "examples/perplexity/perplexity.cpp"
#undef main

#include <sstream>

extern "C" {

// log_softmax(n_vocab, logits, uint16_t * log_prob, tok): one record of 2*((n_vocab+1)/2) + 4 uint16 (the caller zero-fills it, as the
// reference's buffer is); returns nll = max + log(sum) - logits[tok] as the reference computes it (float, widened)
double ppl_ref_logprobs_u16(int n_vocab, const float * logits, uint16_t * record, int tok) {
    return log_softmax(n_vocab, logits, record, tok);
}

// log_softmax(n_vocab, logits, base_log_prob, tok, kld): adds one row to the accumulated sums in acc (kl_divergence_result's layout:
// 10 doubles, then float max_p_diff, then size_t n_same_top and count), returns the row's KLD and writes its p_diff
double ppl_ref_kld(int n_vocab, const float * logits, const uint16_t * base, int tok, kl_divergence_result * acc, float * p_diff) {
    const std::pair<double, float> r = log_softmax(n_vocab, logits, base, tok, *acc);
    *p_diff = r.second;
    return r.first;
}

int ppl_ref_result_bytes(void) { return (int) sizeof(kl_divergence_result); }

// the writer's process_logits: n_token rows of logits scored against tokens[1..n_token]; records [n_token][nv] as it writes them to the
// base file, nll / nll2 accumulated
void ppl_ref_process_logits_u16(int n_vocab, const float * logits, const int * tokens, int n_token, uint16_t * records, double * nll,
                                double * nll2) {
    std::vector<std::thread> workers;
    const int nv = 2*((n_vocab + 1)/2) + 4;
    std::vector<uint16_t> log_probs((size_t) n_token * nv);
    std::ostringstream out;
    process_logits(out, n_vocab, logits, tokens, n_token, workers, log_probs, *nll, *nll2);
    const std::string s = out.str();
    std::memcpy(records, s.data(), s.size());
}

// the compare mode's process_logits: n_token rows against base records [n_token][nv]; sums into acc, per-row KLD and p_diff
void ppl_ref_process_logits_kld(int n_vocab, const float * logits, const int * tokens, int n_token, const uint16_t * base,
                                kl_divergence_result * acc, float * kld_values, float * p_diff_values) {
    std::vector<std::thread> workers;
    const int nv = 2*((n_vocab + 1)/2) + 4;
    const std::vector<uint16_t> base_log_probs(base, base + (size_t) n_token * nv);
    process_logits(n_vocab, logits, tokens, n_token, workers, base_log_probs, *acc, kld_values, p_diff_values);
}

}  // extern "C"
