// Decode of the two-layer decoder (EXTENSION, BASELINE.json configs[3]; semantics: oracle/ref_ext.py decoder2_forward without
// dropout): layer 1 is the torch flavour's attention LSTM, layer 2 nn.LSTMCell(D, D) over h1_t from a zero state, logits_t =
// fc(h2_t).  A third flavour of the shared decode loops (greedy_loop / beam_loop): TorchDecode's prologue, cell step and state
// gather, plus layer 2.  Part of the lo_decoder.cu translation unit, after lo_lstmseq.cuh; it adds no kernel: layer 2's cell is
// seq_lstm_pw_fwd_kernel, its state gather gather_rows_kernel, its products the step-GEMM dispatcher of layer 1.

namespace lo {

// layer 2's device scratch (lo_decoder2_layer.scratch): only the current state is kept, in two slots that alternate
struct Dec2Ws {
  float* gates;     // f32 [B][4D]  pre-activations, then activations (seq_lstm_pw_fwd_kernel)
  float* h;         // f32 [2][B][D]
  float* c;         // f32 [2][B][D]
  bf16* h_bf;       // bf16 [2][B][D]  mirror of h, the A operand of the tensor-core GEMMs
  float* bsum;      // f32 [4D] = b_ih + b_hh
  size_t bytes;
};

static Dec2Ws dec2_carve(void* base, int B, int D) {
  size_t off = 0;
  auto take = [&](size_t bytes) -> void* {
    void* p = base ? (char*)base + off : nullptr;
    off += (bytes + 255) & ~(size_t)255;
    return p;
  };
  const size_t n = (size_t)B * D;
  Dec2Ws w{};
  w.gates = (float*)take(4 * n * 4);
  w.h = (float*)take(2 * n * 4);
  w.c = (float*)take(2 * n * 4);
  w.h_bf = (bf16*)take(2 * n * 2);
  w.bsum = (float*)take((size_t)4 * D * 4);
  w.bytes = off;
  return w;
}

// the refusals of both two-layer entry points that concern the layer and the modes it does not support
static int check_decoder2(const lo_decoder_args* a, const lo_decoder2_layer* l2) {
  LO_CHECK_ARG(a, "null args");
  LO_CHECK_ARG(l2, "null lo_decoder2_layer");
  LO_CHECK_ARG(l2->w_ih && l2->w_hh && l2->b_ih && l2->b_hh && l2->scratch, "null layer-2 weight, bias or scratch");
  LO_CHECK_ARG(a->phase == 0, "the two-layer decode runs whole steps: phase must be 0");
  LO_CHECK_ARG(!a->ss_prob, "scheduled sampling (ss_prob) is a training mode: not available in the two-layer decode");
  return LO_OK;
}

// the two-layer decoder in the decode loops: TorchDecode for layer 1 (its next tokens, finished flags, parent rows and attention
// rows), then per step h1_t W_ih^T + b_ih + b_hh and += h2 W_hh^T on the step-GEMM dispatcher (one K slice each, as layer 1's
// forward step GEMMs: a bf16 decode repeats its bits), the cell, and the head on h2.  `s`: the slot holding the current h2, c2.
struct TwoLayerDecode : TorchDecode {
  const lo_decoder2_layer* l2;
  Dec2Ws w;
  int s = 0;
  TwoLayerDecode(const lo_decoder_args* a_, int64_t start, int32_t* finished, int32_t* parent_rows, const lo_decoder2_layer* l2_)
      : TorchDecode(a_, start, finished, parent_rows), l2(l2_), w(dec2_carve(l2_->scratch, d.B, d.D)) {}
  int prologue(cudaStream_t st) {
    LO_TRY(TorchDecode::prologue(st));
    seq_bias_sum_kernel<<<cdiv(d.G, 256), 256, 0, st>>>(l2->b_ih, l2->b_hh, w.bsum, d.G);
    LO_LAUNCH_OK();
    s = 0;
    seq_init_kernel<<<cdiv((long)d.B * d.D, 256), 256, 0, st>>>(nullptr, nullptr, w.h, w.c, bv.on ? w.h_bf : nullptr, d.B * d.D);
    LO_LAUNCH_OK();
    return LO_OK;
  }
  int step(int t, cudaStream_t st) {
    LO_TRY(forward_step(a, d, t, d.B, c.ragged(), c.next_tok, 1, nullptr, 0, nullptr, st));
    const int64_t n = (int64_t)d.B * d.D, h1 = (int64_t)(t + 1) * n, p = s * n, q = (1 - s) * n;
    LO_TRY(step_gemm_nt(bv.on, a->hall + h1, bv.on ? bv.hall + h1 : nullptr, d.D, l2->w_ih, a->dt, d.D, w.gates, d.G, d.B, d.G, d.D,
                        w.bsum, 0, 1, 0, st));
    LO_TRY(step_gemm_nt(bv.on, w.h + p, bv.on ? w.h_bf + p : nullptr, d.D, l2->w_hh, a->dt, d.D, w.gates, d.G, d.B, d.G, d.D, nullptr,
                        1, 1, 1, st));
    LO_CUDA(launch_pdl(seq_lstm_pw_fwd_kernel, dim3(cdiv((long)n, 256)), dim3(256), (size_t)0, st, w.gates, (const float*)(w.c + p),
                       w.c + q, w.h + q, bv.on ? w.h_bf + q : (bf16*)nullptr, (float*)nullptr, (void*)nullptr, 0, (int64_t)0, d.B, d.D));
    LO_LAUNCH_OK();
    s = 1 - s;
    return head_nt(a, bv.on, w.h + q, bv.on ? w.h_bf + q : nullptr, d.D, a->logits, d.V, d.B, st);
  }
  // layer 1's gather, then h2 (with its bf16 mirror) and c2 by parents from the current slot into the other one
  int reorder(int t, cudaStream_t st) {
    LO_TRY(TorchDecode::reorder(t, st));
    const int64_t n = (int64_t)d.B * d.D, p = s * n, q = (1 - s) * n;
    gather_rows_kernel<<<cdiv((long)n, 256), 256, 0, st>>>(w.h + p, c.parent_rows, w.h + q, bv.on ? w.h_bf + q : nullptr, d.B, d.D);
    LO_LAUNCH_OK();
    gather_rows_kernel<<<cdiv((long)n, 256), 256, 0, st>>>(w.c + p, c.parent_rows, w.c + q, nullptr, d.B, d.D);
    LO_LAUNCH_OK();
    s = 1 - s;
    return LO_OK;
  }
};

}  // namespace lo

using namespace lo;

extern "C" {

int64_t lo_sizeof_decoder2_layer(void) { return (int64_t)sizeof(lo_decoder2_layer); }

int64_t lo_decoder2_scratch_bytes(const lo_decoder_args* a) {
  if (!a || a->B < 1 || a->D < 1) return 0;
  return (int64_t)dec2_carve(nullptr, a->B, a->D).bytes;
}

int lo_decoder2_greedy(const lo_decoder_args* a, const lo_decoder2_layer* l2, int64_t start_id, int64_t end_id, int max_steps,
                       int64_t* tokens, int32_t* finished, int32_t* fin_hist, void* stream) {
  LO_TRY(check_decoder2(a, l2));
  LO_TRY(check_args(a));
  LO_TRY(check_reg_off(a, true));
  TwoLayerDecode f(a, start_id, finished, nullptr, l2);
  return greedy_loop(f, end_id, max_steps, tokens, fin_hist, (cudaStream_t)stream);
}

int lo_decoder2_sample(const lo_decoder_args* a, const lo_decoder2_layer* l2, const lo_sample_args* s, int64_t start_id, int64_t end_id,
                       int max_steps, int64_t* tokens, int32_t* finished, int32_t* fin_hist, void* stream) {
  LO_TRY(check_decoder2(a, l2));
  LO_TRY(check_decoder_sample(a, s));
  TwoLayerDecode f(a, start_id, finished, nullptr, l2);
  return sample_loop(f, s, end_id, max_steps, tokens, fin_hist, (cudaStream_t)stream);
}

int lo_decoder2_beam(const lo_decoder_args* a, const lo_decoder2_layer* l2, int64_t start_id, int64_t end_id, int max_steps,
                     int64_t* ids, int64_t* parents, int32_t* fin_hist, float* logp, float div_gamma, float div_prob,
                     const float* div_u, const uint64_t* div_state, const lo_beam_penalty* pen, void* stream) {
  const BeamArgs bm{0, div_gamma, div_prob, div_u, div_state, pen};
  LO_TRY(check_decoder2(a, l2));
  if (pen) LO_TRY(check_beam_penalty(pen, a->rows_per_img, a->V, bm.div_on()));
  return decoder_beam<TwoLayerDecode>(a, start_id, end_id, max_steps, ids, parents, fin_hist, logp, bm, nullptr, stream, l2);
}

int lo_decoder2_greedy_brackets(const lo_decoder_args* a, const lo_decoder2_layer* l2, int64_t start_id, int64_t end_id, int max_steps,
                                int64_t* tokens, int32_t* finished, int32_t* fin_hist, const lo_bracket_rule* br, void* stream) {
  LO_TRY(check_decoder2(a, l2));
  LO_TRY(check_args(a));
  LO_TRY(check_bracket_rule(br, a->V));
  LO_TRY(check_reg_off(a, true));
  TwoLayerDecode f(a, start_id, finished, nullptr, l2);
  return greedy_loop(f, end_id, max_steps, tokens, fin_hist, (cudaStream_t)stream, ArgmaxChoice{}, br);
}

int lo_decoder2_sample_brackets(const lo_decoder_args* a, const lo_decoder2_layer* l2, const lo_sample_args* s, int64_t start_id,
                                int64_t end_id, int max_steps, int64_t* tokens, int32_t* finished, int32_t* fin_hist,
                                const lo_bracket_rule* br, void* stream) {
  LO_TRY(check_decoder2(a, l2));
  LO_TRY(check_decoder_sample(a, s));
  LO_TRY(check_bracket_rule(br, a->V));
  TwoLayerDecode f(a, start_id, finished, nullptr, l2);
  return sample_loop(f, s, end_id, max_steps, tokens, fin_hist, (cudaStream_t)stream, br);
}

int lo_decoder2_beam_brackets(const lo_decoder_args* a, const lo_decoder2_layer* l2, int64_t start_id, int64_t end_id, int max_steps,
                              int64_t* ids, int64_t* parents, int32_t* fin_hist, float* logp, float div_gamma, float div_prob,
                              const float* div_u, const uint64_t* div_state, const lo_beam_penalty* pen, const lo_bracket_rule* br,
                              void* stream) {
  const BeamArgs bm{0, div_gamma, div_prob, div_u, div_state, pen};
  LO_TRY(check_decoder2(a, l2));
  LO_TRY(check_bracket_rule(br, a->V));
  if (pen) LO_TRY(check_beam_penalty(pen, a->rows_per_img, a->V, bm.div_on()));
  return decoder_beam<TwoLayerDecode>(a, start_id, end_id, max_steps, ids, parents, fin_hist, logp, bm, br, stream, l2);
}

}  // extern "C"
