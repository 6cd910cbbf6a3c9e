// stop.cu -- stop strings of generate() on the device: transformers' StopStringCriteria, per row, as one table lookup
// at the end of the graphed decode step.  All string work happens once on the host (engine.StopStrings): an
// Aho-Corasick automaton over the characters of the stop strings, folded with the tokenizer's clean token strings into a
// dense table step[V_tok + 1, S] -- entry (t, s) is the automaton state after token t's string is fed from state s, bit
// 15 set when an occurrence of a stop string ended on the way.  Here each row advances its state by the token the
// sampler has just written and sets its `finished` flag on a hit; the sampler's eos -> pad rule reads that flag on the
// next step.  Integer only, so there is no fp16 twin.
#include "common.cuh"

namespace g4r {

__global__ void stop_step_kernel(const long long* __restrict__ ids, const short* __restrict__ step, long long ld,
                                 int V_tok, int B, int* __restrict__ state, int* __restrict__ finished) {
  const int b = blockIdx.x * blockDim.x + threadIdx.x;
  if (b >= B || finished[b]) return;
  const long long tok = ids[b];
  const long long row = tok < 0 || tok > V_tok ? V_tok : tok;   // ids the tokenizer does not hold: the reset row
  const int e = step[row * ld + state[b]];
  state[b] = e & 0x7FFF;
  if (e < 0) finished[b] = 1;
}

// The per-row form (g4r_stop_step_rows): a continuous batch, whose rows are independent requests, each with its own
// table (null: no stop strings) of S[b] states.  One tokenizer per batch, so V_tok is shared.
__global__ void stop_step_rows_kernel(const long long* __restrict__ ids, const short* const* __restrict__ tables,
                                      const int* __restrict__ S, int V_tok, int B, const int* __restrict__ active,
                                      int* __restrict__ state, int* __restrict__ finished) {
  const int b = blockIdx.x * blockDim.x + threadIdx.x;
  if (b >= B || !active[b] || finished[b]) return;
  const short* step = tables[b];
  if (!step) return;
  const long long tok = ids[b];
  const long long row = tok < 0 || tok > V_tok ? V_tok : tok;
  const int e = step[row * S[b] + state[b]];
  state[b] = e & 0x7FFF;
  if (e < 0) finished[b] = 1;
}

}  // namespace g4r

using namespace g4r;

extern "C" int g4r_stop_step(const long long* ids, const short* step, long long ld, int V_tok, int S, int B, int* state,
                             int* finished, void* stream) {
  G4R_REQUIRE(ids && step && state && finished, "stop_step: null pointer");
  G4R_REQUIRE(B > 0 && S >= 1 && S <= 32767 && V_tok > 0 && ld >= S,
              "stop_step: bad arguments (B=%d S=%d V_tok=%d ld=%lld; S must be 1..32767)", B, S, V_tok, ld);
  stop_step_kernel<<<(B + 127) / 128, 128, 0, (cudaStream_t)stream>>>(ids, step, ld, V_tok, B, state, finished);
  G4R_LAUNCH_CHECK("stop_step");
  return G4R_OK;
}

extern "C" int g4r_stop_step_rows(const long long* ids, const short* const* tables, const int* S, int V_tok, int B,
                                  const int* active, int* state, int* finished, void* stream) {
  G4R_REQUIRE(ids && tables && S && active && state && finished, "stop_step_rows: null pointer");
  G4R_REQUIRE(B > 0 && V_tok > 0, "stop_step_rows: bad arguments (B=%d V_tok=%d)", B, V_tok);
  stop_step_rows_kernel<<<(B + 127) / 128, 128, 0, (cudaStream_t)stream>>>(ids, tables, S, V_tok, B, active, state,
                                                                            finished);
  G4R_LAUNCH_CHECK("stop_step_rows");
  return G4R_OK;
}
