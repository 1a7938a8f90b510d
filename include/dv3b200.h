/* dv3b200 -- C ABI of the H100-native hot path of r9y9/deepvoice3_pytorch.
 *
 * The reference has no FFI of its own (it is pure Python on ATen): the seam it offers is the Python
 * module API (deepvoice3_pytorch.builder.* -> nn.Module, SURVEY.md section 8b).  This header is the
 * C-ABI layer underneath our mirror of that API; each entry point names the reference code whose GPU
 * work (ATen/cuDNN/cuBLAS calls) it replaces.  See INTEGRATION.md for the reference-side binding.
 *
 * Conventions
 *   - every function returns 0 on success, non-zero on failure; dv3_last_error() gives the message of the
 *     most recent failure on the calling thread.  No exceptions, no torch types.
 *   - all pointers are caller-owned DEVICE memory (fp32 unless stated), densely packed, row-major with the
 *     last index fastest; kernels never allocate.  `stream` is a cudaStream_t; every call is asynchronous on
 *     it and re-entrant (no global mutable state besides cached device attributes).
 *   - activations use the reference's conv layout (B, C, T), T fastest.
 *   - dropout: keep(i) is a pure function of (*seed_ptr, salt, element index i); `seed_ptr` points to 8
 *     bytes of device memory (so a captured CUDA graph gets fresh masks by bumping it), `salt` identifies the
 *     call site.  p_drop == 0 or seed_ptr == NULL disables it.
 *   - tensors must have fewer than 2^31 elements.
 */
#ifndef DV3B200_H
#define DV3B200_H

#ifdef __cplusplus
extern "C" {
#endif

const char* dv3_last_error(void);
int dv3_abi_version(void);
/* number of kernels this library has launched in this process (every launch is counted once) */
long long dv3_launch_count(void);

/* ---- weight normalisation: reference modules.py:85,100,109 (nn.utils.weight_norm pre-hook) -------------
 * v is [R][X][k] (k fastest), g is [R]; w = g*v/||v[r]||.  Writes w in up to two packed layouts:
 * out1[r*s1r + x*s1x + j*s1j] and out2[r*s2r + x*s2x + j*s2j] (either may be NULL).
 * inv_norm, scale: [R] outputs (1/||v||, g/||v||), inv_norm is needed by the backward. */
int dv3_weightnorm_fwd(const float* v, const float* g, float* inv_norm, float* scale, float* out1,
                       float* out2, int R, int X, int k, long long s1r, long long s1x, long long s1j,
                       long long s2r, long long s2x, long long s2j, void* stream);
/* dw_partials: [nsplit][R*X*k] partial gradients w.r.t. w (summed here; slot 0 is overwritten with the sum), in
 * v's own layout (r,x,j) when tap_major = 0 or as [j][r][x] when tap_major = 1; outputs dv [R][X][k], dg [R],
 * overwritten (accumulate = 0) or added to (accumulate = 1, e.g. straight into a flat gradient arena). */
int dv3_weightnorm_bwd(float* dw_partials, long long split_stride, int nsplit, int tap_major, const float* v,
                       const float* g, const float* inv_norm, float* dv, float* dg, int R, int X, int k,
                       int accumulate, void* stream);

/* ---- fused ConvBlock forward: reference modules.py:145-164 (Conv1dGLU._forward, mode 0) and
 * modules.py:200-226 (HighwayConv1d._forward, mode 1).
 * x (B,C,T); w_f packed [k][C][2C]; bias [2C]; spk (B,C,T) = softsign(speaker_proj(.)) transposed, or NULL;
 * y (B,C,T); save_a / save_s (B,C,T) = gate pre-activation a(+bias+spk) and sigmoid(b) for the backward, or NULL.
 * causal: left pad (k-1)*dilation; else symmetric (k-1)/2*dilation. Dropout is applied to the conv input only. */
int dv3_convblock_fwd(const float* x, const float* w_f, const float* bias, const float* spk, float* y,
                      float* save_a, float* save_s, int B, int C, int T, int k, int dilation, int causal,
                      int mode, int residual, float p_drop, const unsigned long long* seed_ptr,
                      unsigned salt, void* stream);
/* gate backward: dab (B,2C,T) = [d a ; d b], dbias[2C] += row sums (may be NULL). x only read in mode 1. */
int dv3_convblock_gate_bwd(const float* dy, const float* a, const float* s, const float* x, float* dab,
                           float* dbias, int B, int C, int T, int mode, int residual, void* stream);

/* ---- plain weight-normed Conv1d (+ fused ReLU): reference conv.py:7-15 via modules.py:94-100.
 * x (B,Cin,T); w_f packed [k][Cin][Cout]; y (B,Cout,T). */
int dv3_conv1d_fwd(const float* x, const float* w_f, const float* bias, float* y, int B, int Cin, int Cout,
                   int T, int k, int dilation, int causal, int relu, void* stream);
/* data gradient of a conv with M output rows: dx (B,Cin,T) = mask * convT(dab (B,M,T), w_b [k][M][Cin]) + addend.
 * mask = the forward's input-dropout mask (same seed/salt).  addmode 0: none; 1: + alpha*e1; 2: + e1*(1-e2)
 * (e1, e2 (B,Cin,T)) -- the residual-path gradients of the GLU / highway blocks. */
int dv3_conv1d_dgrad(const float* dab, const float* w_b, float* dx, int B, int M, int Cin, int T, int k,
                     int dilation, int causal, float p_drop, const unsigned long long* seed_ptr,
                     unsigned salt, int addmode, const float* e1, const float* e2, float alpha,
                     void* stream);
/* weight gradient, split over (b,t): writes dv3_conv1d_wgrad_nsplit(...) partials of `split_stride` floats each;
 * element (m, ci, j) of a partial lives at (m%msplit)*s_m + (m/msplit)*s_mh + ci*s_n + j*s_j. */
int dv3_conv1d_wgrad_nsplit(int B, int M, int Cin, int T, int k);
int dv3_conv1d_wgrad(const float* dab, const float* x, float* dw_partials, long long split_stride, int B,
                     int M, int Cin, int T, int k, int dilation, int causal, float p_drop,
                     const unsigned long long* seed_ptr, unsigned salt, int msplit, int s_m, int s_mh,
                     int s_n, int s_j, void* stream);
/* dyr = relu ? dy*(y>0) : (untouched); dbias[C] += sum_{b,t} dyr.  dy,y,dyr (B,C,T). */
int dv3_bias_act_bwd(const float* dy, const float* y, float* dyr, float* dbias, int B, int C, int T,
                     int relu, void* stream);

/* ---- layout change (B,R,C) -> (B,C,R): every x.transpose(1,2) between the attention (B,T,C) and conv (B,C,T)
 * layouts, reference deepvoice3.py:86,93,318,324,340-345,355,359,592,602; nyanko.py:66,206,214-217,230,234,402. */
int dv3_transpose(const float* in, float* out, int B, int R, int C, void* stream);

/* ---- embedding lookup: reference deepvoice3.py:74, nyanko.py:64,201-203,__init__.py:69-71 (F.embedding).
 * ids int64 [N] -> out (N,D); an id outside [0,V) sets *err_flag (device int) to 1 and writes nothing.
 * bwd: dtable[ids[n]] += dy[n] except rows == padding_idx (pass -1 for none); dtable must be pre-zeroed. */
int dv3_embedding_fwd(const long long* ids, const float* table, float* out, int N, int D, int V, int* err_flag,
                      void* stream);
int dv3_embedding_bwd(const long long* ids, const float* dy, float* dtable, int N, int D, int V,
                      long long padding_idx, void* stream);

/* ---- sinusoidal position encoding: reference modules.py:27-31,45-64 (SinusoidalEncoding.forward).
 * pos int64 (B,T) in [0,P); table (P,D) raw (non-sinusoidal) table; w [nw] position rate(s), nw in {1,B};
 * out (B,T,D).  bwd accumulates into pre-zeroed dtable (P,D) and dw [nw] (either may be NULL). */
int dv3_sinusoid_fwd(const long long* pos, const float* table, const float* w, int nw, float* out, int B, int T,
                     int D, int P, int* err_flag, void* stream);
int dv3_sinusoid_bwd(const long long* pos, const float* table, const float* w, int nw, const float* dy,
                     float* dtable, float* dw, int B, int T, int D, int P, void* stream);

/* ---- standalone dropout y = x*mask/(1-p): reference F.dropout at deepvoice3.py:75,80,294,321,588,597.
 * Calling it on the gradient with the same (seed, salt) is the backward. */
int dv3_dropout(const float* x, float* y, long long n, float p, const unsigned long long* seed_ptr, unsigned salt,
                void* stream);

/* ---- masked row softmax + dropout: reference deepvoice3.py:145-148,161-165.
 * s (rows,L); mask (rows/rows_per_b, L) bytes, 1 = padding (-inf), or NULL; probs = softmax (the returned
 * alignment); pd = dropout(probs) (may be NULL).  bwd: ds = P*(g - <g,P>), g = dpd*dropmask + dprobs_ext.
 * One warp per row.  Refused before any launch (return 1): rows < 1, L < 1, rows > INT_MAX / 32, rows_per_b < 1,
 * and, with a mask, rows % rows_per_b != 0.  A row whose keys are all masked is outside the contract. */
int dv3_softmax_fwd(const float* s, const unsigned char* mask, float* probs, float* pd, int rows, int L,
                    int rows_per_b, float p, const unsigned long long* seed_ptr, unsigned salt, void* stream);
int dv3_softmax_bwd(const float* probs, const float* dpd, const float* dprobs_ext, float* ds, int rows, int L,
                    float p, const unsigned long long* seed_ptr, unsigned salt, void* stream);

/* ---- ConvTranspose1d(k=2,s=2) time interleave: reference deepvoice3.py:519,527; nyanko.py:372,377.
 * in (B,2C,T) rows ordered (j,co) -> out (B,C,2T), out[b,co,2t+j] = in[b,j*C+co,t]; inverse=1 undoes it. */
int dv3_interleave2(const float* in, float* out, int B, int C, int T, int inverse, void* stream);

/* ---- length mask of a padded batch (batched synthesis): y = x, with y[b,:,t] = 0 for t >= mult*lengths[b].
 * x, y (B,C,T); x == y allowed; lengths int64 [B] on the device.  Zeroing a row's frames past its end before every
 * conv that mixes time steps makes each row see exactly the zero padding it would see alone. */
int dv3_mask_time(const float* x, float* y, const long long* lengths, int mult, int B, int C, int T, void* stream);
/* y = x with y[b,:,t] = 0 for t >= mult * extent[0] in every row: the logical time extent (int64 in device memory) of a
 * training batch padded to a bucket shape.  The mask is its own adjoint: the same call is its backward. */
int dv3_mask_frames(const float* x, float* y, const long long* extent, int mult, int B, int C, int T, void* stream);

/* ---- batched strided GEMM C[b] = alpha*A_b*B_b (+C): the attention contractions, reference
 * deepvoice3.py:143 (bmm(q,k)), :167 (bmm(p,v)) and their gradients.  A_b(m,k)=A[b*sAb+m*sAm+k*sAk],
 * B_b(k,n)=B[b*sBb+k*sBk+n*sBn], C_b(m,n)=C[b*sCb+m*ldc+n]; each operand needs one unit stride. */
int dv3_bgemm(const float* A, long long sAb, long long sAm, long long sAk, const float* B, long long sBb,
              long long sBk, long long sBn, float* C, long long sCb, int ldc, int batch, int M, int N, int K,
              float alpha, int accumulate, void* stream);
/* the same with alpha = Ts*sqrt(1/Ts), the attention context scale, of the key count ts_log[0] in device memory */
int dv3_bgemm_ctx_scale(const float* A, long long sAb, long long sAm, long long sAk, const float* B, long long sBb,
                        long long sBk, long long sBn, float* C, long long sCb, int ldc, int batch, int M, int N, int K,
                        const long long* ts_log, int accumulate, void* stream);

/* ---- fused tensor-core attention (wgmma, split-bf16 operands staged and split in-kernel): reference
 * deepvoice3.py:132-176 between the projections.  q (B,E,Td), k / v (B,E,Ts), mask (B,Ts) bytes (1 = padding) or
 * null -> probs (B,Td,Ts) = softmax(q^T k) (pre-dropout, returned as the alignment), out (B,E,Td) =
 * scale * v . dropout(probs)^T.  Backward: dout (B,E,Td), dprobs (B,Td,Ts) gradient arriving at the returned
 * probabilities (or null) -> dq, dk, dv; ds is a (B,Td,Ts) scratch.  Shapes: dv3_tc_attn_supported (Ts <= 128,
 * E % 16 == 0, E <= 256); others go through dv3_bgemm + dv3_softmax_*. */
int dv3_tc_attn_supported(int B, int E, int Td, int Ts);
int dv3_tc_attn_fwd(const float* q, const float* k, const float* v, const unsigned char* mask, float* probs,
                    float* out, int B, int E, int Td, int Ts, float scale, float p_drop,
                    const unsigned long long* seed_ptr, unsigned salt, void* stream);
int dv3_tc_attn_bwd(const float* dout, const float* q, const float* k, const float* v, const float* probs,
                    const float* dprobs, float* ds, float* dq, float* dk, float* dv, int B, int E, int Td, int Ts,
                    float scale, float p_drop, const unsigned long long* seed_ptr, unsigned salt, void* stream);
/* the same with scale = Ts*sqrt(1/Ts) of the logical key count ts_log[0] in device memory (a padded bucket batch) */
int dv3_tc_attn_fwd_ext(const float* q, const float* k, const float* v, const unsigned char* mask, float* probs,
                        float* out, int B, int E, int Td, int Ts, const long long* ts_log, float p_drop,
                        const unsigned long long* seed_ptr, unsigned salt, void* stream);
int dv3_tc_attn_bwd_ext(const float* dout, const float* q, const float* k, const float* v, const float* probs,
                        const float* dprobs, float* ds, float* dq, float* dk, float* dv, int B, int E, int Td, int Ts,
                        const long long* ts_log, float p_drop, const unsigned long long* seed_ptr, unsigned salt,
                        void* stream);

/* ---- optimizer step over a flat fp32 arena: reference train.py:756-759 (clip_grad_norm_ + Adam.step).
 * dv3_sumsq: out[0] = sum(x^2), deterministic (per-block partials in `scratch`, summed in index order by the block
 * that finishes last: bit-identical on every data-parallel replica); scratch = dv3_sumsq_scratch_floats() floats,
 * zero-filled once by the caller.  dv3_adam_clip: g' = g*hyper[3]*min(1, max_norm/(||g*hyper[3]||+1e-6))
 * (max_norm <= 0: no clipping), then torch.optim.Adam's update with lr=hyper[0], bias corrections hyper[1], hyper[2].
 * hyper (4 floats) and sumsq live in device memory: no host sync, graph-replayable. */
int dv3_sumsq_scratch_floats(void);
int dv3_sumsq(const float* x, long long n, float* out, float* scratch, void* stream);
int dv3_adam_clip(float* p, const float* g, float* m, float* v, long long n, const float* hyper,
                  const float* sumsq, float beta1, float beta2, float eps, float max_norm, void* stream);
/* dv3_adam_clip_opts: dv3_adam_clip with torch.optim.Adam's other two settings.  weight_decay > 0: L2 decay, the
 * clipped gradient becomes g' + weight_decay*p before the moments.  vmax != NULL: AMSGrad, vmax = max(vmax, v) and
 * the denominator is sqrt(vmax)/sqrt(hyper[2]) + eps.  weight_decay = 0 and vmax = NULL is dv3_adam_clip.  sumsq may
 * cover a larger arena than [p, p+n): a caller whose arena parts have different step counts runs one update per
 * part, each with its own hyper block, after one dv3_sumsq over the whole arena. */
int dv3_adam_clip_opts(float* p, const float* g, float* m, float* v, float* vmax, long long n, const float* hyper,
                       const float* sumsq, float beta1, float beta2, float eps, float max_norm, float weight_decay,
                       void* stream);

/* ---- fused STFT -> linear + mel front-end: reference audio.py:31-34 (spectrogram) and :46-51 (melspectrogram)
 * incl. preemphasis (:21-23), lws sqrt-Hann STFT 1024/256 with 768-sample zero padding (:54-55), mel basis product
 * (:64-68), dB (:79-81) and normalisation (:88-89).  wav (nclips, max_len) fp32; lengths int32 [nclips];
 * mel_basis (n_mels, 513) dense with mel_start/mel_len [n_mels] giving each filter's non-zero span;
 * linear (nclips, max_frames, 513) and mel (nclips, max_frames, n_mels) -- the transposed (T, F) layout the
 * preprocessors store (ljspeech.py:72-73); either output may be NULL.  Frames >= a clip's own count are zero-filled (outputs need no
 * initialisation); n_mels <= 128; min_level_db < 0.  Fastest when wav is 16-byte aligned and max_len % 4 == 0 (bulk /
 * 16-byte staging copies; any other pitch works through 4-byte copies, bit-identical results).  The first call on a
 * device builds a 2.7 KB table with a one-off kernel on the given stream (synchronised unless the stream is capturing). */
int dv3_stft_num_frames(int n_samples);
int dv3_stft_mel(const float* wav, const int* lengths, const float* mel_basis, const int* mel_start,
                 const int* mel_len, float* linear, float* mel, int nclips, int max_len, int max_frames,
                 int n_mels, float preemph, float min_level_db, float ref_level_db, void* stream);
/* The same transform written straight into a training batch's target layout (data.collate after the preprocessing
 * pass): linear (nclips, T_lin, 513) holds clip c's frame f at row lead + f; mel (nclips, ceil(T_lin / downsample_step),
 * n_mels) holds it at row (lead + f) / downsample_step when (lead + f) % downsample_step == 0; every other row of both
 * is written as zero.  Frames computed per clip: at most T_lin - lead.  wav (nclips, max_len) is fp32 or, with
 * wav_int16 != 0, int16 PCM read as x / 32768 (fast staging when 16-byte aligned and max_len % 8 == 0).  peak != NULL
 * (nclips floats on the device, dv3_peak_abs_batched) rescales each clip to x / peak * rescaling_max in fp32.  With
 * lead = 0, downsample_step = 1, T_lin = max_frames and fp32 input this is dv3_stft_mel.  No host synchronisation. */
int dv3_stft_mel_targets(const void* wav, int wav_int16, const int* lengths, const float* peak, float rescaling_max,
                         const float* mel_basis, const int* mel_start, const int* mel_len, float* linear, float* mel,
                         int nclips, int max_len, int T_lin, int lead, int downsample_step, int n_mels, float preemph,
                         float min_level_db, float ref_level_db, void* stream);
/* peak[c] = max |x| over the first lengths[c] samples of clip c (int16 as x / 32768); wav as above. */
int dv3_peak_abs_batched(const void* wav, int wav_int16, const int* lengths, int max_len, int nclips, float* peak,
                         void* stream);

/* ---- corpus front-end ahead of the STFT (csrc/resample.cu): the resampling inside reference audio.py:12-13
 * (load_wav) and the silence trimming of vctk.py:52-68 (librosa.effects.trim), for a ragged batch of clips.
 * dv3_resample_poly_batched: scipy.signal.resample_poly(x.astype(float64), up, down) rounded to fp32 (window
 * ('kaiser', 5.0), zero padding), up / down reduced.  wav (nclips, pitch_in) fp32 or, with wav_int16 != 0, int16 PCM
 * read as x / 32768; lengths int32 [nclips]; out (nclips, pitch_out) fp32 holds clip c's
 * dv3_resample_out_len(lengths[c], up, down) = ceil(n * up / down) samples, zero after them.  bank (ntaps, up) fp64 is
 * the polyphase filter bank, bank[j][p] = h[p + j * up] of the zero-padded filter h, and pre_remove the outputs
 * resample_poly drops in front (audio.resample_filter_bank).  Products and sums in fp64, in a fixed order per output:
 * a clip is bit-identical alone and in any batch.  The bank and a window of input stay in shared memory
 * (8 * up * ntaps + 4 * (4095 * down / up + ntaps + 2) bytes, at most the device's opt-in limit).
 * dv3_trim_bounds_batched: librosa.effects.trim(y, top_db[c]) (frame 2048, hop 512, ref = max, centred frames,
 * reflect padding; the librosa 0.6-0.9 defaults) of y = clip c's samples [offsets[c], offsets[c] + lengths[c]), in
 * fp64 -> bounds (nclips, 2) int32 (start, end) relative to y, (0, 0) when no frame is above the threshold.  wav as
 * above with row pitch `pitch`; offsets may be NULL (all 0); top_db fp64 [nclips].  No host synchronisation.
 * dv3_resample_segments_batched: part of dv3_resample_poly_batched's output for each of nclips clips, bit for bit.
 * seg int32 (nclips, 6) = {row, n_in, in_start, in_len, seg_start, seg_len} per clip: row `row` of wav (pitch_in, fp32
 * or int16 as above) holds samples [in_start, in_start + in_len) of a source clip of n_in samples (0 <= in_start,
 * in_start + in_len <= n_in, in_len <= pitch_in); row `row` of out (pitch_out fp32) gets the clip's resampled samples
 * [seg_start, seg_start + seg_len) in columns [0, seg_len) and zeros after them.  The caller keeps seg_start +
 * seg_len <= dv3_resample_out_len(n_in), seg_len <= pitch_out, the rows distinct, and [in_start, in_start + in_len)
 * covering every input sample the segment reads (audio.input_span): the kernel reads nothing else, and a sample
 * outside the row counts as 0.  up = down = 1 with the one-tap bank {1.0} copies (int16 as x / 32768). */
int dv3_resample_out_len(int n_samples, int up, int down);
int dv3_resample_poly_batched(const void* wav, int wav_int16, const int* lengths, int pitch_in, float* out,
                              int pitch_out, int nclips, const double* bank, int up, int down, int ntaps,
                              int pre_remove, void* stream);
int dv3_resample_segments_batched(const void* wav, int wav_int16, int pitch_in, const int* seg, int nclips, float* out,
                                  int pitch_out, const double* bank, int up, int down, int ntaps, int pre_remove,
                                  void* stream);
int dv3_trim_bounds_batched(const void* wav, int wav_int16, const int* lengths, const int* offsets, int pitch,
                            int nclips, const double* top_db, int* bounds, void* stream);

/* ---- inverse audio path: reference audio.py:37-43 (inv_spectrogram) and :26-28 (inv_preemphasis).
 * dv3_spec_to_amp: normalised dB (n) -> (10^((S*(-min)+min+ref)/20))^power.  dv3_deemphasis: y[n] = x[n] + coef*y[n-1]
 * per clip.  Griffin-Lim and the inverse STFT between them are the _geom entry points below, for every frame; LWS has
 * the specialised 1024 / 256 entry points here and the _geom ones for every other frame. */
int dv3_spec_to_amp(const float* spec_norm, float* amp, long long n, float min_level_db, float ref_level_db,
                    float power, void* stream);
/* LWS phase recovery at 1024 / 256 (csrc/lws.cu; Local Weighted Sums, the algorithm of the reference's lws.run_lws --
 * parity UNPINNED, the package's source is absent).  mag (nframes,513) target magnitude; spec (nframes,513,2) [re,im];
 * weights: 7 x 11 complex fp32 [q+3][d+5] = beta_q(d) = (1/1024) sum_n w(n) w(n-256q) e^{-2 pi i d n/1024}
 * (audio._lws_weights).  dv3_lws_nofuture: the no-future initialisation -> spec (frames in order from their 3 past
 * frames, then init_iters in-frame Jacobi passes).  dv3_lws_iterate: one batch iteration spec_in -> spec_out (distinct
 * buffers).  Batched forms: clip c has nframes[c] <= max_frames frames at spec + c*max_frames*513*2 (mag with 513
 * floats per frame), nframes int32 [nclips] on the device; frames past a clip's count are neither read nor written. */
int dv3_lws_nofuture(const float* mag, float* spec, const float* weights, int nframes, int init_iters, void* stream);
int dv3_lws_iterate(const float* mag, const float* spec_in, float* spec_out, const float* weights, int nframes,
                    void* stream);
int dv3_lws_nofuture_batched(const float* mag, float* spec, const float* weights, const int* nframes, int max_frames,
                             int nclips, int init_iters, void* stream);
int dv3_lws_iterate_batched(const float* mag, const float* spec_in, float* spec_out, const float* weights,
                            const int* nframes, int max_frames, int nclips, void* stream);
int dv3_deemphasis(const float* x, float* y, int nclips, int n_samples, long long stride, float coef, void* stream);

/* ---- the audio path for any supported STFT frame (csrc/stft_any.cu, csrc/lws_any.cu; audio.check_geometry):
 * n_fft even in [256, 4096] with n_fft / 2 free of prime factors above 5, hop = n_fft / Q with Q in [2, 8]; K =
 * n_fft / 2 + 1 bins; padding n_fft - hop samples on both sides.  An unsupported geometry returns an error before any
 * launch.  table: 3 * n_fft + 2 floats on the device -- window (n_fft), twiddles exp(-2 pi i j / (n_fft/2)) and split
 * factors exp(-2 pi i k / n_fft) as [re, im] pairs, computed in fp64 and rounded once (audio._geometry_table).
 * The forward mel path and LWS have specialised 1024 / 256 forms (dv3_stft_mel / dv3_stft_mel_targets and the LWS
 * entry points above); the complex STFT and inverse STFT entry points here are Griffin-Lim's path for every frame,
 * 1024 / 256 included.
 * dv3_stft_num_frames_geom: frames of an n-sample clip, ceil((n + n_fft - 2 hop) / hop) + 1.
 * dv3_stft_mel_geom: dv3_stft_mel_targets for the geometry (linear rows of K floats, mel_basis (n_mels, K) with the
 * same sparse span description; lead = 0, downsample_step = 1, T_lin = max_frames is the dv3_stft_mel layout).
 * Batched forms: clip c has n_samples[c] samples at wav + c*wav_pitch and nframes[c] <= max_frames frames at
 * spec + c*max_frames*K*2 (mag and prev likewise, mag with K floats per frame); both count arrays are int32 [nclips] on
 * the device.  Samples and frames past a clip's counts are neither read nor written.
 * dv3_stft_complex_geom: wav -> spec (frames, K, 2) [re, im]; mag != NULL projects the result onto that magnitude,
 * spec = mag * X / |X| ((mag, 0) where X == 0): the Griffin-Lim step x <- istft(mag * exp(i angle(stft(x)))), driven
 * by the host (audio.griffin_lim_batch).  dv3_istft_geom: wav += overlap-added windowed frames (zero wav first); the
 * overlap-add runs as Q ordered launches (frames f and f + Q do not overlap) with plain stores, deterministic.
 * dv3_stft_complex_momentum_geom: the fast Griffin-Lim step (Perraudin, Balazs & Sondergaard, WASPAA 2013;
 * audio.griffin_lim_batch with momentum > 0, DESIGN.md section 7.3): the transform of dv3_stft_complex_geom, then per
 * bin C = X - beta * prev, prev <- X (in place), spec = mag * C / |C| ((mag, 0) where C == 0); mag and prev are
 * required; beta in [0, 1) (= momentum / (1 + momentum)); beta == 0 gives dv3_stft_complex_geom's projected spec bit
 * for bit.
 * dv3_lws_nofuture_geom / dv3_lws_iterate_geom: the batched LWS forms with K bins; weights ((2Q - 1) * 11 + Q)
 * [re, im] fp32 pairs = beta_q(d) e^{2 pi i d q / Q} at [q + Q - 1][d + 5], |q| <= Q - 1, |d| <= 5, then the Q roots
 * e^{-2 pi i r / Q} (audio._lws_tables_fp64).
 * Every form: each clip of a ragged batch is bit-identical alone. */
int dv3_stft_num_frames_geom(int n_samples, int n_fft, int hop);
int dv3_stft_mel_geom(const void* wav, int wav_int16, const int* lengths, const float* peak, float rescaling_max,
                      const float* table, const float* mel_basis, const int* mel_start, const int* mel_len,
                      float* linear, float* mel, int nclips, int max_len, int T_lin, int lead, int downsample_step,
                      int n_mels, int n_fft, int hop, float preemph, float min_level_db, float ref_level_db,
                      void* stream);
int dv3_stft_complex_geom(const float* wav, const int* n_samples, long long wav_pitch, const float* mag, float* spec,
                          const int* nframes, int max_frames, int nclips, const float* table, int n_fft, int hop,
                          void* stream);
int dv3_istft_geom(const float* spec, float* wav, const int* n_samples, long long wav_pitch, const int* nframes,
                   int max_frames, int nclips, const float* table, int n_fft, int hop, void* stream);
int dv3_stft_complex_momentum_geom(const float* wav, const int* n_samples, long long wav_pitch, const float* mag,
                                   float* prev, float* spec, const int* nframes, int max_frames, int nclips,
                                   float beta, const float* table, int n_fft, int hop, void* stream);
int dv3_lws_nofuture_geom(const float* mag, float* spec, const float* weights, const int* nframes, int max_frames,
                          int nclips, int init_iters, int n_fft, int hop, void* stream);
int dv3_lws_iterate_geom(const float* mag, const float* spec_in, float* spec_out, const float* weights,
                         const int* nframes, int max_frames, int nclips, int n_fft, int hop, void* stream);

/* ================= tensor-core ConvBlock / conv path: wgmma + TMA, split 16-bit operands =================
 * Same reference code as dv3_convblock_fwd / dv3_conv1d_fwd / dv3_conv1d_dgrad / dv3_conv1d_wgrad (modules.py:94-100,
 * 145-164, 200-226 and their autograd).  Every fp32 operand is split into a (hi, lo) pair of 16-bit planes (below) and
 * each GEMM issues hi*hi + hi*lo + lo*hi.  Plane buffers are 16-bit device memory laid out [npl][...]; channel pitches
 * are padded to a multiple of 8.  Callers use the exact-fp32 entry points for unsupported shapes.
 * npl = 2 is the (hi, lo) pair.  npl = 1 is the single-pass mode: every buffer holds plane hi alone ([1][...], the same
 * bits as plane 0 of the pair: fp16 rn(x) clamped to +-65504 for forward operands, bf16 rn(x) for gradients and the
 * weight-gradient copy of the input) and each GEMM issues hi*hi only -- TF32-class forward GEMMs, bf16-class gradient
 * GEMMs, fp32 accumulation.  Entry points without an `npl` argument work on pairs; their _npl forms take both. */
int dv3_tc_supported(int B, int C, int T, int k);           /* gated block: C % 128 == 0, k <= 8 */
int dv3_tc_conv_supported(int B, int Cin, int Cout, int T, int k);   /* plain conv: k == 1 or Cout % 128 == 0 */
/* Operand planes: every fp32 operand x travels as hi = rn16(x), lo = rn16((x - hi) * 2^11) (csrc/common.cuh).
 * Forward GEMMs multiply fp16 pairs (22-bit operands: fp32-class results; activations and normalised weights are O(1),
 * values are clamped to +-65504); gradient GEMMs multiply bf16 pairs (gradients need the fp32 exponent range for any
 * loss scale) -- a wgmma does not mix operand formats, so a conv input is split into both.
 * x (B,C,T) fp32 -> conv-input dropout -> btc: [2][B][T][Cp] fp16 pair (forward operand, Cp = pad8(C)) and
 * bct (may be NULL): [2][B][T][Cp] bf16 pair of the same values (operand of the weight gradient).  npl = 1: btc and bct
 * hold plane hi alone, [1][B][T][Cp]. */
int dv3_tc_split_input(const float* x, void* btc, int npl, void* bct, int B, int C, int T, int k, int dilation,
                       int causal, float p_drop, const unsigned long long* seed_ptr, unsigned salt, void* stream);
/* gate backward writing dAB = [da ; db] as planes btc: [2][B][T][2C], the operand of both the data and the weight
 * gradient; bct is reserved and must be NULL. */
int dv3_tc_gate_bwd_split(const float* dy, const float* a, const float* s, const float* x, void* btc, void* bct,
                          float* dbias, int B, int C, int T, int mode, int residual, void* stream);
/* plain-conv backward prologue: g = dy*(relu ? y>0 : 1) -> btc: [2][B][T][Cp] (the operand of both gradient GEMMs);
 * bct is reserved and must be NULL; dbias[C] += sums. */
int dv3_tc_grad_split(const float* dy, const float* y, void* btc, void* bct, float* dbias, int B, int C, int T,
                      int relu, void* stream);
/* The three splits with an optional logical time extent in device memory (a training batch padded to a bucket):
 * tlen NULL = the calls above; else frames t >= tmult * tlen[0] of x (forward operand) / of dy (gradient) are taken as
 * 0: the extent time mask and its gradient, folded into passes that read those tensors anyway. */
int dv3_tc_split_input_ext(const float* x, void* btc, int npl, void* bct, int B, int C, int T, float p_drop,
                           const unsigned long long* seed_ptr, unsigned salt, const long long* tlen, int tmult,
                           void* stream);
int dv3_tc_gate_bwd_split_ext(const float* dy, const float* a, const float* s, const float* x, void* btc, void* bct,
                              float* dbias, int B, int C, int T, int mode, int residual, const long long* tlen,
                              int tmult, void* stream);
int dv3_tc_grad_split_ext(const float* dy, const float* y, void* btc, void* bct, float* dbias, int B, int C, int T,
                          int relu, const long long* tlen, int tmult, void* stream);
/* Both gradient splits with the plane count: btc [npl][B][T][2C] / [npl][B][T][Cp], npl in {1, 2}; tlen / tmult as the
 * _ext forms (tlen NULL: no extent).  npl = 2 gives what the calls above give. */
int dv3_tc_gate_bwd_split_npl(const float* dy, const float* a, const float* s, const float* x, void* btc, int npl,
                              void* bct, float* dbias, int B, int C, int T, int mode, int residual,
                              const long long* tlen, int tmult, void* stream);
int dv3_tc_grad_split_npl(const float* dy, const float* y, void* btc, int npl, void* bct, float* dbias, int B, int C,
                          int T, int relu, const long long* tlen, int tmult, void* stream);
/* weight norm + split: v (Cout,Cin,k), g [Cout] -> wfwd: [npl][k][Cout][Cinp] (forward), wbwd: [npl][k][Cin][Coutp]
 * (dgrad); npl in {1, 2}. */
int dv3_tc_weightnorm_fwd(const float* v, const float* g, float* inv_norm, float* scale, void* wfwd, int npl,
                          void* wbwd, int Cout, int Cin, int k, void* stream);
/* ConvTranspose1d(k=2,s=2) weight v (Cin,Cout,2), g [Cin] as a 1x1 conv with 2*Cout rows ordered (j,co):
 * wfwd: [npl][2*Cout][Cinp], wbwd: [npl][Cin][pad8(2*Cout)]; npl in {1, 2}. */
int dv3_tc_weightnorm_convt_fwd(const float* v, const float* g, float* inv_norm, float* scale, void* wfwd, int npl,
                                void* wbwd, int Cin, int Cout, void* stream);
/* ConvTranspose1d(k=s, stride=s), s in [2, 8]: v (Cin,Cout,s), g [Cin] as a 1x1 conv with s*Cout rows ordered (j,co):
 * wfwd: [npl][s*Cout][Cinp], wbwd: [npl][Cin][pad8(s*Cout)] (the k = 2 layer keeps dv3_tc_weightnorm_convt_fwd). */
int dv3_tc_weightnorm_convt_s_fwd(const float* v, const float* g, float* inv_norm, float* scale, void* wfwd, int npl,
                                  void* wbwd, int Cin, int Cout, int stride, void* stream);
/* Batched weight norm (csrc/wn_batched.cu): one record per weight-normed conv (v (Cout,Cin,k), g [Cout]); the table
 * lives in DEVICE memory, blk_* are the first block of the record in the batched norm / pack / backward launches
 * (ascending over the table), pack_gx = ceil(Cin*k / 32).  Layouts as dv3_tc_weightnorm_fwd with npl = 2; the
 * backward consumes tap-major partials [nsplit][k][Cout][Cin] (what dv3_tc_wgrad_mn writes; slot 0 is scratch). */
typedef struct Dv3WnEntry {
    const float* v; const float* g; float* inv_norm; float* scale;
    void* wfwd; void* wbwd;
    float* partials; float* dv; float* dg;
    long long split_stride;
    int Cout, Cin, k, nsplit;
    int blk_norm, blk_pack, blk_bwd, pack_gx;
} Dv3WnEntry;
/* norm + pack of every record: 2 launches (replaces 2 launches per layer).  The _npl form packs npl in {1, 2} planes
 * per layout (wfwd [npl][k][Cout][Cinp], wbwd [npl][k][Cin][Coutp]); the plain form is npl = 2. */
int dv3_tc_weightnorm_fwd_batched(const Dv3WnEntry* table_dev, int n, int norm_blocks, int pack_blocks,
                                  void* stream);
int dv3_tc_weightnorm_fwd_batched_npl(const Dv3WnEntry* table_dev, int n, int norm_blocks, int pack_blocks, int npl,
                                      void* stream);
/* split-K reduction + dg / dv of every record: 1 launch; accumulate = 1 adds into dv / dg. */
int dv3_weightnorm_bwd_batched(const Dv3WnEntry* table_dev, int n, int bwd_blocks, int accumulate, void* stream);
/* gated forward: xd = btc planes of dv3_tc_split_input, w = wfwd planes [npl][k][2C][C]; npl in {1, 2}, fuse is
 * reserved and must be NULL. */
int dv3_tc_convblock_fwd(const void* xd, const void* w, int npl, const float* bias, const float* spk,
                         const float* res, float* y, float* save_a, float* save_s, int B, int C, int T, int k,
                         int dilation, int causal, int mode, int residual, const void* fuse, void* stream);
/* generic conv / data gradient: out (B,Nc,T) = sum_j A[b,t+off_j,:].W[j,n,:], then *dropmask, +bias, +addend, relu.
 * a: [npl][B][T][pad8(Kc)], w: [npl][k][Nc][pad8(Kc)] (fp16 planes for a forward conv, bf16 planes for a data
 * gradient); transpose_taps = 1 for a data gradient.  npl in {1, 2}, fuse is reserved and must be NULL. */
int dv3_tc_conv(const void* a, const void* w, int npl, float* out, int B, int Kc, int Nc, int T, int k, int dilation,
                int causal, int transpose_taps, const float* bias, int relu, float p_drop,
                const unsigned long long* seed_ptr, unsigned salt, int addmode, const float* e1, const float* e2,
                float alpha, const void* fuse, void* stream);
/* weight gradient from the (B,T,C) planes (MN-major operands, tap shift = TMA row coordinate):
 * dy: [2][B][T][pad8(Mw)], xd: [2][B][T][pad8(Nw)]; partial element (m,n,j) of split s at
 * dw_partials + s*split_stride + (m%msplit)*s_m + (m/msplit)*s_mh + n*s_n + j*s_j; dv3_tc_wgrad_nsplit(...) splits. */
int dv3_tc_wgrad_nsplit(int B, int Mw, int Nw, int T, int k);
int dv3_tc_wgrad_mn(const void* dy, const void* xd, float* dw_partials, long long split_stride, int B, int Mw,
                    int Nw, int T, int k, int dilation, int causal, int msplit, long long s_m, long long s_mh,
                    long long s_n, long long s_j, void* stream);
/* the same with the plane count: dy [npl][B][T][pad8(Mw)], xd [npl][B][T][pad8(Nw)], npl in {1, 2} */
int dv3_tc_wgrad_mn_npl(const void* dy, const void* xd, int npl, float* dw_partials, long long split_stride, int B,
                        int Mw, int Nw, int T, int k, int dilation, int causal, int msplit, long long s_m,
                        long long s_mh, long long s_n, long long s_j, void* stream);

/* ---- fused training losses + gradients: reference train.py:537-601 (spec_loss, guided_attention) and :704-740.
 * dv3_spec_loss: pairs (y_hat[b,t], y[b,t+r]), t < T-r; lengths int64 [B] valid target frames; adds
 * (1-bw)*L1 + bw*binary_divergence (each = w*masked_mean + (1-w)*mean) to loss[0]; grad (B,T,D) = dLoss/dy_hat.
 * priority_bin > 0 and priority_weight > 0: L1 = (1-pw)*L1(all D bins) + pw*L1(bins < priority_bin), train.py:559-567.
 * dv3_aux_loss: adds BCE(done_hat, done) and, if use_attn, mean(attn*W) with the guided-attention mask
 * W[b,t,n] = 1-exp(-(n/in_len[b] - t/dec_len[b])^2/(2 sigma^2)) built on the fly; writes both gradients. */
int dv3_spec_loss(const float* y_hat, const float* y, const long long* lengths, float* grad, float* loss, int B,
                  int T, int D, int r, float masked_loss_weight, float binary_divergence_weight, int priority_bin,
                  float priority_weight, void* stream);
int dv3_aux_loss(const float* done_hat, const float* done, float* d_done, long long n_done, const float* attn,
                 float* d_attn, const long long* in_len, const long long* dec_len, int A, int B, int Td, int Ts,
                 float sigma, int use_attn, float* loss, void* stream);
/* Extent variants for a batch padded to a bucket shape (logical extents in device memory, read by the kernels):
 * dv3_spec_loss_ext: pairs t >= t_log[0] - r leave the loss and the means (which divide by B*(t_log-r)*D);
 * dv3_aux_loss_ext: done_hat / done are (B, Td); ext = {decoder steps, text positions}: steps >= ext[0] and text
 * positions >= ext[1] leave both means (B*ext[0] and A*B*ext[0]*ext[1]).  Gradients there are written as 0. */
int dv3_spec_loss_ext(const float* y_hat, const float* y, const long long* lengths, const long long* t_log,
                      float* grad, float* loss, int B, int T, int D, int r, float masked_loss_weight,
                      float binary_divergence_weight, int priority_bin, float priority_weight, void* stream);
int dv3_aux_loss_ext(const float* done_hat, const float* done, float* d_done, const float* attn, float* d_attn,
                     const long long* in_len, const long long* dec_len, const long long* ext, int A, int B, int Td,
                     int Ts, float sigma, int use_attn, float* loss, void* stream);
/* The same kernels with the extents nullable (NULL: the full tensors) and the loss split into the terms reference
 * train.py logs (:761-776).  terms (nullable) is a float block with the DV3_TERM_* slots below, zeroed by the caller;
 * each call adds its two parts to two consecutive slots:
 *   dv3_spec_loss_terms: terms[0] += L1 part (priority bins combined), terms[1] += binary-divergence part (0 when
 *     binary_divergence_weight <= 0) -- pass terms + DV3_TERM_MEL_L1 or terms + DV3_TERM_LIN_L1;
 *   dv3_aux_loss_terms: terms[0] += done BCE, terms[1] += guided-attention term -- pass terms + DV3_TERM_DONE.
 * loss and every gradient are exactly those of the calls without terms.  The other four entry points are these with
 * terms = NULL. */
enum { DV3_TERM_MEL_L1 = 0, DV3_TERM_MEL_BD = 1, DV3_TERM_LIN_L1 = 2, DV3_TERM_LIN_BD = 3, DV3_TERM_DONE = 4,
       DV3_TERM_ATTN = 5, DV3_TERM_COUNT = 6 };
int dv3_spec_loss_terms(const float* y_hat, const float* y, const long long* lengths, const long long* t_log,
                        float* grad, float* loss, float* terms, int B, int T, int D, int r, float masked_loss_weight,
                        float binary_divergence_weight, int priority_bin, float priority_weight, void* stream);
int dv3_aux_loss_terms(const float* done_hat, const float* done, float* d_done, long long n_done, const float* attn,
                       float* d_attn, const long long* in_len, const long long* dec_len, const long long* ext, int A,
                       int B, int Td, int Ts, float sigma, int use_attn, float* loss, float* terms, void* stream);

/* ---- deterministic mode (ops.deterministic, DESIGN.md section 2.10): twins of the five entry-point families whose
 * kernels accumulate floats with cross-block atomics.  Each gives the same values with every sum formed in an order
 * fixed by the tensor shapes, so two runs give identical bits.  Like their twins they ADD to loss / terms / dbias /
 * dtable.  The caller owns the scratch; no kernel waits for another block (the last block to finish does the tail, or
 * a second small launch does).
 *   losses: every block stores its partial sums in `scratch` (dv3_loss_det_scratch_floats() floats, zero-filled once
 *     by the caller; the last word is a ticket the kernel leaves at zero); the block that draws the last ticket adds
 *     them in block order.  t_log / ext / terms are nullable: one call for the plain, _ext and _terms forms.
 *   bias gradients: partial sums per utterance (exact-fp32 kernels) or per (utterance, 64-frame tile) (tensor-core
 *     operand splits; frames past tmult * tlen[0] stay out) go to scratch[partial][channel], needing
 *     dv3_bias_det_scratch_floats(B, channels, T, tiled) floats (channels = 2C for the gated forms; tiled = 1 for the
 *     tensor-core splits); a second launch adds them to dbias in partial order.  dbias is required.
 *   table gradients: one CTA per table row gathers its tokens in index order; D <= 1024. */
int dv3_loss_det_scratch_floats(void);
int dv3_spec_loss_det(const float* y_hat, const float* y, const long long* lengths, const long long* t_log,
                      float* grad, float* loss, float* terms, float* scratch, int B, int T, int D, int r,
                      float masked_loss_weight, float binary_divergence_weight, int priority_bin,
                      float priority_weight, void* stream);
int dv3_aux_loss_det(const float* done_hat, const float* done, float* d_done, long long n_done, const float* attn,
                     float* d_attn, const long long* in_len, const long long* dec_len, const long long* ext, int A,
                     int B, int Td, int Ts, float sigma, int use_attn, float* loss, float* terms, float* scratch,
                     void* stream);
long long dv3_bias_det_scratch_floats(int B, int nch, int T, int tiled);
int dv3_convblock_gate_bwd_det(const float* dy, const float* a, const float* s, const float* x, float* dab,
                               float* dbias, float* scratch, long long scratch_floats, int B, int C, int T, int mode,
                               int residual, void* stream);
int dv3_bias_act_bwd_det(const float* dy, const float* y, float* dyr, float* dbias, float* scratch,
                         long long scratch_floats, int B, int C, int T, int relu, void* stream);
int dv3_tc_gate_bwd_split_det(const float* dy, const float* a, const float* s, const float* x, void* btc, int npl,
                              float* dbias, float* scratch, long long scratch_floats, int B, int C, int T, int mode,
                              int residual, const long long* tlen, int tmult, void* stream);
int dv3_tc_grad_split_det(const float* dy, const float* y, void* btc, int npl, float* dbias, float* scratch,
                          long long scratch_floats, int B, int C, int T, int relu, const long long* tlen, int tmult,
                          void* stream);
int dv3_embedding_bwd_det(const long long* ids, const float* dy, float* dtable, int N, int D, int V,
                          long long padding_idx, void* stream);
int dv3_sinusoid_bwd_det(const long long* pos, const float* table, const float* w, int nw, const float* dy,
                         float* dtable, float* dw, int B, int T, int D, int P, void* stream);

/* ---- incremental (autoregressive) decoding: reference conv.py:17-46, deepvoice3.py:367-485, nyanko.py:250-338 ----
 * All loop state lives in device memory so that one decoder step is the same launch sequence every time (CUDA-graph
 * replay): *t_ptr is the step counter; every row pointer advances by a per-step stride: row b of step t of operand
 * X is X + b*X_ld + t*X_t (floats). */
typedef struct Dv3IncStep {
    const float* x; long long x_ld, x_t;          /* current input (B, Cin) */
    const float* add; long long add_ld, add_t;    /* optional, added to the input (position encoding) */
    float* ring;                                   /* (B, (k-1)*dilation+1, Cin) zero-initialised history; NULL: k = 1 */
    const float* w; const float* bias;             /* normalised weight linearised as [Cout][k][Cin]; [Cout] */
    const float* spk; long long spk_ld;            /* GLU: softsign(speaker_proj(embed)) (B, C) or NULL */
    const float* res1; long long res1_ld, res1_t;  /* y = (y + res1)*sqrt(.5) if non-NULL, then the same with res2 */
    const float* res2; long long res2_ld, res2_t;
    float* y; long long y_ld, y_t;
    float* y2; long long y2_ld, y2_t;              /* optional second output, see y2_mode */
    const float* yadd; long long yadd_ld, yadd_t;  /* y2_mode 2: y2 = y + yadd (position encoding of the query) */
    const int* t_ptr;
    int B, Cin, Cout, k, dilation;
    int mode;                                      /* 0 plain conv, 1 GLU (a*sigmoid(b)), 2 highway */
    int act;                                       /* plain: 0 none, 1 ReLU, 2 sigmoid */
    int vec4;                                      /* 1: Cin % 4 == 0 and every input row is 16-byte aligned */
    int y2_mode;                                   /* 1: y2 = sigmoid(y); 2: y2 = y + yadd */
} Dv3IncStep;
int dv3_inc_conv_step(const Dv3IncStep* step, void* stream);
typedef struct Dv3IncAttn {
    const float* q; long long q_ld;                /* projected query (B, E) */
    const float* keys; const float* values;        /* (B, E, Ts) pre-transposed, (B, Ts, E): projected once */
    float* ctx; long long ctx_ld;                  /* context * float(Ts*sqrt(1/Ts)) (B, E) */
    float* align; long long align_ld, align_t;     /* probabilities * align_scale, or NULL */
    int* last_attended;                            /* int[2] (slot t&1 read, (t+1)&1 written) or NULL: no window */
    const int* t_ptr;
    float align_scale;
    int B, E, Ts, window_backward, window_ahead;   /* E + Ts <= 12279: with 9 floats of scratch, 48 KB of smem */
} Dv3IncAttn;
int dv3_inc_attn_step(const Dv3IncAttn* attn, void* stream);
/* Ragged batch: row b attends to s < text_len[b] only (text_len: int32 [B] on the device, 1 <= text_len[b] <= Ts),
 * its context is scaled by text_len[b]*sqrt(1/text_len[b]) and alignment entries s >= text_len[b] are 0.  A non-NULL
 * last_attended holds B cursors per slot, int[2][B] (slot t&1 read, (t+1)&1 written): every row keeps its own
 * monotonic window, clamped to its own text length.  Each row gives what dv3_inc_attn_step gives for that row alone
 * with Ts = text_len[b], bit for bit. */
int dv3_inc_attn_step_rows(const Dv3IncAttn* attn, const int* text_len, void* stream);
int dv3_inc_advance(int* t_ptr, void* stream);

/* ---- continuous batching: a fixed set of B decoder slots, each running its own utterance at its own step ----
 * The _slots step variants read t_ptr as int[B]: row b runs step t_ptr[b] (every per-step stride, the ring slot of
 * each tap, the filing slot, the alignment row and the cursor parity follow it) with the same per-output arithmetic
 * as dv3_inc_conv_step / dv3_inc_attn_step_rows, so a row at step t gets the bits those give at step t. */
int dv3_inc_conv_step_slots(const Dv3IncStep* step, void* stream);
int dv3_inc_attn_step_slots(const Dv3IncAttn* attn, const int* text_len, void* stream);
/* The reference stop rule on each row: after step t[b] wrote done[b*done_ld + t[b]], n = t[b]+1 steps ran; if
 * stop[b] == 0 and (done > 0.5 and n > min_steps, or n > max_steps), stop[b] = n.  done_ld > max_steps. */
int dv3_inc_stop_rows(const float* done, long long done_ld, const int* t, int* stop, int B, int min_steps,
                      int max_steps, void* stream);
/* ---- guided decoding (DESIGN.md section 2.22): the attention window's centre follows a prescribed token path ----
 * The _path variants are dv3_inc_attn_step_rows / dv3_inc_attn_step_slots with the cursor of row b at step t read as
 * path[b*path_ld + t] (int32, device) instead of from last_attended, which they neither read nor write; the window
 * [c - window_backward, c + window_ahead) clamped to [0, text_len[b]), the softmax, alignment and context are those
 * of the _rows step.  path_ld >= the steps the program runs. */
int dv3_inc_attn_step_path(const Dv3IncAttn* attn, const int* text_len, const int* path, long long path_ld,
                           void* stream);
int dv3_inc_attn_step_slots_path(const Dv3IncAttn* attn, const int* text_len, const int* path, long long path_ld,
                                 void* stream);
/* The guided stop rule: if stop[b] == 0 and t[b] + 1 >= total[b], stop[b] = t[b] + 1 (total[b] >= 1 steps, set per
 * utterance); the done flags play no part. */
int dv3_inc_stop_rows_total(const int* t, int* stop, const int* total, int B, void* stream);
/* t[b] += 1 for every row with stop[b] == 0 (every row when stop is NULL).  A stopped row keeps its step and so
 * recomputes it bit for bit; the host gathers it and refills the slot. */
int dv3_inc_advance_rows(int* t, const int* stop, int B, void* stream);
/* One row copy of a slot refill: row b of dst (at dst + b*dst_row_stride bytes) <- row i of src (src + i*src_row_stride)
 * for the i-th refilled slot b, or zeros when src is NULL.  Pointers, row_bytes and strides are multiples of 4. */
typedef struct Dv3IncRefill {
    void* dst; const void* src;
    long long row_bytes, dst_row_stride, src_row_stride;
} Dv3IncRefill;
/* table: n_entries Dv3IncRefill in device memory; slots: n_slots slot indices (int32, device).  One launch resets the
 * listed slots (ring rows, cursors, counters, go frame) and loads their next utterances' constants from staging. */
int dv3_inc_refill(const Dv3IncRefill* table, int n_entries, const int* slots, int n_slots, void* stream);

/* ---- duration predictor loss (duration.cu, DESIGN.md section 2.22) ----
 * y (B, L) predicted log-durations with row stride y_ld, durations (B, L) int32 target steps with row stride d_ld,
 * lengths int32 [B]: row b's tokens j < lengths[b] count.  1 <= L <= dv3_duration_max_tokens() = 1024, B <= 65535.
 * dv3_duration_loss_fwd: row_loss[b] = (1/n_b) sum_j (y - log d)^2 summed in fp64 in token order, then
 * *loss = fp32((1/B) sum_b row_loss[b]) summed in row order; no atomics.  A row with lengths[b] outside [1, L] or a
 * duration < 1 among its tokens sets *err_flag and counts 0.
 * dv3_duration_loss_bwd: dy (B, L) dense = fp32(d_loss[0] * 2 (y - log d) / (n_b B)) for j < n_b, 0 past it and for
 * the rows the forward counts 0. */
int dv3_duration_max_tokens(void);
int dv3_duration_loss_fwd(const float* y, long long y_ld, const int* durations, long long d_ld, const int* lengths,
                          int B, int L, double* row_loss, float* loss, int* err_flag, void* stream);
int dv3_duration_loss_bwd(const float* y, long long y_ld, const int* durations, long long d_ld, const int* lengths,
                          int B, int L, const float* d_loss, float* dy, void* stream);

/* ---- speaker adaptation: embedding gradient of a speaker-conditioned site with its weights frozen (spk_adapt.cu) ----
 * The site's share of d_e[b*S + s] = sum_{t < T_b} m(b,t,s)/(1-p) * sum_c w[c*S + s] * G(b,c,t) * (1 - |y(b,c,t)|)^2
 * is written as dv3_spk_grad_splits() partial rows: partials[(k*B + b)*S + s], k < splits (every one written).
 * y = softsign(z) of the site's forward; w (C, S) its folded weight; m the dropout mask of the stack's (B,T,S)
 * expanded embedding at element (b*T + t)*S + s (seed_ptr / salt of that dropout call; p = 0 or seed_ptr NULL: none).
 * T_b = min(T, ext[0] * ext_mult) when ext is given, else T.  Fixed summation order, no atomics.  S <= 64,
 * B <= 65535.
 * Layouts of G: _planes  bf16 [npl][B][T][ldg] operand planes of the gate split (channels [0, C) are the "a" half),
 *                        plane_stride elements apart, value hi + lo * 2^-11; y (B,C,T)
 *               _bct     fp32 (B,C,T) with batch stride g_bstride (the a half of the exact path's (B,2C,T) gate
 *                        gradient); y (B,C,T)
 *               _btc     fp32 (B,T,C) residual-stream gradient; y (B,T,C)
 * dv3_spk_grad_reduce: d_e[b*S + s] = sum over i < nparts, in order, of partials[(i*B + b)*S + s] -- the partial rows
 * of every site of a pass, laid out one after the other. */
int dv3_spk_grad_splits(void);
int dv3_spk_grad_planes(const void* g_planes, int npl, long long plane_stride, int ldg, const float* y_bct,
                        const float* w, float* partials, int B, int C, int T, int S, const long long* ext,
                        int ext_mult, float p, const unsigned long long* seed_ptr, unsigned salt, void* stream);
int dv3_spk_grad_bct(const float* g_bct, long long g_bstride, const float* y_bct, const float* w, float* partials,
                     int B, int C, int T, int S, const long long* ext, int ext_mult, float p,
                     const unsigned long long* seed_ptr, unsigned salt, void* stream);
int dv3_spk_grad_btc(const float* g_btc, const float* y_btc, const float* w, float* partials, int B, int C,
                     int T, int S, const long long* ext, int ext_mult, float p, const unsigned long long* seed_ptr,
                     unsigned salt, void* stream);
int dv3_spk_grad_reduce(const float* partials, long long nparts, float* d_e, int B, int S, void* stream);
/* grad[j*S + s] = sum over rows b (ascending) with ids[b] == lo + j of d_e[b*S + s] (+ d_e2[b*S + s] when non-NULL),
 * j < n; rows whose id lies outside [lo, lo + n) contribute nothing and set *err_flag = 1 (when non-NULL). */
int dv3_spk_rows_grad(const float* d_e, const float* d_e2, const long long* ids, long long lo, int n, float* grad,
                      int* err_flag, int B, int S, void* stream);

/* ---- speaker encoder: masked temporal mean and cloning-sample attention (spk_enc.cu) ----
 * dv3_spkenc_pool_fwd: y[r*C + c] = sum_{t < len[r]} x[(r*C + c)*T + t] / len[r], summed in an order fixed by
 * (C, len[r]) alone.  dv3_spkenc_pool_bwd: dx[(r*C + c)*T + t] = dy[r*C + c] / len[r] for t < len[r], else 0.  A
 * length outside [1, T] sets *err_flag = 1 and yields 0 (nothing is read out of bounds).
 * dv3_spkenc_attn_fwd: one CTA per speaker b over its counts[b] in [1, N] valid rows h (B, N, C):
 * q, k, v = W h + b (W (C, C), row-major [out][in]); o = multi-head softmax(q k^T / sqrt(C/heads)) v, keys masked
 * past counts[b]; s = w_s.o + b_s; a = softmax over the valid rows; e = W_e h + b_e (W_e (S, C)); out[b*S + s] =
 * sum_i a_i e_i[s].  ws: dv3_spkenc_ws_floats(N, C, S, heads) floats per speaker, what the backward reads.  With a
 * target (B, S), loss_partials[b] = sum_s |out - target|.  A count outside [1, N] sets *err_flag and yields 0.
 * dv3_spkenc_attn_bwd: d(out) = d_out (B, S) (nullable) + d_loss[0] * loss_scale * sign(out - target) (when both
 * are non-NULL); writes d_h (B, N, C) (rows >= counts[b]: 0) and one partial gradient row of
 * dv3_spkenc_param_floats(C, S) floats per speaker: W_q, W_k, W_v, b_q, b_k, b_v, w_s, b_s, W_e, b_e in that order.
 * dv3_spkenc_reduce: grad[p] = sum_{b < B} partials[b*P + p] in index order (partials nullable); loss[0] = loss_scale
 * * sum_b loss_partials[b] in index order (loss nullable).  N <= 32, C <= 256, S <= 64, heads <= 8 dividing C.
 * No atomics. */
long long dv3_spkenc_ws_floats(int N, int C, int S, int heads);
long long dv3_spkenc_param_floats(int C, int S);
int dv3_spkenc_pool_fwd(const float* x, const int* lengths, float* y, int* err_flag, int R, int C, int T,
                        void* stream);
int dv3_spkenc_pool_bwd(const float* dy, const int* lengths, float* dx, int* err_flag, int R, int C, int T,
                        void* stream);
int dv3_spkenc_attn_fwd(const float* h, const int* counts, const float* w_q, const float* b_q, const float* w_k,
                        const float* b_k, const float* w_v, const float* b_v, const float* w_s, const float* b_s,
                        const float* w_e, const float* b_e, const float* target, float* out, float* ws,
                        float* loss_partials, int* err_flag, int B, int N, int C, int S, int heads, void* stream);
int dv3_spkenc_attn_bwd(const float* h, const int* counts, const float* w_q, const float* b_q, const float* w_k,
                        const float* b_k, const float* w_v, const float* b_v, const float* w_s, const float* b_s,
                        const float* w_e, const float* b_e, const float* target, const float* d_out,
                        const float* d_loss, float loss_scale, float* ws, float* d_h, float* partials,
                        int* err_flag, int B, int N, int C, int S, int heads, void* stream);
int dv3_spkenc_reduce(const float* partials, long long P, const float* loss_partials, float loss_scale, float* grad,
                      float* loss, int B, void* stream);

/* ---- speaker verifier: enrollment / test embeddings, PLDA-like pair scores, balanced BCE (spk_ver.cu) ----
 * dv3_spkver_embed_fwd: row b reads counts[b] in [1, N] valid rows h[b*ld + i*C + c] (i < counts[b], C channels):
 * hbar[b*C + c] = their mean (summed in i order); out[b*D + d] = sum_c w[d*C + c] hbar[b*C + c] + c[d] (w (D, C)).
 * ld >= N*C is the float stride between rows b (a test row of a (B, N+1, C) batch: h offset by N*C, ld (N+1)*C).
 * dv3_spkver_embed_bwd: d_h[b*ld + i*C + c] = sum_d w[d*C + c] d_out[b*D + d] / counts[b] for i < counts[b], 0 for
 * counts[b] <= i < N; one partial row of D*C + D floats per row b: d w = d_out hbar^T, then d c = d_out.  A count
 * outside [1, N] sets *err_flag = 1 and yields 0 (nothing is read out of bounds).
 * dv3_spkver_score_fwd: scores[e*B_t + t] = x_e.y_t - x_e^T S x_e - y_t^T S y_t + bias[0] for x (B_e, D), y (B_t, D),
 * S (D, D); qx (B_e) / qy (B_t) receive the quadratic terms, computed once per row.  A pair's bits depend on its two
 * rows alone.  With int64 speaker ids ids_e (B_e) / ids_t (B_t) (nullable, with loss_partials), pair (e, t) is a
 * same-speaker pair when the ids are equal; loss_partials (dv3_spkver_loss_floats(B_e, B_t) floats, row-major over
 * (e, 32-pair column tile)) receive sum over the tile's t of softplus(-L) / (2 n_same) (same) or softplus(L) /
 * (2 n_diff) (different), n_same / n_diff counted on the device over the whole batch (an empty class weighs 0).
 * dv3_spkenc_reduce(NULL, 0, loss_partials, 1, NULL, loss, dv3_spkver_loss_floats(B_e, B_t)) sums them in order.
 * dv3_spkver_score_bwd: G = d_scores (nullable) + d_loss[0] * d(loss)/d(scores) (when ids and d_loss are non-NULL);
 * dx_e = sum_t G[e,t] y_t - g_e (S + S^T) x_e with g_e = sum_t G[e,t], dy likewise; one partial row of D*D + 1 floats
 * per row of x (rows 0..B_e-1) then of y: d S = -g z z^T, then d bias (g_e on x rows, 0 on y rows).
 * N <= 32, C <= 256, D <= 128.  Every sum runs in an order fixed by the shapes; no atomics. */
long long dv3_spkver_loss_floats(int B_e, int B_t);
int dv3_spkver_embed_fwd(const float* h, long long ld, const int* counts, const float* w, const float* c, float* hbar,
                         float* out, int* err_flag, int B, int N, int C, int D, void* stream);
int dv3_spkver_embed_bwd(const float* d_out, const float* hbar, const int* counts, const float* w, float* d_h,
                         long long ld, float* partials, int* err_flag, int B, int N, int C, int D, void* stream);
int dv3_spkver_score_fwd(const float* x, const float* y, const float* S, const float* bias, const long long* ids_e,
                         const long long* ids_t, float* qx, float* qy, float* scores, float* loss_partials, int B_e,
                         int B_t, int D, void* stream);
int dv3_spkver_score_bwd(const float* x, const float* y, const float* S, const float* scores, const long long* ids_e,
                         const long long* ids_t, const float* d_scores, const float* d_loss, float* dx, float* dy,
                         float* partials, int B_e, int B_t, int D, void* stream);

/* ---- speaker classifier: logits, log-sum-exp, argmax and softmax cross-entropy over K classes (spk_cls.cu) ----
 * dv3_spkcls_fwd: logits[r*K + k] = sum_c h[r*ld + c] w[k*C + c] + bias[k] (summed in c order) for R rows of C
 * channels (ld >= C floats apart) and w (K, C); lse[r] = log sum_k exp(logits[r*K + k]) over a thread partition fixed
 * by K alone; pred[r] = argmax_k logits[r*K + k], ties to the lowest index.  With int64 labels (R) (nullable, with
 * loss_partials): loss_partials[r] = lse[r] - logits[r*K + labels[r]];
 * dv3_spkenc_reduce(NULL, 0, loss_partials, 1/R, NULL, loss, R) gives the mean cross-entropy.  A row's logits, lse and
 * pred depend on that row alone.
 * dv3_spkcls_bwd: G[r,k] = d_logits[r*K + k] (nullable) + d_loss[0] * loss_scale * (exp(logits[r*K + k] - lse[r]) -
 * [k == labels[r]]) (the second term when labels and d_loss are non-NULL), never stored; d_h[r*C + c] = sum_k G[r,k]
 * w[k*C + c] (k in order, d_h dense); d_w[k*C + c] = sum_r G[r,k] h[r*ld + c] and d_bias[k] = sum_r G[r,k] (r in
 * order), written directly.  A label outside [0, K) sets *err_flag = 1; its row adds 0 to the loss and nothing to the onehot.
 * C <= 256, 2 <= K <= 8192, R*K < 2^31.  No atomics. */
int dv3_spkcls_fwd(const float* h, long long ld, const float* w, const float* bias, const long long* labels,
                   float* logits, float* lse, int* pred, float* loss_partials, int* err_flag, int R, int C, int K,
                   void* stream);
int dv3_spkcls_bwd(const float* h, long long ld, const float* w, const float* logits, const float* lse,
                   const long long* labels, const float* d_logits, const float* d_loss, float loss_scale, float* d_h,
                   float* d_w, float* d_bias, int* err_flag, int R, int C, int K, void* stream);

/* ---- mel-cepstral distortion after dynamic time warping (mcd.cu) ----
 * dv3_mel_cepstra: cep[(q*T_max + t)*K + k] = sum_m basis[k*M + m] mels[(q*T_max + t)*M + m] (m in order) for the
 * n_seq sequences of lengths[q] (int32) frames each; basis (K, M) is the orthonormal DCT-II rows 1..K times
 * -min_level_db ln10 / 20 (mcd.py).  Frames t >= lengths[q] are not read and give zeros.  2 <= M <= 128,
 * 1 <= K <= min(M - 1, 64), T_max <= dv3_mcd_max_frames().
 * dv3_dtw_mcd: for each row (pair, a_row, N, b_row, M, ws_off) of the int64 work list (P, 6), the DTW of the N cepstra
 * starting at row a_row of cep (K floats a row) against the M starting at b_row: cost[pair] = D(N, M) and
 * path_len[pair] = L (DESIGN.md section 2.17; ties to the diagonal, then (i-1, j), then (i, j-1)).  workspace: per row
 * 2 * roundup(M, 32) floats at ws_off (a multiple of 32).  One warp per row, launched in list order.  A pair's result
 * depends on its own cepstra alone.  No atomics. */
int dv3_mcd_max_frames(void);
int dv3_mel_cepstra(const float* mels, const int* lengths, const float* basis, float* cep, int n_seq, int T_max, int M,
                    int K, void* stream);
int dv3_dtw_mcd(const float* cep, int K, const long long* work, float* workspace, float* cost, int* path_len, int P,
                void* stream);

/* ---- pitch of synthesized speech: YIN F0 and the DTW warping path (pitch.cu) ----
 * dv3_yin_frames_per_cta: the frames one CTA of dv3_yin_f0 handles at this tau_max (0 outside [1, 1024]).
 * dv3_yin_f0: YIN F0 (DESIGN.md section 2.18) of frames of several clips in two launches.  blocks: int64 rows
 * (sample_off, n_samples, out0, t0, nf), one per CTA: frames t0 .. t0 + nf - 1 (nf <= dv3_yin_frames_per_cta) of the clip
 * of n_samples samples at wav + sample_off, written at rows out0 .. of f0, aperiodicity and energy.  Frame t reads
 * samples t R + R - W/2 - floor((W + tau_max)/2) + m, m < W + tau_max, zero outside [0, n_samples).  f0 in Hz (0:
 * unvoiced or below the gate), aperiodicity = d'(tau*), energy = sum of the W squared samples.  clips: int64 rows
 * (out_off, n_frames), one per clip: the second launch sets f0 = 0 where energy < gate * the clip's largest energy.
 * diff: null, or (rows, 2, tau_max) floats that receive d(tau) and d'(tau), tau = 1 .. tau_max, of every frame.
 * 2 <= W <= 4096, 1 <= R <= W, 2 <= tau_min <= tau_max <= 1024, threshold in (0, 1], gate in [0, 1].  A clip's results
 * depend on its own samples alone.  No atomics.
 * dv3_dtw_path: dv3_dtw_mcd (the same work rows, workspace, cost and path_len, bit for bit) that also stores each cell's
 * predecessor, 2 bits (0 diagonal, 1 (i-1, j), 2 (i, j-1)), 16 columns a word: row r's N * ceil(M/16) words start at
 * dirs + path_work[2r] (path_work: int64 (P, 2)).
 * dv3_dtw_backtrace: one thread per work row walks those words from (N, M) to (1, 1) and writes the cells of the path
 * as 0-based int32 (i, j) pairs, last cell first, at path + 2 * path_work[2r + 1] (a slot of N + M - 1 pairs), and their
 * count at path_rows[pair] (L for a finite cost).  On row 1 it moves left and on column 1 up, so the walk stays in the
 * grid even where a non-finite D left codes that point outside it. */
int dv3_yin_frames_per_cta(int tau_max);
int dv3_yin_f0(const float* wav, const long long* blocks, int n_blocks, const long long* clips, int n_clips, float* f0,
               float* aperiodicity, float* energy, float* diff, int W, int R, int tau_min, int tau_max, float threshold,
               float gate, float sample_rate, void* stream);
int dv3_dtw_path(const float* cep, int K, const long long* work, const long long* path_work, float* workspace,
                 unsigned* dirs, float* cost, int* path_len, int P, void* stream);
int dv3_dtw_backtrace(const long long* work, const long long* path_work, const unsigned* dirs, int* path, int* path_rows,
                      int P, void* stream);

/* ---- attention alignments: monotonic alignment search and per-step statistics (align.cu) ----
 * Row b (b < B) is the alignment A[b*stride_b + t*stride_t + j] of steps[b] decoder steps t by tokens[b] tokens j (int32,
 * 1 <= steps[b] <= N_max, 1 <= tokens[b] <= L_max); lp(t, j) = logf(fmaxf(A, 1e-8f)), so a NaN cell counts as the floor.
 * dv3_mas_max_tokens: the largest L_max (1024).
 * dv3_mas_dir_words: the 32-bit direction words of one row, steps * ceil(tokens / 32) (0 for arguments out of range).
 * dv3_mas_forward: Q(0, 0) = lp(0, 0), Q(t, j) = lp(t, j) + max(Q(t-1, j), Q(t-1, j-1)), -inf at every cell off all paths
 * from (0, 0) to (steps - 1, tokens - 1) (j > t or tokens - 1 - j > steps - 1 - t).  Tie rule: where
 * Q(t-1, j) == Q(t-1, j-1) the path stays on token j.  Bit j % 32 of word dirs[dir_off[b] + t*ceil(tokens/32) + j/32] is 1
 * where Q(t, j) is on a path and came from (t-1, j-1).  score[b] = Q(steps - 1, tokens - 1) (-inf when steps < tokens).
 * In the same pass: argmax[b*N_max + t] = the lowest j < tokens with the largest A (NaN cells count as -inf), maxv[b*N_max
 * + t] = that A, coverage[b*L_max + j] = sum_t A (t in increasing order); entries past a row's steps or tokens are not
 * written.  One CTA of roundup(L_max, 32) threads per row, one barrier per step.  stride_t >= L_max; the alignment extent,
 * B*N_max and B*L_max must stay below 2^31.
 * dv3_mas_backtrace: durations[b*L_max + j] = the steps the path of row b spends on token j: >= 1 and summing to steps[b]
 * for j < tokens[b] (also where non-finite cells left bits off the grid), 0 past tokens[b], and all 0 when steps[b] <
 * tokens[b] (no path).  One warp per row.  Both kernels: a row's results depend on its own cells and lengths alone; no
 * atomics. */
int dv3_mas_max_tokens(void);
long long dv3_mas_dir_words(int steps, int tokens);
int dv3_mas_forward(const float* A, long long stride_b, long long stride_t, const int* steps, const int* tokens, int B,
                    int N_max, int L_max, const long long* dir_off, unsigned* dirs, int* argmax, float* maxv,
                    float* coverage, float* score, void* stream);
int dv3_mas_backtrace(const int* steps, const int* tokens, int B, int L_max, const long long* dir_off,
                      const unsigned* dirs, int* durations, void* stream);

/* ---- intelligibility: STOI and ESTOI of clips at 10 kHz (stoi.cu, DESIGN.md section 2.20) ----
 * clips: int64 rows (wav_off, n, frame_off, ola_off, mask_clip), one per clip: n samples at wav + wav_off, with
 * F0 = len(range(0, n - 256, 128)) frames whose per-frame slots start at frame_off (energy, keep, kept_idx; the band
 * envelopes at env + 15 frame_off, band i frame t at i F0 + t; the features at feat + 15 frame_off, frame t band i at
 * 15 t + i); its compacted signal takes (F0 - 1) 128 + 256 floats (0 when F0 = 0) from ola + ola_off on; it uses the
 * keep mask of clip mask_clip, which must have the same n.
 * dv3_stoi_frames: one CTA per clip: energy (fp64 dB) and keep (0 / 1) of every frame, kept_idx = the kept frames in
 * order, kept[c] = their count.  win: the 256 fp64 window values.  n_clips <= 65535.
 * dv3_stoi_overlap_add: the mask clip's kept frames of each clip, windowed by the first 256 floats of table and
 * overlap-added at hop 128 into its compacted signal; frames[c] = max(kept[mask_clip] - 1, 0).  max_samples: the
 * largest compacted capacity of any clip.
 * dv3_stoi_bands: blocks: int32 (clip, t0) rows, one per CTA of 8 frames t0 .. t0 + 7 (those < frames[clip] are done).
 * table: the fft_any.cuh table of N = 512 (3 * 512 + 2 floats) whose window is the 256-point one followed by 256 zeros;
 * bands: int32 lo[15] then hi[15], band i summing bins [lo_i, hi_i) < 256.  env: X[i, t]; feat: null, or
 * 10 log10(max(X^2, 1e-10)).  n_blocks = 0 launches nothing.
 * dv3_stoi_segments: pairs: int64 rows (clean clip, processed clip, path_off, seg_off); pair p has steps[p] path
 * steps, int32 (i, j) frame pairs at path + 2 path_off, and max(steps[p] - 29, 0) segments whose (stoi band sum,
 * estoi) fp64 values go to seg + 2 seg_off.  blocks: int32 (pair, s0) rows, one per CTA of 4 segments s0 .. s0 + 3.
 * Then result[2p] = STOI, result[2p + 1] = ESTOI (NaN without segments), counts[2p] = segments, counts[2p + 1] =
 * kept[clean clip].  n_blocks = 0 runs the second launch alone.
 * Every sum has a fixed order and there are no atomics: a pair's results depend on its own clips alone. */
int dv3_stoi_frames(const float* wav, const long long* clips, int n_clips, const double* win, double* energy, int* keep,
                    int* kept_idx, int* kept, void* stream);
int dv3_stoi_overlap_add(const float* wav, const long long* clips, int n_clips, long long max_samples,
                         const float* table, const int* kept_idx, const int* kept, float* ola, int* frames,
                         void* stream);
int dv3_stoi_bands(const float* ola, const long long* clips, const int* blocks, int n_blocks, const float* table,
                   const int* bands, const int* frames, float* env, float* feat, void* stream);
int dv3_stoi_segments(const float* env, const long long* clips, const long long* pairs, int n_pairs, const int* blocks,
                      int n_blocks, const int* path, const int* steps, const int* kept, double* seg, double* result,
                      int* counts, void* stream);

/* ---- token recognition: CTC loss and gradient, greedy CTC decoding, edit distance (ctc.cu, DESIGN.md section 2.21) ----
 * Logits z[b*stride_b + v*stride_v + t] of B rows, V classes (2 <= V <= dv3_ctc_max_vocab() = 1024) and T frames
 * (stride_v >= T; rows do not overlap).  Class 0 is the CTC blank.  Row b has frames[b] in [1, T] frames and
 * target_lengths[b] in [0, L] int32 targets in [1, V) at targets[b*tgt_stride + k]; 1 <= L <= 1024; B*V*T < 2^31.
 * dv3_ctc_ws_bytes: the workspace of dv3_ctc_fwd / dv3_ctc_bwd (0 for arguments out of range).
 * dv3_ctc_fwd: lse[b, t] = the fp64 log-sum-exp of z over V, then the fp64 alpha recursion (one CTA per row, one
 * barrier per frame) -> nll[b] = -log p_b and partials[b] = -log p_b / max(L_b, 1) (fp32).  A row without a feasible
 * path (frames < L_b + repeated adjacent labels, or log p = -inf) gets nll = partials = 0 and infeasible[b] = 1
 * (0 otherwise).  A length or target id out of range sets *err_flag = 1 and leaves the row out the same way.
 * dv3_ctc_bwd: dz (B, V, T) dense = d_loss[0] * scale / max(L_b, 1) * (softmax(z[b, :, t]) - the state occupancies
 * of class v) for t < frames[b], 0 past it and for every row the forward left out; ws as dv3_ctc_fwd left it.
 * dv3_ctc_greedy: hyps (B, T) int32 dense: row b's first hyp_lengths[b] entries are the per-frame argmax classes (ties
 * to the lowest index) over t < frames[b] with repeats collapsed and blanks dropped.
 * dv3_edit_ws_ints: the int32 workspace of dv3_edit_distance for P pairs of hypotheses up to M_max tokens.
 * dv3_edit_distance: pair p compares hyp[p*hyp_stride + j], j < hyp_len[p] <= M_max <= 65535, with reference
 * ref[p*ref_stride + i], i < ref_len[p] <= N_max <= 1024 -> out[4p..4p+3] = (Levenshtein distance, substitutions,
 * deletions, insertions) along the path whose ties prefer the diagonal, then the deletion, then the insertion.
 * One warp per pair.  Every entry point: no atomics, fixed summation orders, a row's or pair's results depend on its
 * own data alone. */
int dv3_ctc_max_vocab(void);
long long dv3_ctc_ws_bytes(int B, int T, int L);
int dv3_ctc_fwd(const float* z, long long stride_b, long long stride_v, const int* frames, const int* targets,
                long long tgt_stride, const int* target_lengths, int B, int V, int T, int L, void* ws, float* nll,
                float* partials, int* infeasible, int* err_flag, void* stream);
int dv3_ctc_bwd(const float* z, long long stride_b, long long stride_v, const int* frames, const int* targets,
                long long tgt_stride, const int* target_lengths, int B, int V, int T, int L, const void* ws,
                const float* d_loss, float scale, float* dz, void* stream);
int dv3_ctc_greedy(const float* z, long long stride_b, long long stride_v, const int* frames, int B, int V, int T,
                   int* hyps, int* hyp_lengths, int* err_flag, void* stream);
long long dv3_edit_ws_ints(int P, int M_max);
int dv3_edit_distance(const int* hyp, long long hyp_stride, const int* hyp_len, const int* ref, long long ref_stride,
                      const int* ref_len, int P, int M_max, int N_max, int* ws, int* out, int* err_flag,
                      void* stream);

/* ---- neural vocoder (vocoder.cu, DESIGN.md section 2.23) ----
 * Multi-resolution STFT loss, one resolution (n_fft, hop) per dv3_mrstft_loss_fwd call.  spec_y / spec_x: the
 * (B, max_frames, n_fft/2 + 1) complex half spectra (float2) of the generated and the target waveform, as
 * dv3_stft_complex_geom writes them; clip c has lengths[c] in [1, n] samples and its first num_frames(lengths[c])
 * frames count.  ws: dv3_mrstft_ws_doubles(B, max_frames) doubles.  stats (B, 4) fp64 = (sum (A_x - A_y)^2,
 * sum A_x^2, sum |log A_x - log A_y|, frames * bins) over the clip's frames and bins (x the target), with
 * A = sqrt(max(re^2 + im^2, 1e-7)), summed in a fixed order without atomics; an invalid length or a non-finite sum
 * sets *err_flag and stores zeros (the clip then counts 0 in the loss and the gradient).
 * dv3_mrstft_loss_total: stats (M, B, 4) of M resolutions -> clip_loss[c] (fp64, may be NULL) = (1/M) sum_m
 * (sqrt(num/den) + lg/count) and *loss = fp32((1/B) sum_c clip_loss[c]).
 * dv3_mrstft_loss_bwd: dspec (B, max_frames, K) float2 = dL/dX of the generated spectrum for d_loss[0] = dL, every
 * bin written (0 past a clip's frames); adjoint = 1 writes instead the spectrum whose dv3_istft_geom is dL/dy:
 * N dL/dX / 2 at 0 < k < N/2, N Re(dL/dX) at k = 0 and N/2.
 * dv3_vocoder_gather: for each of B rows, cond[b, k, s] = lin[b, starts[b] + s, k] (lin (B, lin_rows, K) as
 * dv3_stft_mel_geom writes it, frames[b] valid rows) and target[b, u] = fp32(x[p] - preemph x[p-1]) (fp64 arithmetic)
 * at p = starts[b] hop - (n_fft - hop)/2 + u, u < S hop, x = wav row b (pitch samples, lengths[b] valid), zero outside
 * the clip.  A start outside [0, frames[b] - S] sets *err_flag and writes zeros for the row.  The spectrogram is
 * transposed through shared-memory tiles: reads and writes are coalesced.
 * dv3_interleave: in (B, s*C, T) rows ordered (j, c) -> out (B, C, s*T), out[b,c,s*t+j] = in[b,j*C+c,t], s in
 * [2, 8]; inverse = 1 undoes it. */
long long dv3_mrstft_ws_doubles(int B, int max_frames);
int dv3_mrstft_loss_fwd(const float* spec_y, const float* spec_x, const int* lengths, int n, int B, int max_frames,
                        int n_fft, int hop, double* ws, double* stats, int* err_flag, void* stream);
int dv3_mrstft_loss_total(const double* stats, int M, int B, double* clip_loss, float* loss, void* stream);
int dv3_mrstft_loss_bwd(const float* spec_y, const float* spec_x, const double* stats, int B, int max_frames,
                        int n_fft, int hop, int M, const float* d_loss, int adjoint, float* dspec, void* stream);
int dv3_vocoder_gather(const float* lin, int lin_rows, const int* frames, const float* wav, long long pitch,
                       const int* lengths, const int* starts, int B, int S, int n_fft, int hop, double preemph,
                       float* cond, float* target, int* err_flag, void* stream);
int dv3_interleave(const float* in, float* out, int B, int C, int T, int stride, int inverse, void* stream);

#ifdef __cplusplus
}
#endif
#endif /* DV3B200_H */
