/* fadtk_b200 - C ABI of the H100-native (sm_90a) Frechet-Audio-Distance hot path.
 *
 * The reference (microsoft/fadtk) has no native layer: its hot path is Python calling
 * third-party PyTorch models and numpy/scipy.  This header is the boundary a maintainer
 * binds instead (ctypes stub in INTEGRATION.md); every entry point names the reference code
 * it replaces.  Conventions:
 *   - extern "C", plain C types, no C++ exceptions cross the boundary;
 *   - every function returns 0 on success, non-zero on failure with a message available from
 *     fad_last_error() (thread-local);
 *   - all data buffers are CALLER-OWNED DEVICE pointers (e.g. torch.Tensor.data_ptr()) unless
 *     the parameter name ends in _host; `stream` is a cudaStream_t passed as void*;
 *   - a fad_handle belongs to one device and must not be used from two threads at once;
 *     distinct handles are independent;
 *   - a fad_*_load checks all its arguments before it frees the model loaded before: a rejected
 *     call changes nothing.  A CUDA failure while the new model is built leaves no model loaded,
 *     and its forward fails until a load succeeds;
 *   - there is NO CPU fallback: without a CUDA device every compute entry point fails.
 */
#ifndef FADTK_B200_H
#define FADTK_B200_H

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

typedef struct fad_handle fad_handle;

/* ---- library ------------------------------------------------------------------------ */
int         fad_version(void);
const char* fad_last_error(void);

/* One handle per (process, device).  max_examples bounds the number of 0.96-s VGGish examples
 * processed per internal batch (workspace ~0.7 MB per example). */
int  fad_create(int device, int max_examples, fad_handle** out);
int  fad_destroy(fad_handle* h);

/* ---- VGGish embedder: replaces VGGishModel.load_model/_get_embedding ------------------
 * (fadtk/model_loader.py:89-108 -> torchvggish front-end + VGG stack) and the float32 ->
 * float16 conversion of ModelLoader.get_embedding (fadtk/model_loader.py:40-50). */
typedef struct {
    const float*    conv1_w_host;   /* [64, 9]  fp32                                      */
    const float*    conv1_b_host;   /* [64]                                               */
    const uint16_t* conv_w_host[5]; /* conv2..conv6: fp16 [Cout, 9*Cin], k=(kh*3+kw)*Cin+c */
    const float*    conv_b_host[5];
    const uint16_t* fc_w_host[3];   /* fc1..fc3: fp16 [out, in]                           */
    const float*    fc_b_host[3];
    /* bit i set (i = 0..7: conv2, conv3_1, conv3_2, conv4_1, conv4_2, fc1, fc2, fc3): that layer's
     * weights are an fp16 hi/lo pair W = Wh + Wl stored as [2*Cout, K] with the 128 hi rows of
     * each 128-channel tile followed by its 128 lo rows.  fp16-only weights are a fixed model
     * perturbation worth ~1.4e-4 relative on FAD (DESIGN.md), the split removes it. */
    uint32_t        split_mask;
} fad_vggish_weights;

int fad_vggish_load(fad_handle* h, const fad_vggish_weights* w);

/* Examples (rows of the embedding) produced by a clip of n_samples at 16 kHz:
 * 1 + floor((T - 96) / 96) with T = 1 + floor((n_samples - 400) / 160); 0 if too short. */
long long fad_vggish_num_examples(long long n_samples);

/* Host-side planning: clip_offsets_host[n_clips + 1] (sample offsets into one flat PCM
 * buffer) -> start sample of every example.  Returns the number of examples; writes at most
 * `capacity` entries to ex_start_host (pass NULL/0 to only count).  rows_per_clip_host (may be
 * NULL) receives the per-clip example counts. */
long long fad_vggish_plan(const long long* clip_offsets_host, long long n_clips,
                          long long* ex_start_host, long long capacity,
                          long long* rows_per_clip_host);

/* pcm: int16 mono 16 kHz (device).  ex_start: int64 [n_examples] (device).
 * emb_out: fp16 [n_examples, 128] (device) - exactly what the reference caches as .npy. */
int fad_vggish_forward(fad_handle* h, const int16_t* pcm, const long long* ex_start,
                       long long n_examples, void* emb_out_f16, void* stream);

/* Stage-level entry points (used by the parity tests and profiling). */
int fad_vggish_logmel(fad_handle* h, const int16_t* pcm, const long long* ex_start,
                      long long n_examples, float* logmel_out /* [n,96,64] */, int use_double,
                      void* stream);
/* conv1 of the VGG stack alone (3x3, 1 -> 64, pad 1, + bias, ReLU, 2x2 max-pool; CUDA-core fp32 stencil) with the
 * loaded weights: logmel fp32 [n, 96, 64] -> fp16 NHWC [n, 48, 32, 64]. */
int fad_vggish_conv1(fad_handle* h, const float* logmel, long long n_examples, void* out_f16, void* stream);
/* One tensor-core layer: 3x3 conv pad 1 (taps = 9) or fully connected (taps = 1, H = W = 1) on
 * NHWC fp16 input x[NB,H,W,Cin] with fp16 weights w[Cout, taps*Cin] (split_w = 0) or fp16 hi/lo tiles
 * w[2*Cout, taps*Cin] laid out as in fad_vggish_weights.split_mask (split_w = 1); any other split_w fails and
 * launches nothing.  Fused bias, optional ReLU, optional 2x2 max-pool; fp16 NHWC output (and optional fp32 copy of
 * the un-pooled output). */
int fad_umma_layer(fad_handle* h, const void* x_f16, int NB, int H, int W, int Cin,
                   const void* w_f16, const float* bias, int Cout, int taps, int relu, int pool,
                   int split_w, void* out_f16, float* out_f32_or_null, void* stream);
/* The Linear / 1-D convolution GEMM every transformer and Encodec layer runs (csrc/clap_host.inc clap_gemm):
 *   C = act(A W^T + bias), act 0 none, 1 ReLU, 2 GELU (erf form), 3 ELU (alpha = 1).
 * a_f16: fp16 rows of k_cols elements, row r starting at a_f16 + r * lda (lda = 0: k_cols; lda < k_cols gives
 * overlapping rows); w_f16: [2 * pad128(n_cols), pad64(k_cols)] fp16 hi/lo tiles (split_w = 1, see
 * weights.split_hi_lo_tiles) or [pad128(n_cols), pad64(k_cols)] fp16 (split_w = 0); bias: fp32 [pad128(n_cols)].
 * Outputs (any of them may be NULL): out_f16 / out_f32 [rows, n_cols]; resid fp32 [tokens, resid_C]:
 * resid[token(r)][0:resid_C] += C[r][0:resid_C], token(r) = r (resid_res = 0) or the token of window-ordered row r
 * of resid_res x resid_res images in 8 x 8 windows cyclically shifted by resid_shift.
 * k_cols, n_cols and lda must be multiples of 8, resid_C a multiple of 32 and at most n_cols, every pointer
 * 16-byte aligned; otherwise the call fails and launches nothing.  With split_w = 1 every call first checks, on the
 * stream and synchronously, whether the lo parts are all zero (weights exact in fp16): the truncation compensation
 * depends on it. */
int fad_linear(fad_handle* h, const void* a_f16, long long rows, int k_cols, long long lda, const void* w_f16,
               int split_w, const float* bias, int n_cols, int act, void* out_f16, float* out_f32,
               float* resid, int resid_C, int resid_res, int resid_shift, void* stream);

/* ---- CLAP-LAION audio embedder (HTSAT-tiny): replaces CLAPLaionModel.load_model/_get_embedding
 * (fadtk/model_loader.py:382-418 -> laion_clap.CLAP_Module + torchlibrosa front-end).
 * tensors_host: 180 (HTSAT-tiny = clap-laion-audio) or 258 (HTSAT-base = clap-laion-music,
 * model_loader.py:385) host pointers in the order documented at the top of csrc/clap_host.inc; the count
 * selects the variant
 * (produced by fadtk_b200/weights_clap.py).  max_chunks bounds the 10-s windows per internal batch
 * (~12 MB of workspace each). */
int fad_clap_load(fad_handle* h, const void* const* tensors_host, int n_tensors, int max_chunks);

/* Windows of a clip: one every 48 000 samples (range(0, T, sr), model_loader.py:396-398), each
 * covering up to 480 000 samples and zero padded.  Returns the number of windows; fills
 * chunk_start_host (sample offset into the flat PCM buffer) and chunk_valid_host (samples available). */
long long fad_clap_plan(const long long* clip_offsets_host, long long n_clips, long long* chunk_start_host,
                        int* chunk_valid_host, long long capacity, long long* rows_per_clip_host);

/* Frame pool: windows of one clip are 1-s shifts of the same audio, so every STFT frame that does
 * not touch a window edge is shared by up to ten windows.  fad_clap_plan_frames lists each DISTINCT
 * frame once - pool_start (sample offset of the window it is taken from), pool_valid, pool_frame
 * (frame index inside that window) - and fills frame_index [n_chunks][1001]: pool row of every
 * (window, frame).  Returns the pool size (pass NULL outputs to only count). */
long long fad_clap_plan_frames(const long long* clip_offsets_host, long long n_clips, long long* pool_start_host,
                               int* pool_valid_host, int* pool_frame_host, long long pool_capacity,
                               int* frame_index_host);

/* pcm: int16 mono 48 kHz; pool_* [n_pool] and frame_index [n_chunks*1001] from fad_clap_plan_frames (all
 * device).  emb_out: fp16 [n_chunks, 512], L2-normalised - what the reference caches as .npy. */
int fad_clap_forward(fad_handle* h, const int16_t* pcm, const long long* pool_start, const int* pool_valid,
                     const int* pool_frame, long long n_pool, const int* frame_index, long long n_chunks,
                     void* emb_out_f16, void* stream);
/* stage entry point: BatchNorm-ed log-mel rows [n_pool, 64] fp32 */
int fad_clap_logmel(fad_handle* h, const int16_t* pcm, const long long* pool_start, const int* pool_valid,
                    const int* pool_frame, long long n_pool, float* out, void* stream);
/* Stage entries of the loaded CLAP model (parity tests), each calling the launch code of fad_clap_forward and
 * failing, before launching or writing anything, on arguments it could not honour; so do fad_clap_logmel and
 * fad_clap_forward (n_pool, n_chunks >= 0; a pointer may be NULL only when its count is 0).  B in [1, max_chunks];
 * device pointers the kernels read or write aligned to their element size (the streams x / out are only copied and
 * may have any alignment).  E = 96 (HTSAT-tiny) or 128 (HTSAT-base); the stream entering
 * stage s is [B][res^2][C] with res = 64 >> s, C = E << s.
 * fad_clap_patch_embed: pool fp32 [n_pool][64] (fad_clap_logmel's rows), frame_index [B][1001] with every value in
 * [0, n_pool) (not checked: it lives on the device) -> x_out fp32 [B][4096][E].
 * fad_clap_block: Swin block blk in [0, 12 | 18) (stage-major), x fp32 [B][res^2][C] -> out fp32 [B][res^2][C].
 * fad_clap_merge: patch merge s in {0, 1, 2}, x fp32 [B][res^2][C] -> out fp32 [B][res^2 / 4][2 C].
 * fad_clap_head: x fp32 [B][64][8 E] -> out fp16 [B][512], L2-normalised. */
int fad_clap_patch_embed(fad_handle* h, const float* pool, long long n_pool, const int* frame_index, long long B,
                         float* x_out, void* stream);
int fad_clap_block(fad_handle* h, int blk, const float* x, long long B, float* out, void* stream);
int fad_clap_merge(fad_handle* h, int s, const float* x, long long B, float* out, void* stream);
int fad_clap_head(fad_handle* h, const float* x, long long B, void* out_f16, void* stream);

/* ---- Whisper: replaces WhisperModel.load_model / _get_embedding (fadtk/model_loader.py:657-669):
 * WhisperFeatureExtractor (clip padded / truncated to 30 s, log-mel 80 x 3000) and
 * transformers.WhisperModel(input_features, decoder_input_ids = [[sot, sot]]).last_hidden_state.
 * cfg: {d_model, heads (= d_model / 64), encoder layers, decoder layers, ffn dim}; tensors_host: host pointers in
 * the order documented at the top of csrc/whisper_host.inc (5 + 12 L_enc + 3 + 20 L_dec + 2), packed by
 * fadtk_b200/weights_whisper.py.  max_clips bounds the clips per launch sequence (45 MB of workspace each at
 * d_model = 768). */
int fad_whisper_load(fad_handle* h, const int* cfg, const void* const* tensors_host, int n_tensors, int max_clips);
/* pcm: int16 mono 16 kHz; clip_start int64 / clip_len int32 [n_clips] (all device).
 * emb_out: fp16 [n_clips][2][d_model]. */
int fad_whisper_forward(fad_handle* h, const int16_t* pcm, const long long* clip_start, const int* clip_len,
                        long long n_clips, void* emb_out_f16, void* stream);
/* stage entry point: out = fp32 [n_clips*3000*80] log10 mel (time-major) followed by [n_clips] per-clip maxima;
 * the features are (max(x, max - 8) + 4) / 4. */
int fad_whisper_logmel(fad_handle* h, const int16_t* pcm, const long long* clip_start, const int* clip_len,
                       long long n_clips, float* out, void* stream);
/* Stage entries of the loaded Whisper model (parity tests), each calling the launch code of fad_whisper_forward and
 * failing, before launching or writing anything, on arguments it could not honour.  B in [1, max_clips]; 16-byte
 * aligned device pointers.
 * fad_whisper_conv: conv c of the stem.  c = 0: x fp32 [B][3000][80] raw log10 mel (as fad_whisper_logmel returns it)
 * and clip_max fp32 [B] -> floor, (x + 4) / 4, conv1 + GELU -> out fp16 [B][3000][d];  c = 1: x fp16 [B][3000][d]
 * (conv 0's output; clip_max unused) -> out fp32 [B][1500][d] = embed_positions + GELU(conv2(x)).
 * fad_whisper_enc_layer: encoder layer l in [0, enc_layers), x fp32 [B][1500][d] -> out fp32 [B][1500][d].
 * fad_whisper_encode: the whole encoder including encoder.layer_norm for n_clips >= 1 clips (any count, run in chunks of
 * max_clips) -> out fp16 [n_clips][1500][d], the encoder output the decoder reads.
 * fad_whisper_dec_layer: decoder layer l in [0, dec_layers), xd fp32 [B][2][d] and enc_out fp16 [B][1500][d] ->
 * out fp32 [B][2][d]. */
int fad_whisper_conv(fad_handle* h, int c, const void* x, const float* clip_max, long long B, void* out, void* stream);
int fad_whisper_enc_layer(fad_handle* h, int l, const float* x, long long B, float* out, void* stream);
int fad_whisper_encode(fad_handle* h, const int16_t* pcm, const long long* clip_start, const int* clip_len,
                       long long n_clips, void* out_f16, void* stream);
int fad_whisper_dec_layer(fad_handle* h, int l, const float* xd, const void* enc_out_f16, long long B, float* out,
                          void* stream);

/* ---- Encodec: replaces EncodecEmbModel.load_model / _get_frame for the 24 kHz variant
 * (fadtk/model_loader.py:123-130, 155-166): EncodecModel.encodec_model_24khz().encoder(audio) -> [T/320, 128].
 * tensors_host: 78 host pointers in the order documented at the top of csrc/encodec_host.inc, packed by
 * fadtk_b200/weights_encodec.py (weight-norm folded, im2col column order, fp16 hi/lo tiles).
 * variant 0: encodec_model_24khz (causal, mono, whole file); 1: encodec_model_48khz (non-causal, GroupNorm(1, C)
 * after every conv, the mono file duplicated to stereo; the caller passes the 1-s segments of :139-152 as clips).
 * max_chunk_samples bounds clips x samples per convolution chunk (0.55 KB of workspace per sample). */
int fad_encodec_load(fad_handle* h, const void* const* tensors_host, int n_tensors, long long max_chunk_samples, int variant);
/* pcm: int16 mono 24 kHz [n_clips][T] (device), all clips of one call have the same length T.
 * emb_out: fp16 [n_clips][ceil(T/320)][128] (device). */
int fad_encodec_forward(fad_handle* h, const int16_t* pcm, long long n_clips, int T, void* emb_out_f16, void* stream);
/* Stage entries (parity tests) of the loaded encoder; each calls the launch code fad_encodec_forward calls and fails,
 * launching nothing, on arguments it could not honour.  16-byte aligned device pointers.
 * fad_encodec_conv: conv `layer` in the order of the load (0 input conv; 1 + 4 s, 2 + 4 s, 3 + 4 s, 4 + 4 s the k = 3
 * conv, k = 1 conv, shortcut and down conv of stage s; 17 the last conv) with the variant's padding.  x fp32
 * [B][T_in][Cin] (ELU applied to it first if elu_in) -> out fp32 [B][ceil(T_in / stride)][Cout]; groupnorm != 0 (48 kHz
 * model only) applies the GroupNorm(1, Cout) that follows the conv.  B in [1, 4096], B * T_in <= max_chunk_samples.
 * fad_encodec_lstm: z fp32 [n_clips][TF][512] -> out fp32 [n_clips][TF][512] = LSTM(z) + z (two layers), in groups of
 * 512 clips; TF at most the frames of max_chunk_samples. */
int fad_encodec_conv(fad_handle* h, int layer, const float* x_f32, long long B, int T_in, int elu_in, int groupnorm,
                     float* out_f32, void* stream);
int fad_encodec_lstm(fad_handle* h, const float* z_f32, long long n_clips, int TF, float* out_f32, void* stream);

/* ---- wav2vec 2.0 / HuBERT / MERT: replaces W2V2Model, HuBERTModel, MERTModel load_model / _get_embedding
 * (fadtk/model_loader.py:254-288, 525-596) for the "group-norm feature encoder + post-LN transformer" checkpoints
 * (wav2vec2-base-960h, hubert-base-ls960, MERT-v1-95M): processor normalisation, Wav2Vec2Model / HubertModel
 * forward with output_hidden_states, hidden_states[layer].
 * cfg: {d_model, heads (= d_model / 64), layers, ffn}; tensors_host in the order of csrc/wav2vec_host.inc
 * (39 + 12 layers), packed by fadtk_b200/weights_w2v.py. */
int fad_w2v_load(fad_handle* h, const int* cfg, const void* const* tensors_host, int n_tensors, int max_clips, int max_len);
/* pcm: int16 mono [n_clips][L] (device), equal lengths; emb_out: fp16 [n_clips][frames(L)][d_model]. */
int fad_w2v_forward(fad_handle* h, const int16_t* pcm, long long n_clips, int L, int layer, void* emb_out_f16, void* stream);
/* Several layers of one forward.  taps: host int[n_taps], strictly increasing, each in [0, layers]; out: fp16
 * [n_taps][n_clips][frames(L)][d_model], 16-byte aligned, slice t = hidden_states[taps[t]], bitwise what
 * fad_w2v_forward(..., taps[t], ...) writes.  The encoder runs once per max_clips chunk, up to the deepest tap.
 * Fails, launching nothing and writing nothing, on a missing load, null pcm / taps / out, n_clips < 1,
 * n_taps outside [1, layers + 1], taps out of order or range, a misaligned out, or L outside [400, max_len]. */
int fad_w2v_forward_taps(fad_handle* h, const int16_t* pcm, long long n_clips, int L, const int* taps, int n_taps,
                         void* out_f16, void* stream);
/* Stage entries (parity tests); each calls the launch code fad_w2v_forward calls and fails, launching nothing and
 * writing nothing, on arguments it could not honour.  B in [1, max_clips]; 16-byte aligned device pointers.
 * fad_w2v_normalize (no load needed): pcm int16 [n_clips][L] -> out fp32 [n_clips][L], (x - mean) / sqrt(var + 1e-7).
 * fad_w2v_conv: feature-encoder conv c in [0, 7) of the loaded variant at the frames T_c of clips of L samples
 * (400 <= L <= max_len): c = 0 x fp32 [B][L] (normalised) -> out fp16 [B][T_1][512]; c = 1..5 x fp16 [B][T_c][512] ->
 * out fp16 [B][T_c+1][512]; c = 6 -> out fp32 [B][T_7][512].
 * fad_w2v_posconv: x fp32 [B][S][d] -> out = x + GELU(pos_conv(x)), S in [1, frames(max_len)].
 * fad_w2v_layer: encoder layer l in [0, layers), x fp32 [B][S][d] the stream entering it (post-LN: the previous
 * LayerNorm's output; pre-LN: the raw stream) -> out fp32 [B][S][d] the stream leaving it. */
int fad_w2v_normalize(fad_handle* h, const int16_t* pcm, long long n_clips, int L, float* out_f32, void* stream);
int fad_w2v_conv(fad_handle* h, int c, const void* x, long long B, int L, void* out, void* stream);
int fad_w2v_posconv(fad_handle* h, const float* x_f32, long long B, int S, float* out_f32, void* stream);
int fad_w2v_layer(fad_handle* h, int l, const float* x_f32, long long B, int S, float* out_f32, void* stream);

/* ---- statistics: replaces calc_embd_statistics (fadtk/fad.py:42-48) and
 * _process_file / calculate_embd_statistics_online (fadtk/utils.py:13-46) ----------------
 * Packed fp64 accumulator of length fad_stats_acc_len(d):
 *   acc[0] = n, acc[1..d] = sum(x - shift) (exact), acc[1+d..1+d+d*d) = sum y y^T (d x d),
 *   acc[1+d+d*d..] = sum y,   y = x - shift (the same values as acc[1..d])
 * It is additive: accumulate batches into it, all-reduce (sum) it across GPUs, then finalize.
 * `shift` (fp16 [d], device) must be identical for every contribution to one accumulator. */
size_t fad_stats_acc_len(int d);
/* tensor_core = 0 (default everywhere in the product): E^T E on the FP64 TENSOR pipe (mma.sync
 * m8n8k4 f64 -> DMMA): the products (x - s)(x - s)^T of fp16 data are exact in fp64 and the
 * accumulation is fp64 in a fixed order, so the result is the Gram matrix of the data to ~1e-16,
 * positive semi-definite and bit-reproducible (rank-deficient per-song sets and covariances with
 * cond ~1e9 need that, DESIGN.md section 5.4).
 * tensor_core = 2: the same exact arithmetic on the CUDA cores (DFMA + fp64 atomics): verification.
 * Any other value fails and launches nothing. */
int fad_stats_accumulate(fad_handle* h, const void* emb_f16, long long n_rows, int d,
                         const void* shift_f16, double* acc, int tensor_core, void* stream);
/* ---- multi-GPU: the ONE exchange step of the path (SURVEY.md section 8 (e)) ----------
 * Ranks embed disjoint shards of the clips and accumulate with the SAME shift vector; the packed accumulators are
 * then summed over NVLink and every rank finalises identical statistics.  The reference has no counterpart (it is
 * single-device); this replaces the pickled per-file scatter matrices of its process map (fadtk/utils.py:35-45).
 * NCCL is loaded at run time (dlopen of libnccl.so.2, or $FADTK_NCCL_LIB); nothing is linked.
 *   fad_comm_unique_id   rank 0 creates the 128-byte rendezvous id (ncclGetUniqueId); the host ships it to the
 *                        other ranks however it likes (file, MPI, torch.distributed, a socket)
 *   fad_comm_init        every rank joins; the communicator belongs to the handle
 *   fad_stats_allreduce  in-place sum of acc[fad_stats_acc_len(d)] on `stream`; nccl_comm_or_null = an existing
 *                        ncclComm_t of the host application, or NULL for the handle's own communicator
 *   fad_allreduce_sum_f64  the same for any fp64 device buffer (e.g. both datasets packed into one call) */
#define FAD_COMM_ID_BYTES 128
int fad_comm_unique_id(void* id_out_host);
int fad_comm_init(fad_handle* h, const void* id_host, int rank, int world);
int fad_comm_destroy(fad_handle* h);
int fad_stats_allreduce(fad_handle* h, void* nccl_comm_or_null, double* acc, int d, void* stream);
int fad_allreduce_sum_f64(fad_handle* h, void* nccl_comm_or_null, double* buf, long long n_values, void* stream);

/* The reference's DIRECTORY statistics (per-file np.mean rounded to fp16, per-file scatter, Chan merge:
 * fadtk/utils.py:13-46) for n_files files of rows_per_file rows each, without leaving the device:
 *   fad_file_means               m64[f], m16[f] (fp64 rows [n_files, d]): the exact mean of file f and its mean as the
 *                                reference's _process_file returns it (fp32 accumulation rounded to fp16)
 *   fad_stats_accumulate_f64     exact Gram statistics (DMMA) of fp64 rows, unshifted, into a packed accumulator
 *   fad_stats_finalize_mirrored  (mu, cov) exactly as calculate_embd_statistics_online returns them, from the packed
 *                                accumulators of the rows, of m64 and of m16 (all three additive: all-reduce them first);
 *                                rows_per_file == 1 gives the reference's all-NaN covariance (utils.py:16) */
int fad_file_means(fad_handle* h, const void* emb_f16, long long n_files, int rows_per_file, int d,
                   double* m64_out, double* m16_out, void* stream);
int fad_stats_accumulate_f64(fad_handle* h, const double* rows, long long n_rows, int d, double* acc, void* stream);
int fad_stats_finalize_mirrored(fad_handle* h, const double* acc, const double* acc_means64, const double* acc_means16,
                                const void* shift_f16, int rows_per_file, int d, double* mu_out, double* cov_out, void* stream);
/* rows emb[idx[i]] for i < n_idx (FAD-inf bootstrap, fadtk/fad.py:333-336) */
int fad_stats_accumulate_gather(fad_handle* h, const void* emb_f16, long long n_src_rows,
                                const long long* idx, long long n_idx, int d,
                                const void* shift_f16, double* acc, void* stream);
int fad_stats_finalize(fad_handle* h, const double* acc, const void* shift_f16, int d,
                       double* mu_out, double* cov_out, void* stream);

/* ---- Frechet distance: replaces calc_frechet_distance (fadtk/fad.py:51-120) ------------
 * mu/cov fp64 device arrays.  out (device, 8 doubles): [0] FAD, [1] tr sqrt(C1 C2),
 * [2] relative residual of the final square root, [3] iterations, [4] |mu1-mu2|^2,
 * [5] tr C1, [6] tr C2, [7] reserved.  iters <= 0 selects the default. */
int fad_frechet(fad_handle* h, const double* mu1, const double* cov1, const double* mu2,
                const double* cov2, int d, int iters, double* out, void* stream);

/* The baseline's square root can be computed once and reused (FAD-inf, per-song scoring):
 * fad_sqrt_psd -> sqrt_out (d*d doubles) and scal_out (2 doubles: |C|_F, tr C), both device. */
int fad_sqrt_psd(fad_handle* h, const double* cov, int d, int iters, double* sqrt_out, double* scal_out,
                 void* stream);
int fad_frechet_presqrt(fad_handle* h, const double* mu1, const double* sqrt1, const double* scal1,
                        const double* mu2, const double* cov2, int d, int iters, double* out, void* stream);

/* Ragged-batched form for per-file scoring: replaces the loop of FrechetAudioDistance.score_individual
 * (fadtk/fad.py:353-395; per file calc_embd_statistics fad.py:42-48 + calc_frechet_distance :51-120).
 * emb_f16: fp16 [N, d] (device); offsets: int64 [n_items + 1] (device), item z = rows
 * [offsets[z], offsets[z+1]).  Per item the mean is rounded to fp16 (np.mean dtype rule) and the
 * covariance is the exact fp64 ddof=1 Gram.  out: fp64 [n_items][8] in fad_frechet's layout with
 * [7] = row count; an item with fewer than two rows gets NaN in [0], [1] (the reference asserts). */
int fad_frechet_batched(fad_handle* h, const double* mu1, const double* sqrt1, const double* scal1,
                        const void* emb_f16, const long long* offsets, long long n_items, int d, int iters,
                        double* out, void* stream);

/* ---- Kernel Audio Distance (KAD, Chung et al. 2025): the reference has no counterpart (a metric beyond fadtk).
 * Unbiased MMD^2 between embedding sets X [m, d] and Y [n, d] under k(a, b) = exp(-|a - b|^2 / (2 sigma^2)), sigma =
 * the median of the pairwise distances of X (DESIGN.md section 5.11).  fp16 rows (the cached embeddings), d a multiple
 * of 8, m, n >= 2, 16-byte-aligned pointers; otherwise the call fails and launches nothing.  Workspace belongs to the
 * handle.  Both results are bitwise reproducible (fixed work units, integer histogram counts, no float atomics).
 *   fad_kad_median_sq  out (device fp64 [2]) = the two middle values of {|x_i - x_j|^2 : i < j} (the same value twice
 *                      when m (m - 1) / 2 is odd), selected exactly among the fp32 values fad_kad_sums uses
 *   fad_kad_sums       z = [X; Y] (fp16 [m + n, d], X first), sigma = device fp64 scalar;
 *                      out (device fp64 [3]) = S_xx (i < j), S_yy (i < j), S_xy (all pairs) of k */
int fad_kad_median_sq(fad_handle* h, const void* x_f16, long long m, int d, double* out, void* stream);
int fad_kad_sums(fad_handle* h, const void* z_f16, long long m, long long n, int d, const double* sigma, double* out,
                 void* stream);
/* Per-song KAD sums against one baseline: z = [X; Y_1; ...; Y_K] (fp16 [m + n_total, d], X first); offsets = device
 * int64 [n_items + 1], song k = rows [offsets[k], offsets[k+1]) of the Y part (offsets[0] = 0, non-decreasing,
 * n_total = offsets[n_items]; read back to the host, so the call synchronises the stream once); sigma = device fp64
 * scalar.  out (device fp64 [1 + 2 n_items]) = S_xx, then per song S_yy,k (i < j within the song), S_xy,k (all pairs
 * with X).  S_xx and the shift are computed once; a song of 0 or 1 rows gets S_yy,k = 0 (and S_xy,k = 0 when empty).
 * Each value is the quantity fad_kad_sums gives for [X; Y_k], bitwise reproducible (fixed work units, no atomics). */
int fad_kad_song_sums(fad_handle* h, const void* z_f16, long long m, const long long* offsets, long long n_items, int d,
                      const double* sigma, double* out, void* stream);
/* The same three computations split over shards of contiguous work units (DESIGN.md section 5.11, sharding); the
 * outputs are bitwise equal to the entries above for any number of shards.
 *   local_shards == 0  collective over nccl_comm_or_null, or the handle's own communicator (fad_comm_init) when NULL;
 *                      rank and size come from the communicator, and every rank gets the whole output.  Every rank
 *                      calls with its own z (the same rows), offsets and sigma.  Before any tile work the ranks compare
 *                      m, n, d, n_items, a digest of the offsets, the bits of sigma, a digest of z and whether each
 *                      rank accepted its arguments; any difference fails the call on every rank with the same message.
 *                      Fails without a communicator.
 *   local_shards >= 1  this device computes the shards 0 .. local_shards - 1 one after another and adds their outputs in
 *                      shard order (the arithmetic of the all-reduce); nccl_comm_or_null must be NULL.  1 = the entries
 *                      above, which are this call.
 * fad_kad_shard_plan (host only): the cut of `units` work units of unit_tiles[u] >= 1 tiles each into `shards`
 * contiguous ranges, shard s = [bounds[s], bounds[s + 1]) (bounds: [shards + 1]); each holds at most total / shards
 * plus one unit's tiles, and shards may be empty when there are more shards than units. */
int fad_kad_median_sq_sharded(fad_handle* h, void* nccl_comm_or_null, int local_shards, const void* x_f16, long long m,
                              int d, double* out, void* stream);
int fad_kad_sums_sharded(fad_handle* h, void* nccl_comm_or_null, int local_shards, const void* z_f16, long long m,
                         long long n, int d, const double* sigma, double* out, void* stream);
int fad_kad_song_sums_sharded(fad_handle* h, void* nccl_comm_or_null, int local_shards, const void* z_f16, long long m,
                              const long long* offsets, long long n_items, int d, const double* sigma, double* out,
                              void* stream);
int fad_kad_shard_plan(const long long* unit_tiles, long long units, int shards, long long* bounds);

/* ---- Precision, recall, density and coverage (PRDC; Kynkaanniemi et al. 2019, Naeem et al. 2020) of an eval set
 * Y [n, d] against a baseline X [m, d] (DESIGN.md section 5.12).  z = [X; Y] (fp16 [m + n, d], X first, 16-byte
 * aligned), d a multiple of 8, q(a, b) = |a - b|^2 computed as for KAD (same shift, split and fp32 q).  Every argument
 * is checked first (null or misaligned pointers, 1 <= k <= 16, m > k and n > k, d, at most 2^30 rows); a rejected call
 * launches nothing and writes nothing.  Both outputs are bitwise reproducible (selected fp32 values, integer counts).
 *   fad_knn_radii_sq  radii_sq (device fp32 [m + n]) = for each row of X, the k-th smallest q to the other rows of X
 *                     (the self pair excluded by index: duplicates are neighbours at 0); then the same for each row of
 *                     Y within Y.  The exact k-th smallest of the fp32 q values the kernel computes.
 *   fad_prdc_counts   radii_sq (device fp32 [m + n], r_i^2 then s_j^2, e.g. from the call above; m, n >= 2) ->
 *                     inside (device int32 [n]) = #{i : q(x_i, y_j) < r_i^2}; flags (device uint8 [m]) = bit 0 when
 *                     some q(x_i, y_j) < r_i^2 (covered), bit 1 when some q(x_i, y_j) < s_j^2 (recalled).  Each xy pair's
 *                     q is computed once. */
int fad_knn_radii_sq(fad_handle* h, const void* z_f16, long long m, long long n, int d, int k, float* radii_sq,
                     void* stream);
int fad_prdc_counts(fad_handle* h, const void* z_f16, long long m, long long n, int d, const float* radii_sq, int* inside,
                    unsigned char* flags, void* stream);
/* The same two passes split over shards of contiguous work units (DESIGN.md section 5.12, sharding over GPUs);
 * local_shards means what it means for fad_kad_*_sharded, and the outputs are bitwise equal to the entries above
 * (which are the local_shards = 1 case) for any number of shards.  Collective calls compare, before any tile work, m, n,
 * d, a digest of z, whether each rank accepted its arguments, and k (radii) or a digest of radii_sq (counts); any
 * difference fails the call on every rank with the same message. */
int fad_knn_radii_sq_sharded(fad_handle* h, void* nccl_comm_or_null, int local_shards, const void* z_f16, long long m,
                             long long n, int d, int k, float* radii_sq, void* stream);
int fad_prdc_counts_sharded(fad_handle* h, void* nccl_comm_or_null, int local_shards, const void* z_f16, long long m,
                            long long n, int d, const float* radii_sq, int* inside, unsigned char* flags, void* stream);
/* Per-song PRDC against one baseline (DESIGN.md section 5.12, per-song PRDC): z = [X; Y_1; ...; Y_K] (fp16
 * [m + n_total, d], X first); offsets = device int64 [n_items + 1], song s = rows [offsets[s], offsets[s+1]) of the Y
 * part (offsets[0] = 0, non-decreasing, n_items >= 1, n_total = offsets[n_items]; read back to the host, so the call
 * synchronises the stream once).  Every song must have more than k rows (the counts: at least 2).  The other checks are
 * fad_knn_radii_sq's (m > k), and int32 outputs are 4-byte aligned; a rejected call launches nothing and writes nothing.
 * Song s's values are the ones fad_knn_radii_sq / fad_prdc_counts give for [X; Y_s], bitwise.
 *   fad_knn_song_radii_sq  radii_sq (device fp32 [m + n_total]) = r_i^2 of X as fad_knn_radii_sq, then for each row of Y
 *                          the k-th smallest q to the other rows of its own song
 *   fad_prdc_song_counts   radii_sq (device fp32 [m + n_total], e.g. from the call above) -> inside (device int32
 *                          [n_total]) = #{i : q(x_i, y_j) < r_i^2}; song_counts (device int32 [n_items][2]) = per song
 *                          #{i : some y_j of the song has q(x_i, y_j) < r_i^2} (covered), then the same with s_j^2
 *                          (recalled)
 * The _sharded forms split the tile work as fad_knn_radii_sq_sharded / fad_prdc_counts_sharded do, bitwise equal for
 * any number of shards; collective calls also compare n_items and a digest of the offsets.  The unsharded entries are
 * the local_shards = 1 case.
 * fad_prdc_song_spans (host only): the counts pass's cut of the songs (host int64 offsets [n_items + 1], every song at
 * least one row) for a baseline of m rows into spans, runs of whole songs in order of at most G * 128 rows (G as
 * fad_prdc_counts chooses its column runs) and at most 512 songs, a longer song alone; spans (host int64
 * [n_items][4]) = {first row, end row, first song, songs} per span, *n_spans = their number. */
int fad_knn_song_radii_sq(fad_handle* h, const void* z_f16, long long m, const long long* offsets, long long n_items,
                          int d, int k, float* radii_sq, void* stream);
int fad_prdc_song_counts(fad_handle* h, const void* z_f16, long long m, const long long* offsets, long long n_items,
                         int d, const float* radii_sq, int* inside, int* song_counts, void* stream);
int fad_knn_song_radii_sq_sharded(fad_handle* h, void* nccl_comm_or_null, int local_shards, const void* z_f16,
                                  long long m, const long long* offsets, long long n_items, int d, int k,
                                  float* radii_sq, void* stream);
int fad_prdc_song_counts_sharded(fad_handle* h, void* nccl_comm_or_null, int local_shards, const void* z_f16,
                                 long long m, const long long* offsets, long long n_items, int d,
                                 const float* radii_sq, int* inside, int* song_counts, void* stream);
int fad_prdc_song_spans(const long long* offsets, long long n_items, long long m, long long* spans, long long* n_spans);
/* Per-sample realism (Kynkaanniemi et al. 2019) and nearest baseline row of each eval row (DESIGN.md section 5.13):
 * z = [X; Y] (fp16 [m + n, d], X first, 16-byte aligned), d a multiple of 8, q as for PRDC.  Every argument is checked
 * first (null or misaligned pointers, 1 <= k <= 16, m > k, n >= 1, d, at most 2^30 rows); a rejected call launches
 * nothing and writes nothing.  The radii are read back to the host, so the call synchronises the stream once.
 *   kept_radii_sq (device fp32 [m]) = r~_i^2: r_i^2, the radius fad_knn_radii_sq gives row i of X (bitwise), where
 *                 r_i^2 <= T and 0 otherwise; T = numpy.median of the m values r_i^2 in fp64 (for even m the fp64 mean of
 *                 the two middle values), also written to *threshold_sq (host fp64)
 *   realism       (device fp32 [n]) = sqrt(max_i r~_i^2 / q(x_i, y_j)) over the rows with r~_i^2 > 0: +inf where such a
 *                 row has q = 0, 0 where every r~_i^2 is 0 (fl(sqrt(max_i fl(r~_i^2 / q))), exactly)
 *   nearest       (device int32 [n]) = argmin_i q(x_i, y_j) over all rows of X, ties to the smallest i;
 *   nearest_sq    (device fp32 [n]) = that q
 * All outputs are bitwise reproducible and depend on y_j and X alone.  fad_realism_sharded splits the tile work as
 * fad_knn_radii_sq_sharded does (local_shards as for fad_kad_*_sharded; collective calls compare m, n, d, k and a digest
 * of z), bitwise equal to fad_realism, which is its local_shards = 1 case. */
int fad_realism(fad_handle* h, const void* z_f16, long long m, long long n, int d, int k, float* kept_radii_sq,
                float* realism, int* nearest, float* nearest_sq, double* threshold_sq, void* stream);
int fad_realism_sharded(fad_handle* h, void* nccl_comm_or_null, int local_shards, const void* z_f16, long long m,
                        long long n, int d, int k, float* kept_radii_sq, float* realism, int* nearest, float* nearest_sq,
                        double* threshold_sq, void* stream);
/* The k nearest distinct baseline groups of each eval row (DESIGN.md section 5.14): z = [X; Y] (fp16 [m + n, d], X first,
 * 16-byte aligned), d a multiple of 8, q as for PRDC.  The baseline is cut into groups by base_offsets (device int64
 * [n_groups + 1], 8-byte aligned: offsets[0] = 0, non-decreasing, offsets[n_groups] = m; empty groups allowed), group g =
 * rows [offsets[g], offsets[g + 1]) of X; base_offsets = NULL makes every row its own group (a plain k-NN; n_groups is
 * then ignored).  Every argument is checked first (null or misaligned pointers, 1 <= k <= 16, m >= 1, n >= 1, d, at most
 * 2^30 rows, the offsets read back once); a rejected call launches nothing and writes nothing.
 *   nearest    (device int32 [n][k]): for eval row j, the rows of X ordered by the key (q(x_i, y_j), i); each group is
 *              represented by its smallest key; the k groups with the smallest representative keys, ascending, each as
 *              the row i of that key; -1 where fewer than k groups are non-empty
 *   nearest_sq (device fp32 [n][k]) = those q values (+inf for the empty slots)
 * With k = 1 and no offsets, the outputs are bitwise fad_realism's nearest and nearest_sq.  All outputs are bitwise
 * reproducible and depend on y_j and X (and its groups) alone.  fad_nearest_sharded splits the tile work as
 * fad_realism_sharded does (local_shards as for fad_kad_*_sharded; collective calls compare m, n, d, k, the number of
 * groups, a digest of the offsets and a digest of z), bitwise equal to fad_nearest, which is its local_shards = 1 case. */
int fad_nearest(fad_handle* h, const void* z_f16, long long m, long long n, int d, int k, const long long* base_offsets,
                long long n_groups, int* nearest, float* nearest_sq, void* stream);
int fad_nearest_sharded(fad_handle* h, void* nccl_comm_or_null, int local_shards, const void* z_f16, long long m,
                        long long n, int d, int k, const long long* base_offsets, long long n_groups, int* nearest,
                        float* nearest_sq, void* stream);
/* A prepared baseline (DESIGN.md section 5.15): the baseline-only work of KAD, PRDC and realism done once, then eval
 * passes that take its results as device inputs and run no tile of X against X.  z = [X; Y] as above (fp16, X first,
 * 16-byte aligned), d a multiple of 8, q as for PRDC.  Every argument is checked first (null or misaligned pointers, d,
 * k, the row limits of the unprepared entry each one stands in for); a rejected call launches nothing and writes nothing.
 *   fad_pair_digest        out (device uint64, 8-byte aligned) = the order-dependent digest of the rows fp16 [rows, d]
 *                          that the _sharded entries compare across ranks; a saved preparation records it for its rows
 *   fad_knn_lists_sq       x = X alone (fp16 [m, d]), 1 <= k_max <= 16, m > k_max; lists (device fp32 [m][k_max]) = per
 *                          row of X the k_max smallest q to the other rows of X, ascending.  Column k - 1 is bitwise the
 *                          r_i^2 fad_knn_radii_sq gives at k, for every k <= k_max (both exact selections of one set of
 *                          fp32 values)
 *   fad_kad_eval_sums      fad_kad_song_sums without the S_xx pass (offsets, sigma and their checks as there; a whole eval
 *                          set is one item); out (device fp64 [n_items][2]) = S_yy,k, S_xy,k, bitwise the values
 *                          fad_kad_song_sums gives from the same work list
 *   fad_knn_eval_radii_sq  the Y part of fad_knn_radii_sq (offsets NULL: Y = n_items rows, one set; checks as there) or
 *                          of fad_knn_song_radii_sq (offsets as there); radii_sq (device fp32 [n]) = s_j^2, bitwise those
 *                          calls' Y values.  With r_i^2 from a list, [r_i^2 | s_j^2] is the radii_sq input of
 *                          fad_prdc_counts / fad_prdc_song_counts
 *   fad_realism_prepared   the realism tile pass of fad_realism alone (m >= 2, n >= 1) on the caller's kept radii
 *                          (device fp32 [m]); realism, nearest, nearest_sq as fad_realism writes them, bitwise equal when
 *                          given the kept_radii_sq fad_realism writes
 * The _sharded forms split the tile work as their unprepared counterparts do (local_shards as for fad_kad_*_sharded),
 * bitwise equal for any number of shards.  Collective calls also compare k_max or k, the bits of sigma, the number of
 * items and a digest of the offsets, and a digest of the kept radii, as each entry takes them. */
int fad_pair_digest(fad_handle* h, const void* z_f16, long long rows, int d, unsigned long long* out, void* stream);
int fad_knn_lists_sq(fad_handle* h, const void* x_f16, long long m, int d, int k_max, float* lists, void* stream);
int fad_knn_lists_sq_sharded(fad_handle* h, void* nccl_comm_or_null, int local_shards, const void* x_f16, long long m,
                             int d, int k_max, float* lists, void* stream);
int fad_kad_eval_sums(fad_handle* h, const void* z_f16, long long m, const long long* offsets, long long n_items, int d,
                      const double* sigma, double* out, void* stream);
int fad_kad_eval_sums_sharded(fad_handle* h, void* nccl_comm_or_null, int local_shards, const void* z_f16, long long m,
                              const long long* offsets, long long n_items, int d, const double* sigma, double* out,
                              void* stream);
int fad_knn_eval_radii_sq(fad_handle* h, const void* z_f16, long long m, const long long* offsets, long long n_items,
                          int d, int k, float* radii_sq, void* stream);
int fad_knn_eval_radii_sq_sharded(fad_handle* h, void* nccl_comm_or_null, int local_shards, const void* z_f16,
                                  long long m, const long long* offsets, long long n_items, int d, int k, float* radii_sq,
                                  void* stream);
int fad_realism_prepared(fad_handle* h, const void* z_f16, long long m, long long n, int d, const float* kept_radii_sq,
                         float* realism, int* nearest, float* nearest_sq, void* stream);
int fad_realism_prepared_sharded(fad_handle* h, void* nccl_comm_or_null, int local_shards, const void* z_f16, long long m,
                                 long long n, int d, const float* kept_radii_sq, float* realism, int* nearest,
                                 float* nearest_sq, void* stream);
/* Permutation tests of KAD (DESIGN.md section 5.16).  A pool z of N fp16 rows [N, d] (16-byte aligned, d a multiple of
 * 8); a labelling marks `a` of them (2 <= a <= N - 2), B = labellings in [1, 9999].  Labelling 0 marks rows 0 .. a - 1;
 * labelling b >= 1 marks the a rows with the smallest (pair_mix64(pair_mix64(seed + b) ^ i), i) in wrapping uint64
 * (pair_mix64 = the splitmix64 finaliser, kad.cuh).  Every argument is checked first; a rejected call launches nothing
 * and writes nothing.
 *   fad_perm_labels    bits (device uint32 [B + 1][4 ceil(N / 128)], 16-byte aligned): bit i & 31 of word i >> 5 of
 *                      labelling b is row i's label; 0 past N
 *   fad_perm_dot       out (device fp64 [B + 1]) = per labelling the sum of v (device fp64 [N]) over the rows it marks,
 *                      from bits as fad_perm_labels writes them; a fixed order, bitwise reproducible
 *   fad_kad_perm_sums  out (device fp64 [B + 1][3]) = (S_aa, S_bb, S_ab) of every labelling: the sums of
 *                      exp(-q / (2 sigma^2)) (sigma: device fp64) over the pairs i < j with both rows marked, neither,
 *                      and one, each kernel value rounded to fp16 once.  Bitwise reproducible and independent of the grid
 * fad_kad_perm_sums_sharded splits the tile passes as fad_kad_sums_sharded does, bitwise equal for any number of shards;
 * collective calls also compare a, B, the seed and the bits of sigma. */
int fad_perm_labels(fad_handle* h, long long N, long long a, int labellings, unsigned long long seed, uint32_t* bits,
                    void* stream);
int fad_perm_dot(fad_handle* h, const uint32_t* bits, long long N, int labellings, const double* v, double* out,
                 void* stream);
int fad_kad_perm_sums(fad_handle* h, const void* z_f16, long long N, long long a, int d, const double* sigma,
                      int labellings, unsigned long long seed, double* out, void* stream);
int fad_kad_perm_sums_sharded(fad_handle* h, void* nccl_comm_or_null, int local_shards, const void* z_f16, long long N,
                              long long a, int d, const double* sigma, int labellings, unsigned long long seed,
                              double* out, void* stream);

/* ---- Permutation test of the FAD difference between two systems (DESIGN.md section 5.17).  A pool of n_units units
 * (files: rows [offsets[u], offsets[u + 1]) of emb_f16 [N, d], no empty unit), the first a of them system A's.  d a
 * positive multiple of 64 (at most 2048), 16-byte-aligned device pointers.  Labelling 0 marks units 0 .. a - 1;
 * labelling b >= 1 marks the a units fad_perm_labels marks (its rule over units).  Every argument is checked first
 * (offsets are read back, one stream synchronisation); a rejected call launches nothing and writes nothing.
 *   fad_record_len       R(d) = 1 + d + d (d + 1) / 2 (host only)
 *   fad_unit_records     records (device fp64 [n_units][R(d)]) = per unit [n_u | sum y | upper triangle of sum y y^T,
 *                        row by row], y = x - shift (shift_f16: device fp16 [d]); exact products, fp64 sums
 *   fad_perm_record_sums sums (device fp64 [B + 1][2][R(d)]) = per labelling the sum of the records of the units it
 *                        marks ([b][0]) and of those it does not ([b][1]); bits as fad_perm_labels writes them for
 *                        n_units rows.  Fixed order, bitwise reproducible
 *   fad_frechet_records  out (device fp64 [items][8], fad_frechet's layout, [7] = n) = the FAD against the baseline
 *                        (mu1, sqrt1 = C1^(1/2), scal1 = {|C1|_F, tr C1}) of the statistics of each of `items` sums:
 *                        mu = shift + sum y / n, C = (sum y y^T - sum y sum y^T / n) / (n - 1); NaN below 2 rows
 *   fad_frechet_perm     out (device fp64 [B + 1][2][8]) = the two FADs of every labelling: the whole pass above with
 *                        the fp16 mean of the pool as shift (written to shift_out, device fp16 [d]), B = labellings in
 *                        [1, 9999], 2 <= a <= n_units - 2.  Bitwise equal to replaying the three stage entries over
 *                        all units with shift_out */
long long fad_record_len(int d);
int fad_unit_records(fad_handle* h, const void* emb_f16, const long long* offsets, long long n_units, int d,
                     const void* shift_f16, double* records, void* stream);
int fad_perm_record_sums(fad_handle* h, const double* records, long long n_units, int d, const uint32_t* bits,
                         int labellings, double* sums, void* stream);
int fad_frechet_records(fad_handle* h, const double* mu1, const double* sqrt1, const double* scal1, const double* sums,
                        long long items, int d, const void* shift_f16, int iters, double* out, void* stream);
int fad_frechet_perm(fad_handle* h, const double* mu1, const double* sqrt1, const double* scal1, const void* emb_f16,
                     const long long* offsets, long long n_units, long long a, int d, int labellings,
                     unsigned long long seed, int iters, void* shift_out, double* out, void* stream);

/* ---- Bootstrap confidence intervals of FAD and KAD (DESIGN.md section 5.18).  An eval set of n_units >= 2 units
 * (files: rows [offsets[u], offsets[u + 1]) of a fp16 [N, d] array, no empty unit) is resampled B = resamples times
 * (2 <= B <= 9999) with replacement, whole units at a time; the baseline is held fixed.  Resample 0 is the observed
 * set (every multiplicity 1); resample b >= 1 makes F = n_units draws t = 0 .. F - 1, draw t picking unit
 * floor(pair_mix64(pair_mix64(seed + b) ^ t) * F / 2^64) (the high word of the 128-bit product), and w_b(u) counts
 * the draws of u.  16-byte-aligned device pointers; every argument is checked first (offsets are read back, one
 * stream synchronisation); a rejected call launches nothing and writes nothing.
 *   fad_boot_counts      counts (device uint32 [B + 1][n_units]) = w_b(u); integer counts, bitwise reproducible
 *   fad_boot_record_sums sums (device fp64 [B + 1][R(d)]) = sum_u counts[b][u] records[u] (records as
 *                        fad_unit_records writes them, counts as fad_boot_counts does); fixed order, bitwise the same
 *                        however the units are cut into chunks and the resamples into passes
 *   fad_frechet_boot     out (device fp64 [B + 1][8], fad_frechet's layout, [7] = n_b) = the FAD of every resample
 *                        against the baseline (mu1, sqrt1, scal1 as fad_frechet_records takes them): the weighted
 *                        record sums of the units about the fp16 mean of all rows (written to shift_out, device fp16
 *                        [d]), then fad_frechet_records' statistics and chain.  d a multiple of 64, at most 2048
 *   fad_kad_boot_sums    out (device fp64 [B + 1][3]) = (n_b, S_yy(b), S_xy(b)) of every resample of the rows y_f16
 *                        (d a multiple of 8): n_b = sum_u w_u n_u, S_yy(b) = sum_{i<j} v_i v_j K_ij + sum_u n_u w_u
 *                        (w_u - 1) / 2 (v_i the multiplicity of row i's unit, K_ij = exp(-|y_i - y_j|^2 /
 *                        (2 sigma^2)) rounded to fp16 once, weights fed to the tensor cores as fp16), S_xy(b) =
 *                        sum_u w_u g_units[u] (g_units: device fp64 [n_units], per unit the sum of k(x, y) over the
 *                        baseline rows and the unit's rows, e.g. column 1 of fad_kad_eval_sums).  sigma: device fp64
 *                        scalar.  Fails (out not valid) if a multiplicity exceeds 2048, which n_units <= 2048 rules out */
int fad_boot_counts(fad_handle* h, long long n_units, int resamples, unsigned long long seed, uint32_t* counts,
                    void* stream);
int fad_boot_record_sums(fad_handle* h, const double* records, long long n_units, int d, const uint32_t* counts,
                         int resamples, double* sums, void* stream);
int fad_frechet_boot(fad_handle* h, const double* mu1, const double* sqrt1, const double* scal1, const void* emb_f16,
                     const long long* offsets, long long n_units, int d, int resamples, unsigned long long seed,
                     int iters, void* shift_out, double* out, void* stream);
int fad_kad_boot_sums(fad_handle* h, const void* y_f16, const long long* offsets, long long n_units, int d,
                      const double* sigma, const double* g_units, int resamples, unsigned long long seed, double* out,
                      void* stream);

/* ---- audio conversion: replaces the torchaudio branch of FrechetAudioDistance.load_audio
 * (fadtk/fad.py:147-160): mono mix (:150), Resample(lowpass_filter_width=64, rolloff=0.9475937167399596,
 * sinc_interp_kaiser, beta=14.769656459379492) (:151-158), PCM16 quantisation (:160).
 * fad_resample_geometry / _length / _bank are host-only (no GPU): reduced rates orig/new, filter
 * half-width, taps = 2*width + orig; output length ceil(new*length/orig); the [new][taps] float32
 * filter bank exactly as torchaudio builds it.
 * fad_resample: exactly one of in_i16 (interleaved [length][channels], scaled by 1/32768) and in_f32
 * (planar [channels][length]) is given (device); out_pcm int16 [fad_resample_length] (device);
 * out_f32 optional un-quantised copy (device) or NULL. */
int fad_resample_geometry(int sr_in, int sr_out, int* orig, int* new_, int* width, int* taps);
long long fad_resample_length(int sr_in, int sr_out, long long length);
int fad_resample_bank(int sr_in, int sr_out, float* bank_host);
int fad_resample(fad_handle* h, const int16_t* in_i16, const float* in_f32, int channels, long long length,
                 int sr_in, int sr_out, int16_t* out_pcm, float* out_f32, void* stream);

/* ---- measurement ----------------------------------------------------------------------
 * When enabled, CUDA events are recorded on the launching stream around every kernel group;
 * fad_profile_collect synchronises the device and returns accumulated milliseconds and launch
 * counts per category (arrays of FAD_PROF_CATEGORIES entries). */
#define FAD_PROF_LOGMEL        0
#define FAD_PROF_CONV1         1
#define FAD_PROF_LAYER0        2   /* +i: conv2, conv3_1, conv3_2, conv4_1, conv4_2, fc1, fc2, fc3 */
#define FAD_PROF_STATS        10
#define FAD_PROF_STATS_REDUCE 11
#define FAD_PROF_FRECHET      12
#define FAD_PROF_CLAP_FRONT   13   /* log-mel + patch embedding */
#define FAD_PROF_CLAP_GEMM    14   /* wgmma GEMMs of the Swin blocks */
#define FAD_PROF_CLAP_ATTN    15   /* window attention */
#define FAD_PROF_CLAP_OTHER   16   /* LayerNorm, residual adds, head */
#define FAD_PROF_CATEGORIES   20
int fad_profile_enable(fad_handle* h, int on);
int fad_profile_collect(fad_handle* h, double* ms_out, long long* count_out, int reset);

/* Number of CUDA kernels this library has launched through `h` (bench.py's gpu_launches). */
long long fad_launch_count(fad_handle* h);

/* Stage entry (parity test / profiling): the encoder self-attention of the Whisper and wav2vec-family forwards alone.
 * qkv: fp16 [n_clips * S][3 d] (q | k | v, head i at columns i * 64), out: fp16 [n_clips * S][d], softmax(q k^T / 8) v per
 * head.  legacy = 0: wgmma kernel (csrc/attention_wgmma.cuh), which every model but WavLM runs; 1: the mma.sync flash
 * kernel (csrc/whisper.cuh) WavLM runs for its gated relative position bias (here without the bias). */
int fad_attention(fad_handle* h, const void* qkv_f16, long long n_clips, int S, int d, void* out_f16, int legacy, void* stream);

/* Stage entries (parity tests) of the other attention and LayerNorm launches of the transformer forwards; each calls the
 * launch code its forward calls and fails, launching nothing, on arguments that launch could not honour.
 *
 * fad_window_attention: Swin window attention of a CLAP block.  qkv fp16 [n_windows * 64][3 C] (q | k | v, rows in
 * shifted-window order: 8x8 windows of res x res images), relbias fp32 [heads][64][64], out fp16 [n_windows * 64][C];
 * per (window, head): softmax(q k^T / sqrt(C / heads) + relbias (- 100 across shift regions)) v.  C / heads is 24 or 32;
 * res a power of two >= 8, shift 0 or (res > 8) in (0, 8), n_windows whole images.  16-byte aligned pointers. */
int fad_window_attention(fad_handle* h, const void* qkv_f16, long long n_windows, int C, int heads, const float* relbias,
                         int res, int shift, void* out_f16, void* stream);
/* fad_attention_bias: WavLM self-attention, heads of 64 dims, with the gated relative position bias: score(q, k) =
 * q.k / 8 + gate[q][head] * relb[head][k - q + S - 1].  qkv fp16 [n_clips * S][3 d], relb fp32 [d / 64][2 S - 1],
 * gate fp32 [n_clips * S][d / 64], out fp16 [n_clips * S][d]. */
int fad_attention_bias(fad_handle* h, const void* qkv_f16, long long n_clips, int S, int d, const float* relb,
                       const float* gate, void* out_f16, void* stream);
/* fad_wavlm_gate: gate[r][i] = a (b c[i] - 1) + 2 with p = w x[r][64 i : 64 i + 64] + b_lin (w [8][64], b_lin [8]),
 * a = sigmoid(p0 + .. + p3), b = sigmoid(p4 + .. + p7).  x fp32 [rows][d], d = heads * 64; gate_out fp32 [rows][heads]. */
int fad_wavlm_gate(fad_handle* h, const float* x, const float* w, const float* b, const float* c, long long rows, int heads,
                   int d, float* gate_out, void* stream);
/* fad_wavlm_bias_table (host only): the relb table fad_w2v_forward uploads for S positions, out host [heads][2 S - 1]
 * from rel_embed host [320][heads] (bucketed key - query distance, 320 buckets, max distance 800). */
int fad_wavlm_bias_table(int heads, int S, const float* rel_embed, float* out);
/* fad_decoder_self_attention: Whisper decoder self-attention over the two start tokens of each clip (token 0 attends
 * to itself, token 1 to both).  qkv fp16 [n_clips * 2][3 d], out fp16 [n_clips * 2][d]. */
int fad_decoder_self_attention(fad_handle* h, const void* qkv_f16, long long n_clips, int d, void* out_f16, void* stream);
/* fad_cross_attention: Whisper decoder cross-attention of the two queries of each clip to its S encoder positions.
 * q fp16 [n_clips * 2][d], kv fp16 [n_clips * S][2 d] (k | v), out fp16 [n_clips * 2][d]; the 2 S fp32 scores of a
 * (clip, head) must fit in the kernel's shared memory. */
int fad_cross_attention(fad_handle* h, const void* q_f16, const void* kv_f16, long long n_clips, int S, int d, void* out_f16,
                        void* stream);
/* fad_layernorm: one LayerNorm launch (eps 1e-5) as the CLAP / Whisper / wav2vec forwards issue it.  mode 0: output row
 * o normalises token o (res = 0) or the token of window-ordered row o (res > 0, cyclic shift); mode 1: the 2x2
 * patch-merge gather of output row o on a res x res grid, features [x(2i,2j), x(2i+1,2j), x(2i,2j+1), x(2i+1,2j+1)].
 * width = C (mode 0) or 4 C (mode 1) must be one the kernel is built for; gelu != 0 applies exact-erf GELU after the
 * affine.  out fp16 [rows][ld_out], columns width .. ld_out - 1 set to zero; out_f32 optional fp32 [rows][width], which
 * may be x itself only in mode 0 with res = 0. */
int fad_layernorm(fad_handle* h, const float* x, const float* gamma, const float* beta, long long rows, int C, int ld_out,
                  int res, int shift, int mode, int gelu, void* out_f16, float* out_f32, void* stream);

/* ---- measurement utility -------------------------------------------------------------
 * fp64 tensor-pipe (DMMA m8n8k4) rate of this GPU in TFLOP/s, measured with a register-only
 * issue loop: the roofline denominator of the exact-Gram and Newton-Schulz kernels, which
 * MEASURED_PEAKS.json (bf16 GEMM, HBM copy) does not carry.  Synchronous; iters <= 0 = default. */
int fad_bench_dmma_peak(fad_handle* h, int iters, double* tflops_out_host);

#ifdef __cplusplus
}
#endif
#endif /* FADTK_B200_H */
