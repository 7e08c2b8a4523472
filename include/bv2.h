/* libbv2 -- C ABI of the Hopper-native (sm_90a) VITS2 inference engine (Bert-VITS2 v2.3 `SynthesizerTrn.infer`).
 *
 * The reference has no FFI/plugin layer: its seam is the Python class `models.SynthesizerTrn`
 * (reference models.py:811-1074) constructed by `infer.get_net_g` (reference infer.py:84-104) and driven by
 * `infer.infer` / `infer_multilang` (reference infer.py:302-318, 407-423).  This header is what a ctypes
 * binding behind that class binds (bert_vits2_b200/engine.py; INTEGRATION.md shows the reference-side stub).
 *
 * Conventions: every function returns 0 on success or a negative bv2_status; nothing throws or aborts across
 * the ABI; `bv2_last_error` returns a thread-unsafe, engine-owned message for the last failure.  The caller
 * owns every input/output buffer (device pointers unless noted, fp32 contiguous, reference tensor layouts
 * [B,C,T]); the engine owns weights and workspace.  Work is enqueued on the caller's `stream`
 * (a cudaStream_t passed as void*); the only host synchronisation is inside bv2_infer_begin (one read-back of
 * y_lengths, the same data-dependent length the reference syncs on at models.py:1058 / commons.py:120-121).
 * Calls on one engine are serialised by its internal mutex (ctypes drops the GIL), but a request spans two calls
 * (bv2_infer_begin .. bv2_infer_finish*, or a stream up to its last bv2_stream_advance), so one engine serves one request at a
 * time.  To serve several at once, give each its own sibling engine (bv2_create_sibling) and its own CUDA stream.
 * There is NO CPU fallback: creation fails if no sm_90 (H100) device is present.
 */
#ifndef BV2_H_
#define BV2_H_

#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

typedef struct bv2_engine bv2_engine;

typedef enum {
    BV2_OK = 0,
    BV2_ERR_ARG = -1,      /* bad argument / unsupported configuration (reference raises ValueError) */
    BV2_ERR_STATE = -2,    /* call order violated (weights missing, not finalized, begin/finish mismatch) */
    BV2_ERR_CUDA = -3,     /* CUDA runtime error */
    BV2_ERR_INTERNAL = -4
} bv2_status;

#define BV2_MAX_UPS 8
#define BV2_MAX_RESBLOCK_KERNELS 4
#define BV2_MAX_DILATIONS 4

/* `hps.model` + ctor args of reference models.SynthesizerTrn.__init__ (models.py:816-841). */
typedef struct {
    int32_t n_vocab, num_tones, num_languages, bert_dim;
    int32_t inter_channels, hidden_channels, filter_channels, n_heads, n_layers, kernel_size, window_size;
    int32_t gin_channels, n_speakers;
    int32_t n_flow_layer, n_layers_trans_flow, use_transformer_flow, flow_kernel_size, wn_layers;
    int32_t upsample_initial_channel, n_ups;
    int32_t upsample_rates[BV2_MAX_UPS], upsample_kernel_sizes[BV2_MAX_UPS];
    int32_t n_resblock_kernels, n_dilations;
    int32_t resblock_kernel_sizes[BV2_MAX_RESBLOCK_KERNELS];
    int32_t resblock_dilation_sizes[BV2_MAX_RESBLOCK_KERNELS][BV2_MAX_DILATIONS];
    int32_t sdp_filter, sdp_kernel, sdp_n_flows, sdp_dds_layers, sdp_num_bins;
    float sdp_tail_bound;
    int32_t dp_filter, dp_kernel, cond_layer_idx;
    int32_t generator_precision; /* 0 = fp32 SIMT convs; 1 = TF32 wgmma implicit-GEMM convs (flow + Generator); 2 = FP16-operand
                                    wgmma convs (same 11-bit significand as TF32, fp32 accumulate, fp32 activations in HBM) */
    int32_t n_flows;             /* couplings in `flow`: n_flow_layer for TransformerCouplingBlock (models.py:82-145), always 4 for
                                    ResidualCouplingBlock, whose n_layers argument receives n_flow_layer (models.py:403-445, 918-919) */
} bv2_config;

/* replaces: models.SynthesizerTrn(...).to(device) (reference infer.py:95-101) */
int bv2_create(bv2_engine** out, const bv2_config* cfg, int cuda_device);

/* A sibling shares the finalized device weights of `src` (nothing is copied or re-packed) and owns everything a call writes: workspace
 * arenas, per-call state (infer_begin..finish, open Generator stream, attn path, debug taps), pinned read-back buffer, side streams and
 * events, profiling events, launch/grow counters, error text and its own mutex.  Calls on different members of a family do not
 * serialise on the host and may run concurrently on different CUDA streams; their outputs are bit-identical to those of `src`.
 * `src` must be finalized (bv2_finalize or bv2_load_packed), else BV2_ERR_STATE.  A sibling of a sibling joins the same family.
 * bv2_set_weight, bv2_finalize and bv2_load_packed on a sibling return BV2_ERR_STATE; bv2_save_packed works on any member.  The device
 * weights are reference-counted: freed with the family's last member, in any destruction order.  A sibling starts with an empty
 * workspace (bv2_workspace_bytes == 0); a workspace regrowth synchronises the device and so stalls the other members' work:
 * bv2_reserve each sibling up front. */
int bv2_create_sibling(bv2_engine** out, bv2_engine* src);

/* replaces: load_state_dict for one entry of `G_*.pth["model"]` (reference utils.py:65-120).
 * `key` is the reference state_dict key (weight-norm as weight_g/weight_v); host_ptr is HOST memory;
 * dtype: 0 = fp32, 1 = fp16 (compress_model.py:49-52 checkpoints).  Unknown keys (enc_q.*) are ignored. */
int bv2_set_weight(bv2_engine* e, const char* key, const void* host_ptr, const int64_t* shape, int ndim, int dtype);

/* folds weight-norm (incl. ConvTranspose dim-0 = in_channels), folds Flip into coupling weights,
 * packs and uploads.  replaces: net_g.eval() + the per-call weight-norm re-evaluation of the reference. */
int bv2_finalize(bv2_engine* e);

/* Packed engine weight file (SURVEY.md section 8f.4; the reference's only checkpoint tool is compress_model.py:44-53, which drops enc_q and
 * casts to fp16).  bv2_save_packed dumps the finalized engine's weight arena: weight-norm and Flip already folded, SIMT and
 * tensor-core operand images already packed for this configuration + precision.  bv2_load_packed replaces the
 * bv2_set_weight... + bv2_finalize sequence on a fresh engine created with the SAME bv2_config: it rebuilds the (cheap) layout
 * bookkeeping and fills device memory with ONE cudaMemcpy of the file image.  Mismatching configurations are rejected. */
int bv2_save_packed(bv2_engine* e, const char* path);
int bv2_load_packed(bv2_engine* e, const char* path);

/* ---- whole path: SynthesizerTrn.infer (reference models.py:1026-1074), split at the data-dependent length.
 * begin: emb_g -> enc_p -> sdp/dp -> durations.  Inputs as the reference passes them (int64 ids, fp32 feats).
 *   noise_w [B,2,T] replaces torch.randn at models.py:249.  w_ceil_override (optional, [B,T] fp32) teacher-forces
 *   durations for parity harnesses.  Writes y_lengths_host[B] (HOST) and *f_max = max(y_lengths).            */
int bv2_infer_begin(bv2_engine* e, int B, int T, const int64_t* x, const int64_t* x_lengths, const int64_t* sid,
                    const int64_t* tone, const int64_t* language, const float* bert, const float* ja_bert,
                    const float* en_bert, const float* noise_w, float noise_scale_w, float length_scale,
                    float sdp_ratio, const float* w_ceil_override, void* stream, int64_t* y_lengths_host,
                    int32_t* f_max);
/* Per-utterance settings: bv2_infer_begin, except that noise_scale_w, length_scale and sdp_ratio are DEVICE fp32 arrays [B] and
 * utterance b is synthesised with its own entries, and that noise_scale [B] (DEVICE fp32) gives each utterance its own prior-noise
 * scale.  Every bv2_infer_finish* that follows samples utterance b with noise_scale_arg * noise_scale[b] rounded once to fp32, where
 * noise_scale_arg is the finish call's own noise_scale: pass 1.0 there to get exactly noise_scale[b].  bv2_infer_begin clears the
 * per-utterance scale, so after it finish uses noise_scale_arg alone.  Each setting only scales per-utterance elementwise arithmetic,
 * so utterance b's outputs (durations, y_lengths and, for the same F, everything finish writes) are bit-identical to those of the
 * same batch begun by bv2_infer_begin with b's settings as scalars.  Same launches, host read-back and workspace as bv2_infer_begin;
 * the engine copies noise_scale before returning, so the caller may free the four arrays after the call.  A NULL array returns
 * BV2_ERR_ARG. */
int bv2_infer_begin_items(bv2_engine* e, int B, int T, const int64_t* x, const int64_t* x_lengths, const int64_t* sid,
                          const int64_t* tone, const int64_t* language, const float* bert, const float* ja_bert,
                          const float* en_bert, const float* noise_w, const float* noise_scale_w, const float* length_scale,
                          const float* sdp_ratio, const float* noise_scale, const float* w_ceil_override, void* stream,
                          int64_t* y_lengths_host, int32_t* f_max);
/* Speaker mixes: bv2_infer_begin_items, except that utterance b is conditioned on a weighted mix of K speaker embeddings instead of
 * the row of one sid.  mix_sid [B,K] (DEVICE int64) and mix_weight [B,K] (DEVICE fp32) give the mix, and
 *     g[b][c] = fl(w[b][0] * E[id[b][0]][c]),  then for k = 1..K-1:  g[b][c] = fl(g[b][c] + fl(w[b][k] * E[id[b][k]][c]))
 * with E = emb_g.weight, every operation one fp32 round-to-nearest (no FMA), in k order, so the same loop in IEEE fp32 on the host
 * gives the same bits.  Weights are used as given (no normalisation; negative weights and any sum allowed); ids may repeat; K is
 * not bounded by n_speakers.  Everything after g is bv2_infer_begin_items, so utterance b's outputs are bit-identical to those of
 * the same batch on an engine whose emb_g holds g[b] as an extra row and a plain call with sid = that row; K = 1 with weight 1.0
 * is bit-identical to bv2_infer_begin_items with sid = id.  Every bv2_infer_finish* that follows inherits the mix.  Same launches,
 * host read-back and workspace as bv2_infer_begin_items; the mix arrays are only read during the call.  Errors: K < 1,
 * B*K > INT32_MAX or a NULL array: BV2_ERR_ARG before any work; an id outside [0, n_speakers): BV2_ERR_ARG with "index out of
 * range: speaker id" in bv2_last_error; a non-finite weight: BV2_ERR_ARG with "non-finite speaker-mix weight" (and the id message
 * when both occur).  The engine serves the next call normally after any of them. */
int bv2_infer_begin_mix(bv2_engine* e, int B, int T, const int64_t* x, const int64_t* x_lengths, int K, const int64_t* mix_sid,
                        const float* mix_weight, const int64_t* tone, const int64_t* language, const float* bert, const float* ja_bert,
                        const float* en_bert, const float* noise_w, const float* noise_scale_w, const float* length_scale,
                        const float* sdp_ratio, const float* noise_scale, const float* w_ceil_override, void* stream,
                        int64_t* y_lengths_host, int32_t* f_max);

/* finish: length regulation -> prior sample -> flow reverse -> Generator.  noise_z [B,inter,>=F] with row stride
 * noise_ld replaces torch.randn_like at models.py:1071.  Outputs (caller-allocated, any may be NULL except o):
 *   o [B,1,Fg*hop] with Fg = min(F, max_len), attn [B,1,F,T], y_mask [B,1,F], z/z_p/m_p/logs_p [B,inter,F]. */
int bv2_infer_finish(bv2_engine* e, const float* noise_z, int64_t noise_ld, float noise_scale, int32_t max_len,
                     float* o, float* attn, float* y_mask, float* z, float* z_p, float* m_p, float* logs_p,
                     void* stream);

/* Same as bv2_infer_finish, but the waveform leaves the engine as 16-bit PCM o16 [B,1,Fg*hop] (int16), converted exactly as the
 * reference's callers do with gradio.processing_utils.convert_to_16_bit_wav on every infer() result (reference webui.py:86,
 * 129, 198; hiyoriUI.py:343): per utterance, over its valid samples, data / abs(data).max() * 32767 -> astype(int16) in
 * float32 (samples past the valid length and all-zero utterances give 0).  Halves the D2H / peer-store bytes (SURVEY §8f.4). */
int bv2_infer_finish_pcm16(bv2_engine* e, const float* noise_z, int64_t noise_ld, float noise_scale, int32_t max_len,
                           int16_t* o16, float* attn, float* y_mask, float* z, float* z_p, float* m_p, float* logs_p,
                           void* stream);
/* Ragged batch: bv2_infer_finish (o) or bv2_infer_finish_pcm16 (o16), exactly one of the two non-NULL, except that the Generator runs
 * each utterance at its own length min(y_lengths[b], Fg) instead of the padded Fg.  Utterance b's samples [0, min(y_lengths[b], Fg)*hop)
 * are bit-identical to a B=1 run of it at that length (bv2_generator_ragged documents the invariant); its samples past that are 0.
 * This differs from the padded result, whose last ~14 frames of every shorter utterance see the padding's non-zero activations.
 * Everything before the Generator, and y_mask, z, z_p, m_p, logs_p, are those of bv2_infer_finish.  Same launches and workspace
 * (bv2_reserve covers it).  FP16 Generator only (generator_precision 2 or 3): an fp32 or TF32 Generator returns BV2_ERR_ARG. */
int bv2_infer_finish_ragged(bv2_engine* e, const float* noise_z, int64_t noise_ld, float noise_scale, int32_t max_len, float* o,
                            int16_t* o16, float* attn, float* y_mask, float* z, float* z_p, float* m_p, float* logs_p, void* stream);
/* Streaming synthesis: audio leaves the Generator in chunks, before the whole utterance has gone through it.
 * bv2_infer_finish_stream does what bv2_infer_finish does up to and including the flow (same arguments and outputs), then opens a
 * stream over the caller's o [B,1,Fg*hop], which must stay allocated until the stream is closed.  Every
 * generator_precision streams.
 * bv2_stream_advance enqueues on `stream` the Generator work that makes o[..., :min(frames, Fg)*hop] final and writes that sample count
 * to *samples_ready (HOST, may be NULL).  Each layer computes a time window of its output as soon as its input is final far enough
 * ahead (every output element exactly once), so the streamed o is bit-identical to the one bv2_infer_finish writes.  The stream
 * closes when it reaches Fg.  frames not above the frames already final, or an advance without an open stream, return
 * BV2_ERR_STATE.  Every call that resets the workspace (bv2_infer_begin, bv2_infer_finish*, the per-stage entry points, a growing
 * bv2_reserve) closes an open stream.  A stream keeps all Generator activations alive: about 1.19 MB (FP16 Generator) or 2.37 MB (fp32 /
 * TF32) per frame per utterance at the default configuration (engine.cu states the exact figures).  16-bit PCM is not streamed: its peak normalisation needs the whole
 * utterance. */
int bv2_infer_finish_stream(bv2_engine* e, const float* noise_z, int64_t noise_ld, float noise_scale, int32_t max_len,
                            float* o, float* attn, float* y_mask, float* z, float* z_p, float* m_p, float* logs_p, void* stream);
int bv2_stream_advance(bv2_engine* e, int32_t frames, void* stream, int64_t* samples_ready);
/* Bounded stream: bv2_infer_finish_stream with a cap on how far one bv2_stream_advance may move the frontier.  With the FP16
 * Generator (generator_precision 2 or 3) and max_chunk_frames in [1, Fg), each Generator tensor keeps only the rows later windows
 * still read, in storage sized by the cap and not by Fg (bv2_stream_bytes), and the workspace the stream ensures is the encoder/flow
 * part plus that storage.  Each advance may then launch one extra kernel that moves the live rows of the tensors it would overrun
 * to the front of their storage, plus the conversion of the input rows the chunk reads; the audio stays bit-identical to
 * bv2_infer_finish.  An advance with frames - (frames already final) > max_chunk_frames returns BV2_ERR_ARG and leaves the stream
 * open and unchanged.  max_chunk_frames <= 0 or >= Fg: the unbounded stream of bv2_infer_finish_stream (which is this call with 0).
 * On an fp32 or TF32 Generator a cap in [1, Fg) returns BV2_ERR_ARG. */
int bv2_infer_finish_stream_bounded(bv2_engine* e, const float* noise_z, int64_t noise_ld, float noise_scale, int32_t max_len,
                                    int32_t max_chunk_frames, float* o, float* attn, float* y_mask, float* z, float* z_p, float* m_p,
                                    float* logs_p, void* stream);
/* Ragged stream: bv2_infer_finish_stream_bounded (same arguments; max_chunk_frames <= 0: unbounded) whose Generator runs each utterance
 * at its own length L_b = min(y_lengths[b], Fg), as bv2_infer_finish_ragged does.  Once the frontier reaches L_b frames, o[b, :L_b*hop]
 * is final and bit-identical to bv2_infer_finish_ragged's, and o[b, L_b*hop:] is 0 as far as the frontier has gone.  Every window
 * stores the rows of an item at or past its end as zeros, so a bounded stream's slides carry them like any other final rows.  The
 * windows, slides, launches and workspace are those of the padded stream with the same chunks (bv2_stream_bytes and
 * bv2_reserve_stream cover it).  FP16 Generator only (generator_precision 2 or 3): an fp32 or TF32 Generator returns BV2_ERR_ARG. */
int bv2_infer_finish_stream_ragged(bv2_engine* e, const float* noise_z, int64_t noise_ld, float noise_scale, int32_t max_len,
                                   int32_t max_chunk_frames, float* o, float* attn, float* y_mask, float* z, float* z_p, float* m_p,
                                   float* logs_p, void* stream);
/* Workspace bytes of the Generator tensors of a stream over Fg frames of a batch of B with chunks of at most max_chunk_frames: for a
 * cap in [1, Fg) the bounded storage, which does not depend on Fg; else what an unbounded stream allocates.  Negative (a BV2_ERR_*
 * code) for bad arguments, an engine that is not finalized, or a cap in [1, Fg) on an fp32 / TF32 Generator. */
int64_t bv2_stream_bytes(const bv2_engine* e, int B, int32_t Fg, int32_t max_chunk_frames);

/* The same conversion for a waveform batch the caller already holds: wave [B,L] fp32 (device), n_valid [B] int64 (device,
 * may be NULL = L) -> out [B,L] int16 (device). */
int bv2_wave_to_pcm16(bv2_engine* e, int B, int64_t L, const float* wave, const int64_t* n_valid, int16_t* out, void* stream);

/* attn [B,1,F,T] (reference commons.generate_path, commons.py:126-140; returned by infer() at models.py:1074) materialised
 * on demand from the durations of the last bv2_infer_begin: callers that never read it (infer.py:302-318 does not) skip the
 * O(F*T) write by passing attn = NULL to bv2_infer_finish.  Valid until the next bv2_infer_begin on this engine. */
int bv2_attn_path(bv2_engine* e, float* attn, void* stream);

/* Size the workspace for batches up to (B, T tokens, F_cap frames) up front: afterwards no call within those bounds
 * allocates or synchronises the device (the workspace otherwise grows geometrically on first use of a larger shape). */
int bv2_reserve(bv2_engine* e, int B, int T, int F_cap);
/* bv2_reserve plus room for one stream with chunks of at most max_chunk_frames (<= 0: an unbounded stream) over up to F_cap frames:
 * afterwards neither a call nor such a stream within those bounds grows the workspace.  A server reserves each engine of a pool
 * for its largest shape and cap.  Like bv2_reserve, it closes an open stream when it regrows an arena.  A cap in [1, F_cap) on an
 * fp32 / TF32 Generator returns BV2_ERR_ARG. */
int bv2_reserve_stream(bv2_engine* e, int B, int T, int F_cap, int32_t max_chunk_frames);

/* ---- per-stage entry points (parity tests + microbenchmarks; same kernels as the whole path) ---------------
 * text encoder: outputs x [B,H,T], m_p/logs_p [B,inter,T] (reference models.py:377-400)                       */
int bv2_text_encoder(bv2_engine* e, int B, int T, const int64_t* x, const int64_t* x_lengths, const int64_t* sid,
                     const int64_t* tone, const int64_t* language, const float* bert, const float* ja_bert,
                     const float* en_bert, float* x_out, float* m_out, float* logs_out, void* stream);
/* duration predictors on a given encoder output x [B,H,T]: logw_sdp/logw_dp [B,1,T]
 * (reference models.py:197-204,245-256 and 285-299)                                                         */
int bv2_duration(bv2_engine* e, int B, int T, const float* x, const int64_t* x_lengths, const int64_t* sid,
                 const float* noise_w, float noise_scale_w, float* logw_sdp, float* logw_dp, void* stream);
/* flow reverse on z_p [B,inter,F] -> z (reference models.py:142-145 / 442-445)                               */
int bv2_flow_reverse(bv2_engine* e, int B, int F, const float* z_p, const int64_t* y_lengths, const int64_t* sid,
                     float* z, void* stream);
/* Generator: z [B,inter,F], g [B,gin] -> o [B,1,F*hop] (reference models.py:538-557)                          */
int bv2_generator(bv2_engine* e, int B, int F, const float* z, const float* g, float* o, void* stream);
/* Ragged Generator: item b runs at L_b = lengths[b] (int64, DEVICE [B]) clamped to [1, F] on the device.  o[b, :L_b*hop] is
 * bit-identical to bv2_generator(B=1, F=L_b) on z[b, :, :L_b] and g[b]; o[b, L_b*hop:] is 0.  Every layer stores item b's rows below
 * L_b times its rows per frame, then zeros in the G2_PADR rows after them (what a run at L_b has as its zero halo); work wholly past
 * L_b is skipped.  FP16 Generator only, else BV2_ERR_ARG. */
int bv2_generator_ragged(bv2_engine* e, int B, int F, const float* z, const float* g, const int64_t* lengths, float* o, void* stream);

/* Debug tap: copy a named internal stage buffer of the LAST call (converted to [B,C,T]) to HOST memory.
 * Returns the number of floats written, or a negative status.                                               */
int64_t bv2_debug_read(bv2_engine* e, const char* name, float* host_out, int64_t capacity);

/* Stage timing (CUDA events recorded on the caller's stream around "encoder_duration", "flow", "generator"):
 * enable with bv2_set_profiling(e, 1); bv2_stage_ms blocks on the stage's end event and returns the duration of
 * the stage in the LAST call, or a negative value if it was not recorded.  Each bv2_stream_advance records "generator" around the
 * Generator work of its own chunk. */
int bv2_set_profiling(bv2_engine* e, int enable);
float bv2_stage_ms(bv2_engine* e, const char* stage);

/* Counters: kernels launched by the engine since creation / bytes of workspace in use. */
int64_t bv2_launch_count(const bv2_engine* e);
int64_t bv2_workspace_bytes(const bv2_engine* e);
int64_t bv2_workspace_grows(const bv2_engine* e); /* (re)allocations of the workspace arenas since creation */

/* Peer output slab -- the path's one exchange step on a multi-GPU node (SURVEY.md §8e; the reference has no equivalent:
 * its inference is single-device, webui.py:31, 397-399).  The root rank owns a device slab and exports its CUDA IPC
 * handle; every other rank (one process per GPU) opens it and passes a slice of the mapped address as the `o` output
 * pointer of bv2_infer_finish / bv2_generator, so the conv_post+tanh epilogue stores the finished waveform straight
 * into the root's memory over NVLink/NVSwitch (peer stores, no staging copy, no NCCL payload).
 *   bv2_peer_slab_alloc : cudaMalloc `bytes` on `cuda_device`, zero it, return the pointer and the 64-byte IPC handle
 *   bv2_peer_slab_open  : map a slab exported by another process into this one (lazy peer access)
 *   bv2_peer_slab_close : unmap (opener side);  bv2_peer_slab_free : release (owner side)
 *   bv2_peer_write      : async device->device copy of `bytes` into a (possibly peer-mapped) slab address on `stream`
 * All return BV2_OK or a negative status; none of them needs an engine. */
#define BV2_IPC_HANDLE_BYTES 64
int bv2_peer_slab_alloc(int cuda_device, int64_t bytes, void** dptr, unsigned char* handle_out);
int bv2_peer_slab_open(int cuda_device, const unsigned char* handle, void** dptr);
int bv2_peer_slab_close(int cuda_device, void* dptr);
int bv2_peer_slab_free(int cuda_device, void* dptr);
int bv2_peer_write(int cuda_device, void* dst, const void* src, int64_t bytes, void* stream);

const char* bv2_last_error(const bv2_engine* e);
const char* bv2_version(void);
void bv2_destroy(bv2_engine* e);

#ifdef __cplusplus
}
#endif
#endif /* BV2_H_ */
