/* Drop-in C ABI #2: the symbol table onnx-binding/semantic-router.go binds
 * (`#cgo LDFLAGS: ... -lonnx_semantic_router`, OX:11).  It reuses candle-binding symbol NAMES with other SIGNATURES
 * (named classifier slots, no model-type argument on the embedding calls, result structs that carry label, full
 * probabilities and timing), so it is a separate library -- libonnx_semantic_router.so -- linked from the same
 * engine objects as libcandle_semantic_router.so.  It is also the reference's only ABI with a true batched classify.
 *
 *   OX:<n>  = onnx-binding/semantic-router.go line <n> (the C preamble that Go compiles against)
 *   RS: ... = the Rust (ONNX Runtime) implementation this entry replaces
 *
 * Model directories: where the reference opens <dir>/model.onnx, this library opens <dir>/model.safetensors (the HF
 * checkpoint the ONNX file was exported from), <dir>/config.json and <dir>/tokenizer.json.  Head semantics follow
 * the exported HF graph, not candle's hand-written head (sr_model_set_head_flavor(m, 1) in sr_b200.h).
 * Memory: every pointer handed out is malloc'd and released by the matching free_*.
 * Errors: int entries return 0 / -1 and fill the result with its error form; bool entries return false.
 * There is no CPU path: use_cpu / use_gpu are accepted and ignored. */
#ifndef ONNX_SEMANTIC_ROUTER_H_
#define ONNX_SEMANTIC_ROUTER_H_

#include <stdbool.h>

/* the seven entries pkg/classification/unified_classifier.go:66-81 links from this library under -tags=onnx
 * (init_unified_classifier_c, classify_unified_batch, free_unified_batch_result, free_cstring,
 * init_lora_unified_classifier, classify_batch_with_lora, free_lora_batch_result) */
#include "unified_classifier_abi.h"

#if defined(__GNUC__)
#define OSR_API __attribute__((visibility("default")))
#else
#define OSR_API
#endif

#ifdef __cplusplus
extern "C" {
#endif

/* ---- embedding types (OX:19-62; RS: onnx-binding/src/ffi/types.rs) ------------------------------------ */
typedef struct {
  float* data;
  int length;
  bool error;
  int model_type; /* 0 = mmbert, -1 = error */
  int sequence_length; /* whitespace word count of the text (RS: ffi/embedding.rs:181) */
  float processing_time_ms;
} EmbeddingResult; /* OX:19-26 */

typedef struct {
  float similarity;
  int model_type;
  float processing_time_ms;
  bool error;
} EmbeddingSimilarityResult; /* OX:28-33 */

typedef struct {
  int index;
  float similarity;
} SimilarityMatch; /* OX:35-38 */

typedef struct {
  SimilarityMatch* matches;
  int num_matches;
  int model_type;
  float processing_time_ms;
  bool error;
} BatchSimilarityResult; /* OX:40-46 */

typedef struct {
  char* model_name;
  bool is_loaded;
  int max_sequence_length;
  int default_dimension;
  char* model_path;
  bool supports_layer_exit;
  char* available_layers;
} EmbeddingModelInfo; /* OX:48-56 */

typedef struct {
  EmbeddingModelInfo* models;
  int num_models;
  bool error;
} EmbeddingModelsInfoResult; /* OX:58-62 */

/* ---- classification types (OX:68-92; RS: ffi/classification.rs:19-84) --------------------------------- */
typedef struct {
  char* label; /* id2label[class_id] from config.json, "LABEL_<id>" when absent */
  int class_id;
  float confidence;
  int num_classes;
  float* probabilities; /* [num_classes] softmax */
  float processing_time_ms;
  bool error;
} ClassificationResultFFI; /* OX:68-76 */

typedef struct {
  char* text;
  char* entity_type;
  int start; /* byte offsets into the UTF-8 text */
  int end;
  float confidence;
} PIIEntityFFI; /* OX:78-84 */

typedef struct {
  PIIEntityFFI* entities;
  int num_entities;
  float processing_time_ms;
  bool error;
  char* error_message;
} PIIResultFFI; /* OX:86-92 */

typedef struct {
  float* data;
  int length;
  bool error;
  int modality;
  float processing_time_ms;
} MultiModalEmbeddingResult; /* OX:128-134 */

/* ---- embedding functions (OX:98-109; RS: ffi/embedding.rs) --------------------------------------------- */
/* OX:98   RS: ffi/embedding.rs:37 -- a second init returns true (already initialised) */
OSR_API bool init_mmbert_embedding_model(const char* model_path, bool use_cpu);
OSR_API bool is_mmbert_model_initialized(void); /* OX:99  RS: ffi/embedding.rs:82 */
/* OX:100-102  RS: ffi/embedding.rs:117-232.  target_layer <= 0: full depth; target_dim <= 0: hidden size.
 * mean pool (masked) -> truncate -> x / max(||x||, 1e-12) (RS: embedding/pooling.rs:61-71). */
OSR_API int get_embedding(const char* text, EmbeddingResult* result);
OSR_API int get_embedding_with_dim(const char* text, int target_dim, EmbeddingResult* result);
OSR_API int get_embedding_2d_matryoshka(const char* text, int target_layer, int target_dim, EmbeddingResult* result);
/* OX:103  RS: ffi/embedding.rs:245-345 -- ONE packed batch through the encoder */
OSR_API int get_embeddings_batch(const char** texts, int num_texts, int target_layer, int target_dim,
                                 EmbeddingResult* results);
/* OX:104  RS: ffi/embedding.rs:357-430 -- cosine of the two (already unit) embeddings, 0 when a norm is 0 */
OSR_API int calculate_embedding_similarity(const char* text1, const char* text2, int target_layer, int target_dim,
                                           EmbeddingSimilarityResult* result);
/* OX:105  RS: ffi/embedding.rs:439-600 -- query + candidates in one batch, cosine, stable descending sort,
 * top_k <= 0 or > n: all candidates */
OSR_API int calculate_similarity_batch(const char* query, const char** candidates, int num_candidates, int top_k,
                                       int target_layer, int target_dim, BatchSimilarityResult* result);
OSR_API int get_embedding_models_info(EmbeddingModelsInfoResult* result); /* OX:106 RS: ffi/embedding.rs:614 */
OSR_API void free_embedding(float* data, int length);                     /* OX:107 RS: ffi/memory.rs:11 */
OSR_API void free_batch_similarity_result(BatchSimilarityResult* result); /* OX:108 RS: ffi/memory.rs:41 */
OSR_API void free_embedding_models_info(EmbeddingModelsInfoResult* result); /* OX:109 RS: ffi/memory.rs:67 */

/* ---- classification functions (OX:115-122; RS: ffi/classification.rs) ---------------------------------- */
/* Named slots: a second init under the same name replaces the model (HashMap::insert, RS: :183,:245). */
OSR_API bool init_sequence_classifier(const char* name, const char* model_path, bool use_gpu); /* OX:115 RS: :144 */
OSR_API bool init_token_classifier(const char* name, const char* model_path, bool use_gpu);    /* OX:116 RS: :206 */
OSR_API bool is_classifier_loaded(const char* name);                                           /* OX:117 RS: :260 */
/* OX:118 RS: :292-370.  Truncation to 512 tokens; softmax; last max wins (max_by, mmbert_classifier.rs:809-813). */
OSR_API int classify_text(const char* classifier_name, const char* text, ClassificationResultFFI* result);
/* OX:119 RS: :552-632 -- true batch: one packed varlen pass; processing_time_ms = total / num_texts */
OSR_API int classify_batch(const char* classifier_name, const char** texts, int num_texts,
                           ClassificationResultFFI* results);
/* OX:120 RS: :377-470; BIO decode RS: mmbert_classifier.rs:952-1050 (B- opens, same-type I- extends with a running
 * pairwise mean, other-type / orphan I- is ignored, O closes; tokens with offset (0,0) are skipped) */
OSR_API int detect_pii(const char* classifier_name, const char* text, PIIResultFFI* result);
OSR_API void free_classification_result(ClassificationResultFFI* result); /* OX:121 RS: :481 */
OSR_API void free_pii_result(PIIResultFFI* result);                       /* OX:122 RS: :506 */

/* ---- multi-modal embedding (OX:136-140; RS: ffi/multimodal.rs:19,57,112,186,258) -- not an encoder-classifier path:
 * exported so the Go package links; init returns false, encode_* return -1 with error = true. */
OSR_API bool init_multimodal_embedding_model(const char* model_path, bool use_cpu);
OSR_API int multimodal_encode_text(const char* text, int target_dim, MultiModalEmbeddingResult* result);
OSR_API int multimodal_encode_image(const float* pixel_data, int height, int width, int target_dim,
                                    MultiModalEmbeddingResult* result);
OSR_API int multimodal_encode_audio(const float* mel_data, int n_mels, int time_frames, int target_dim,
                                    MultiModalEmbeddingResult* result);
OSR_API void free_multimodal_embedding(float* data, int length);

#ifdef __cplusplus
}
#endif
#endif /* ONNX_SEMANTIC_ROUTER_H_ */
