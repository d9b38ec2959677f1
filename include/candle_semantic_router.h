/* candle_semantic_router.h -- the drop-in C ABI of libcandle_semantic_router for the signal-extraction path.
 *
 * Every declaration below is the C side of an `extern` in the cgo preamble of
 *   candle-binding/semantic-router.go:27-453            (cited as GO:<line>)
 *   src/semantic-router/pkg/classification/unified_classifier.go:5-82   (cited as UC:<line>)
 * with the struct layouts the GO side declares (SURVEY.md section 8b: "the Go cgo preamble is the contract",
 * not candle-binding/src/ffi/types.rs).  The reference implementation of each symbol is the Rust `#[no_mangle]`
 * function named in the comment (candle-binding/src/ffi/<file>:<line>).
 *
 * Ownership: inputs are borrowed for the call; arrays/strings in results are malloc'd by the library and
 * released through the matching free_* (all of them are free(3)).  Errors: init_* -> false; classify_* ->
 * class = -1, confidence = 0; EmbeddingResult.error = true; similarity -1.0; int-returning calls -> -1.
 * There is NO CPU path: `use_cpu` is accepted and ignored (logged once); init fails without an sm_90 (H100) GPU.
 *
 * "LIVE" = implemented on the CUDA engine (BERT / MiniLM / ModernBERT / mmBERT sequence and token classifiers,
 * embeddings, similarity, batch + unified entries, hallucination detector and NLI).  "STUB" = out of the hot-path scope
 * (SURVEY.md section 2 rows 7-8: Qwen3 / Gemma / multimodal / Qwen3Guard / MLP selector / DeBERTa); exported so the Go
 * package still links, returns the documented failure value.
 * Multi-GPU: one process drives every visible GPU -- each init_* replicates its model on the device set and every call
 * goes to the least-loaded replica (SR_B200_DEVICES / SR_B200_DEVICE, include/sr_b200.h).
 */
#ifndef CANDLE_SEMANTIC_ROUTER_H
#define CANDLE_SEMANTIC_ROUTER_H
#include <stdbool.h>
#include <stddef.h>
#include <stdlib.h>

#if defined(__GNUC__)
#define CSR_API __attribute__((visibility("default")))
#else
#define CSR_API
#endif
#ifdef __cplusplus
extern "C" {
#endif

#include "unified_classifier_abi.h"   /* LoRA* / C*Result types, the 7 entries of unified_classifier.go:66-81 */

/* ---- result structures (GO:74-260, 303-433; UC:9-64) ------------------------------------------------- */
typedef struct { char* entity_type; int start; int end; char* text; float confidence; } ModernBertTokenEntity;      /* GO:74-80 */
typedef struct { ModernBertTokenEntity* entities; int num_entities; } ModernBertTokenClassificationResult;          /* GO:82-85 */
typedef struct { char* entity_type; int start; int end; char* text; float confidence; } BertTokenEntity;            /* GO:91-97 */
typedef struct { BertTokenEntity* entities; int num_entities; } BertTokenClassificationResult;                      /* GO:99-102 */
typedef struct { int index; float score; } SimilarityResult;                                                         /* GO:109-112 */
typedef struct { float* data; int length; bool error; int model_type; int sequence_length; float processing_time_ms; } EmbeddingResult; /* GO:115-122 */
typedef struct { float similarity; int model_type; float processing_time_ms; bool error; } EmbeddingSimilarityResult; /* GO:125-130 */
typedef struct { int index; float similarity; } SimilarityMatch;                                                     /* GO:133-136 */
typedef struct { SimilarityMatch* matches; int num_matches; int model_type; float processing_time_ms; bool error; } BatchSimilarityResult; /* GO:139-145 */
typedef struct { char* model_name; bool is_loaded; int max_sequence_length; int default_dimension; char* model_path; } EmbeddingModelInfo; /* GO:148-154 */
typedef struct { EmbeddingModelInfo* models; int num_models; bool error; } EmbeddingModelsInfoResult;                /* GO:157-161 */
typedef struct { int* token_ids; int token_count; char** tokens; bool error; } TokenizationResult;                   /* GO:164-169 */
#ifdef __cplusplus
typedef struct { int class_; float confidence; } ClassificationResult;                                               /* GO:172-175 (`class` in C) */
typedef struct { int class_; float confidence; float* probabilities; int num_classes; } ClassificationResultWithProbs; /* GO:178-183 */
typedef struct { int class_; float confidence; } ModernBertClassificationResult;                                     /* GO:219-222 */
typedef struct { int class_; float confidence; float* probabilities; int num_classes; } ModernBertClassificationResultWithProbs; /* GO:225-230 */
#else
typedef struct { int class; float confidence; } ClassificationResult;
typedef struct { int class; float confidence; float* probabilities; int num_classes; } ClassificationResultWithProbs;
typedef struct { int class; float confidence; } ModernBertClassificationResult;
typedef struct { int class; float confidence; float* probabilities; int num_classes; } ModernBertClassificationResultWithProbs;
#endif
typedef struct { int class_id; float confidence; char* category_name; float* probabilities; int num_categories; bool error; char* error_message; } GenerativeClassificationResult; /* GO:186-194 */
typedef struct { char* raw_output; bool error; char* error_message; } GuardResult;                                   /* GO:207-211 */
typedef struct { float* data; int length; bool error; int modality; float processing_time_ms; } MultiModalEmbeddingResult; /* GO:255-261 */
typedef struct { char* text; int start; int end; float confidence; char* label; } HallucinationSpan;                /* GO:303-309 */
typedef struct { bool has_hallucination; float confidence; HallucinationSpan* spans; int num_spans; bool error; char* error_message; } HallucinationDetectionResult; /* GO:312-319 */
typedef enum { NLI_ENTAILMENT = 0, NLI_NEUTRAL = 1, NLI_CONTRADICTION = 2, NLI_ERROR = -1 } NLILabel;               /* GO:322-327 */
typedef struct { NLILabel label; float confidence; float entailment_prob; float neutral_prob; float contradiction_prob; bool error; char* error_message; } NLIResult; /* GO:330-338 */
typedef struct { char* text; int start; int end; float hallucination_confidence; NLILabel nli_label; float nli_confidence; int severity; char* explanation; } EnhancedHallucinationSpan; /* GO:341-350 */
typedef struct { bool has_hallucination; float confidence; EnhancedHallucinationSpan* spans; int num_spans; bool error; char* error_message; } EnhancedHallucinationDetectionResult; /* GO:353-360 */

/* ---- LIVE: similarity model (BERT / MiniLM-class encoder, mean pool, L2) ------------------------------ */
CSR_API bool init_similarity_model(const char* model_id, bool use_cpu);                    /* GO:32  ffi/init.rs:154 */
CSR_API bool is_similarity_model_initialized(void);                                        /* GO:34  ffi/init.rs:182 */
CSR_API float calculate_similarity(const char* text1, const char* text2, int max_length);  /* GO:36  ffi/similarity.rs:108 */
CSR_API SimilarityResult find_most_similar(const char* query, const char** candidates, int num_candidates, int max_length); /* GO:233 ffi/similarity.rs:157 */
CSR_API EmbeddingResult get_text_embedding(const char* text, int max_length);              /* GO:234 ffi/similarity.rs:12 */
CSR_API TokenizationResult tokenize_text(const char* text, int max_length);                /* GO:250 ffi/tokenization.rs:12 */
CSR_API void free_tokenization_result(TokenizationResult result);                          /* GO:267 ffi/memory.rs:14 */
CSR_API void free_embedding(float* data, int length);                                      /* GO:252 ffi/memory.rs:63 */

/* ---- LIVE: BERT classifiers ---------------------------------------------------------------------------- */
CSR_API bool init_classifier(const char* model_id, int num_classes, bool use_cpu);         /* GO:38  ffi/init.rs:192 */
CSR_API bool init_pii_classifier(const char* model_id, int num_classes, bool use_cpu);     /* GO:40  ffi/init.rs:224 */
CSR_API bool init_jailbreak_classifier(const char* model_id, int num_classes, bool use_cpu); /* GO:42 ffi/init.rs:260 */
CSR_API ClassificationResult classify_text(const char* text);                              /* GO:268 ffi/classify.rs:70 */
CSR_API ClassificationResultWithProbs classify_text_with_probabilities(const char* text);  /* GO:269 ffi/classify.rs:107 */
CSR_API void free_probabilities(float* probabilities, int num_classes);                    /* GO:270 ffi/memory.rs:80 */
CSR_API ClassificationResult classify_pii_text(const char* text);                          /* GO:271 ffi/classify.rs:156 */
CSR_API ClassificationResult classify_jailbreak_text(const char* text);                    /* GO:272 ffi/classify.rs:194 */
CSR_API ClassificationResult classify_bert_text(const char* text);                         /* GO:273 ffi/classify.rs:832 */
CSR_API bool init_candle_bert_classifier(const char* model_path, int num_classes, bool use_cpu);       /* GO:292 ffi/init.rs:1242 */
CSR_API bool init_candle_bert_token_classifier(const char* model_path, int num_classes, bool use_cpu); /* GO:293 ffi/init.rs:1309 */
CSR_API ClassificationResult classify_candle_bert_text(const char* text);                  /* GO:294 ffi/classify.rs:757 */
CSR_API BertTokenClassificationResult classify_candle_bert_tokens(const char* text);       /* GO:295 ffi/classify.rs:629 */
CSR_API BertTokenClassificationResult classify_candle_bert_tokens_with_labels(const char* text, const char* id2label_json); /* GO:296 ffi/classify.rs:529 */
CSR_API bool init_bert_token_classifier(const char* model_path, int num_classes, bool use_cpu);        /* GO:104 ffi/init.rs:1197 */
CSR_API BertTokenClassificationResult classify_bert_pii_tokens(const char* text, const char* id2label_json); /* GO:105 ffi/classify.rs:477 */
CSR_API void free_bert_token_classification_result(BertTokenClassificationResult result);  /* GO:106 ffi/memory.rs:163 */

/* ---- LIVE: ModernBERT / mmBERT classifiers -------------------------------------------------------------- */
CSR_API bool init_modernbert_classifier(const char* model_id, bool use_cpu);               /* GO:44  ffi/init.rs:322 */
CSR_API bool init_modernbert_pii_classifier(const char* model_id, bool use_cpu);           /* GO:46  ffi/init.rs:349 */
CSR_API bool init_modernbert_jailbreak_classifier(const char* model_id, bool use_cpu);     /* GO:48  ffi/init.rs:403 */
CSR_API bool init_modernbert_pii_token_classifier(const char* model_id, bool use_cpu);     /* GO:56  ffi/init.rs:374 */
CSR_API bool init_fact_check_classifier(const char* model_id, bool use_cpu);               /* GO:52  ffi/init.rs:917 */
CSR_API bool init_feedback_detector(const char* model_id, bool use_cpu);                   /* GO:54  ffi/init.rs:975 */
CSR_API ModernBertClassificationResult classify_modernbert_text(const char* text);         /* GO:274 ffi/classify.rs:987 */
CSR_API ModernBertClassificationResultWithProbs classify_modernbert_text_with_probabilities(const char* text); /* GO:275 ffi/classify.rs:1023 */
CSR_API void free_modernbert_probabilities(float* probabilities, int num_classes);         /* GO:276 ffi/memory.rs:284 */
CSR_API ModernBertClassificationResult classify_modernbert_pii_text(const char* text);     /* GO:277 ffi/classify.rs:1079 */
CSR_API ModernBertClassificationResult classify_modernbert_jailbreak_text(const char* text); /* GO:278 ffi/classify.rs:1123 */
CSR_API ModernBertClassificationResult classify_fact_check_text(const char* text);         /* GO:280 ffi/classify.rs:1248 */
CSR_API ModernBertClassificationResult classify_feedback_text(const char* text);           /* GO:281 ffi/classify.rs:1316 */
CSR_API ModernBertTokenClassificationResult classify_modernbert_pii_tokens(const char* text, const char* model_config_path); /* GO:87 ffi/classify.rs:1355 */
CSR_API void free_modernbert_token_result(ModernBertTokenClassificationResult result);     /* GO:88  ffi/memory.rs:301 */
CSR_API bool init_mmbert_classifier(const char* model_id, bool use_cpu);                   /* GO:59  ffi/init.rs:474 */
CSR_API bool init_mmbert_classifier_auto(const char* model_id, bool use_cpu);              /* GO:60  ffi/init.rs:519 */
CSR_API bool init_mmbert_token_classifier(const char* model_id, bool use_cpu);             /* GO:61  ffi/init.rs:556 */
CSR_API bool is_mmbert_model(const char* config_path);                                     /* GO:62  ffi/init.rs:596 */
CSR_API bool init_mmbert_32k_intent_classifier(const char* model_id, bool use_cpu);        /* GO:65  ffi/init.rs:629 */
CSR_API bool init_mmbert_32k_factcheck_classifier(const char* model_id, bool use_cpu);     /* GO:66  ffi/init.rs:671 */
CSR_API bool init_mmbert_32k_jailbreak_classifier(const char* model_id, bool use_cpu);     /* GO:67  ffi/init.rs:713 */
CSR_API bool init_mmbert_32k_feedback_classifier(const char* model_id, bool use_cpu);      /* GO:68  ffi/init.rs:755 */
CSR_API bool init_mmbert_32k_pii_classifier(const char* model_id, bool use_cpu);           /* GO:69  ffi/init.rs:796 */
CSR_API bool init_mmbert_32k_modality_classifier(const char* model_id, bool use_cpu);      /* GO:70  ffi/init.rs:836 */
CSR_API bool is_mmbert_32k_model(const char* config_path);                                 /* GO:71  ffi/init.rs:877 */
CSR_API ModernBertClassificationResult classify_mmbert_32k_intent(const char* text);       /* GO:284 ffi/classify.rs:2059 */
CSR_API ModernBertClassificationResult classify_mmbert_32k_factcheck(const char* text);    /* GO:285 ffi/classify.rs:2106 */
CSR_API ModernBertClassificationResult classify_mmbert_32k_jailbreak(const char* text);    /* GO:286 ffi/classify.rs:2153 */
CSR_API ModernBertClassificationResult classify_mmbert_32k_feedback(const char* text);     /* GO:287 ffi/classify.rs:2200 */
CSR_API ModernBertTokenClassificationResult classify_mmbert_32k_pii_tokens(const char* text); /* GO:288 ffi/classify.rs:2246 */
CSR_API ModernBertClassificationResult classify_mmbert_32k_modality(const char* text);     /* GO:289 ffi/classify.rs:2335 */

/* ---- LIVE: embeddings (mmBERT 2D-Matryoshka slot) and top-k similarity -------------------------------- */
CSR_API bool init_embedding_models(const char* qwen3_model_path, const char* gemma_model_path, bool use_cpu); /* GO:240 ffi/embedding.rs:422 */
CSR_API bool init_embedding_models_with_mmbert(const char* qwen3_model_path, const char* gemma_model_path, const char* mmbert_model_path, bool use_cpu); /* GO:241 ffi/embedding.rs:323 */
CSR_API bool init_mmbert_embedding_model(const char* model_path, bool use_cpu);            /* GO:242 ffi/embedding.rs:252 */
CSR_API bool init_embedding_models_batched(const char* qwen3_model_path, int max_batch_size, unsigned long long max_wait_ms, bool use_cpu); /* GO:244 ffi/embedding.rs:1916 */
CSR_API int get_embedding_smart(const char* text, float quality_priority, float latency_priority, EmbeddingResult* result); /* GO:235 ffi/embedding.rs:865 */
CSR_API int get_embedding_with_dim(const char* text, float quality_priority, float latency_priority, int target_dim, EmbeddingResult* result); /* GO:236 ffi/embedding.rs:887 */
CSR_API int get_embedding_with_model_type(const char* text, const char* model_type, int target_dim, EmbeddingResult* result); /* GO:237 ffi/embedding.rs:1040 */
CSR_API int get_embedding_2d_matryoshka(const char* text, const char* model_type, int target_layer, int target_dim, EmbeddingResult* result); /* GO:238 ffi/embedding.rs:1068 */
CSR_API int get_embedding_batched(const char* text, const char* model_type, int target_dim, EmbeddingResult* result); /* GO:239 ffi/embedding.rs:2019 */
CSR_API int calculate_embedding_similarity(const char* text1, const char* text2, const char* model_type, int target_dim, EmbeddingSimilarityResult* result); /* GO:245 ffi/embedding.rs:1220 */
CSR_API int calculate_similarity_batch(const char* query, const char** candidates, int num_candidates, int top_k, const char* model_type, int target_dim, BatchSimilarityResult* result); /* GO:246 ffi/embedding.rs:1474 */
CSR_API void free_batch_similarity_result(BatchSimilarityResult* result);                  /* GO:247 ffi/embedding.rs:1718 */
CSR_API int get_embedding_models_info(EmbeddingModelsInfoResult* result);                  /* GO:248 ffi/embedding.rs:1752 */
CSR_API void free_embedding_models_info(EmbeddingModelsInfoResult* result);                /* GO:249 ffi/embedding.rs:1843 */

/* ---- LIVE: batch entries (the reference's only real batch API; BASELINE cfg 3): unified_classifier_abi.h ---- */

/* ---- STUB: out of scope, exported so the Go package links (documented failure values) ---------------- */
CSR_API bool init_deberta_jailbreak_classifier(const char* model_id, bool use_cpu);        /* GO:50  -> false */
CSR_API ClassificationResult classify_deberta_jailbreak_text(const char* text);            /* GO:279 -> {-1, 0} */
CSR_API bool init_multimodal_embedding_model(const char* model_path, bool use_cpu);        /* GO:243 -> false */
CSR_API int multimodal_encode_text(const char* text, int target_dim, MultiModalEmbeddingResult* result);  /* GO:263 -> -1 */
CSR_API int multimodal_encode_image(const float* pixel_data, int height, int width, int target_dim, MultiModalEmbeddingResult* result); /* GO:264 -> -1 */
CSR_API int multimodal_encode_audio(const float* mel_data, int n_mels, int time_frames, int target_dim, MultiModalEmbeddingResult* result); /* GO:265 -> -1 */
CSR_API void free_multimodal_embedding(float* data, int length);                           /* GO:266 */
CSR_API void free_generative_classification_result(GenerativeClassificationResult* result); /* GO:196 */
CSR_API void free_categories(char** categories, int num_categories);                       /* GO:197 */
CSR_API int init_qwen3_multi_lora_classifier(const char* base_model_path);                 /* GO:200 -> -1 */
CSR_API int load_qwen3_lora_adapter(const char* adapter_name, const char* adapter_path);   /* GO:201 -> -1 */
CSR_API int classify_with_qwen3_adapter(const char* text, const char* adapter_name, GenerativeClassificationResult* result); /* GO:202 -> -1 */
CSR_API int get_qwen3_loaded_adapters(char*** adapters_out, int* num_adapters);            /* GO:203 -> -1 */
CSR_API int classify_zero_shot_qwen3(const char* text, const char** categories, int num_categories, GenerativeClassificationResult* result); /* GO:204 -> -1 */
CSR_API int init_qwen3_guard(const char* model_path);                                      /* GO:213 -> -1 */
CSR_API int classify_with_qwen3_guard(const char* text, const char* mode, GuardResult* result); /* GO:214 -> -1 */
CSR_API void free_guard_result(GuardResult* result);                                       /* GO:215 */
CSR_API int is_qwen3_guard_initialized(void);                                              /* GO:216 -> 0 */
CSR_API int is_qwen3_multi_lora_initialized(void);                                         /* GO:217 -> 0 */
CSR_API bool init_hallucination_model(const char* model_path, bool use_cpu);               /* GO:363 ffi/init.rs:1483 (ModernBERT token classifier) */
CSR_API bool init_nli_model(const char* model_path, bool use_cpu);                         /* GO:366 ffi/init.rs:1522 (ModernBERT sequence classifier) */
CSR_API bool is_nli_model_initialized(void);                                               /* GO:369 ffi/init.rs:1572 */
CSR_API HallucinationDetectionResult detect_hallucinations(const char* context, const char* question, const char* answer, float threshold); /* GO:373 ffi/classify.rs:1459 */
CSR_API EnhancedHallucinationDetectionResult detect_hallucinations_with_nli(const char* context, const char* question, const char* answer, float threshold); /* GO:382 ffi/classify.rs:1840 */
CSR_API NLIResult classify_nli(const char* premise, const char* hypothesis);               /* GO:390 ffi/classify.rs:1723 */
CSR_API void free_hallucination_detection_result(HallucinationDetectionResult result);     /* GO:396 */
CSR_API void free_enhanced_hallucination_detection_result(EnhancedHallucinationDetectionResult result); /* GO:399 */
CSR_API void free_nli_result(NLIResult result);                                            /* GO:402 */
CSR_API void* candle_mlp_new(void);                                                        /* GO:444 -> NULL */
CSR_API void* candle_mlp_new_with_device(int device_type);                                 /* GO:445 -> NULL */
CSR_API void* candle_mlp_new_with_device_and_dtype(int device_type, int dtype);            /* GO:446 -> NULL */
CSR_API void candle_mlp_free(void* handle);                                                /* GO:447 */
CSR_API char* candle_mlp_select(void* handle, double* query, size_t query_len);            /* GO:448 -> NULL */
CSR_API int candle_mlp_is_trained(void* handle);                                           /* GO:449 -> 0 */
CSR_API char* candle_mlp_to_json(void* handle);                                            /* GO:450 -> NULL */
CSR_API void* candle_mlp_from_json(char* json);                                            /* GO:451 -> NULL */
CSR_API void* candle_mlp_from_json_with_device(char* json, int device_type);               /* GO:452 -> NULL */
CSR_API void* candle_mlp_from_json_with_device_and_dtype(char* json, int device_type, int dtype); /* GO:453 -> NULL */
CSR_API void candle_mlp_free_string(char* ptr);                                            /* GO:454 */

#ifdef __cplusplus
}
#endif
#endif
