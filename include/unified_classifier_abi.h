/* unified_classifier_abi.h -- the cgo preamble of
 *   src/semantic-router/pkg/classification/unified_classifier.go:5-82   (cited as UC:<line>)
 * The router's classification package declares these seven entries itself and links them from WHICHEVER binding the
 * build selects: libcandle_semantic_router (unified_classifier_cgo_candle.go:9) or, under `-tags=onnx`,
 * libonnx_semantic_router (unified_classifier_cgo_onnx.go:9).  Both libraries of this repository therefore export them
 * with the layouts the Go side declares (the same symbols also sit in candle-binding/semantic-router.go:409-438).
 * Reference implementations: candle-binding/src/ffi/{init.rs:1076,1380, classify.rs:258,882, memory.rs:48,97,194};
 * onnx-binding/src/ffi/unified.rs:107-200 only stubs them (init -> false, batch -> error) with struct layouts that do
 * not match the Go declaration -- here the ONNX twin runs the same packed passes as the candle twin.
 */
#ifndef UNIFIED_CLASSIFIER_ABI_H
#define UNIFIED_CLASSIFIER_ABI_H
#include <stdbool.h>
#if defined(__GNUC__)
#define UC_API __attribute__((visibility("default")))
#else
#define UC_API
#endif
#ifdef __cplusplus
extern "C" {
#endif

typedef struct { char* category; float confidence; } LoRAIntentResult;                                              /* GO:409-412 */
typedef struct { bool has_pii; char** pii_types; int num_pii_types; float confidence; } LoRAPIIResult;              /* GO:414-419 */
typedef struct { bool is_jailbreak; char* threat_type; float confidence; } LoRASecurityResult;                      /* GO:421-425 */
typedef struct { LoRAIntentResult* intent_results; LoRAPIIResult* pii_results; LoRASecurityResult* security_results; int batch_size; float avg_confidence; } LoRABatchResult; /* GO:427-433 */
typedef struct { char* category; float confidence; float* probabilities; int num_probabilities; } CIntentResult;    /* UC:10-15 */
typedef struct { bool has_pii; char** pii_types; int num_pii_types; float confidence; } CPIIResult;                 /* UC:17-22 */
typedef struct { bool is_jailbreak; char* threat_type; float confidence; } CSecurityResult;                         /* UC:24-28 */
typedef struct { CIntentResult* intent_results; CPIIResult* pii_results; CSecurityResult* security_results; int batch_size; bool error; char* error_message; } UnifiedBatchResult; /* UC:30-37 */

UC_API bool init_lora_unified_classifier(const char* intent_model_path, const char* pii_model_path, const char* security_model_path, const char* architecture, bool use_cpu); /* GO:436 ffi/init.rs:1380 */
UC_API LoRABatchResult classify_batch_with_lora(const char** texts, int num_texts);       /* GO:437 ffi/classify.rs:882 */
UC_API void free_lora_batch_result(LoRABatchResult result);                               /* GO:438 ffi/memory.rs:194 */
UC_API bool init_unified_classifier_c(const char* modernbert_path, const char* intent_head_path, const char* pii_head_path, const char* security_head_path, const char** intent_labels, int intent_labels_count, const char** pii_labels, int pii_labels_count, const char** security_labels, int security_labels_count, bool use_cpu); /* UC:67 ffi/init.rs:1076 */
UC_API UnifiedBatchResult classify_unified_batch(const char** texts, int num_texts);      /* UC:73 ffi/classify.rs:258 */
UC_API void free_unified_batch_result(UnifiedBatchResult result);                         /* UC:74 ffi/memory.rs:97 */
UC_API void free_cstring(char* s);                                                        /* GO:251 ffi/memory.rs:48 */

#ifdef __cplusplus
}
#endif
#endif /* UNIFIED_CLASSIFIER_ABI_H */
