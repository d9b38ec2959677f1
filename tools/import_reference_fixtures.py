"""Brings the reference-held test vectors of the hot path into tests/golden/ (tests must not depend on a reference checkout).
The only vector the reference holds for this path is candle-binding/test_data/long_prompt_fixtures.json: three prompts
(~3 600 / ~7 300 / ~21 tokens) that its Rust and Go tests push through the 512-token classification cap
(onnx-binding/src/model_architectures/classification/mmbert_classifier.rs:1250-1420,
candle-binding/src/model_architectures/traditional/modernbert_test.rs:1620-1800, candle-binding/semantic-router_test.go:4489-4640).
Kept: id, text, the reference's own token estimates and its cap.      python tools/import_reference_fixtures.py"""
import json
import os

SRC = os.path.join(os.environ.get("SR_REFERENCE_DIR", "reference"), "candle-binding/test_data/long_prompt_fixtures.json")
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))

if __name__ == "__main__":
    d = json.load(open(SRC))
    out = {"source": "candle-binding/test_data/long_prompt_fixtures.json (reference test data, unmodified texts)",
           "max_classification_seq_len": d["max_classification_seq_len"],
           "prompts": [{"id": p["id"], "approx_tokens_untruncated": p["approx_tokens_untruncated"], "text": p["text"]}
                       for p in d["prompts"]]}
    dst = os.path.join(ROOT, "tests", "golden", "reference_long_prompts.json")
    json.dump(out, open(dst, "w"), ensure_ascii=False, indent=0)
    print(dst, [(p["id"], len(p["text"])) for p in out["prompts"]])
