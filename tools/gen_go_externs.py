"""Parses the cgo preambles of the reference's Go files (the drop-in contract, SURVEY.md section 8b) into
tests/golden/go_externs.json: for each of the three preambles the list of C function names Go links.
The reference checkout is not needed at test time: the list is committed as a fixture; re-run here when the reference moves.
    python tools/gen_go_externs.py"""
import json
import os
import re

REF = os.environ.get("SR_REFERENCE_DIR", "reference")   # checkout of vllm-project/semantic-router
FILES = {
    "candle": "candle-binding/semantic-router.go",
    "onnx": "onnx-binding/semantic-router.go",
    "unified": "src/semantic-router/pkg/classification/unified_classifier.go",
}


def externs(path):
    src = open(path).read()
    m = re.search(r"/\*(.*?)\*/\s*import \"C\"", src, re.S)
    pre = m.group(1)
    pre = re.sub(r"//[^\n]*", "", pre)
    pre = re.sub(r"typedef\s+(struct|enum)\s*\{.*?\}\s*\w+\s*;", "", pre, flags=re.S)
    names = []
    for d in re.finditer(r"(?:extern\s+)?[A-Za-z_][\w\s\*]*?\b([A-Za-z_]\w*)\s*\(([^;{}]*)\)\s*;", pre):
        n = d.group(1)
        if n not in names:
            names.append(n)
    return names


if __name__ == "__main__":
    out = {k: {"file": v, "externs": externs(os.path.join(REF, v))} for k, v in FILES.items()}
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    json.dump(out, open(os.path.join(root, "tests", "golden", "go_externs.json"), "w"), indent=1)
    print({k: len(v["externs"]) for k, v in out.items()})
