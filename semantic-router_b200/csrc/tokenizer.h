// Host tokenizer: loads a HuggingFace `tokenizer.json` and reproduces `tokenizers` 0.21 encode() for the
// pipelines the reference's models use -- ids, token strings and BYTE offsets into the original text.
//
// Replaces the third-party `tokenizers 0.21.4` crate behind
//   candle-binding/src/core/tokenization.rs:196,218-247,343-395 (UnifiedTokenizer)
//   candle-binding/src/core/similarity.rs:190-205 (BertSimilarity::get_embedding)
// Supported components: normalizers BertNormalizer / NFC / NFD / NFKC+NFKD (canonical part only) / Lowercase /
// StripAccents / Replace(String) / Prepend / Strip / Sequence; pre-tokenizers BertPreTokenizer / Whitespace /
// WhitespaceSplit / ByteLevel (GPT-2 regex) / Split(String pattern) / Metaspace / Punctuation / Digits / Sequence;
// models WordPiece and BPE (byte_fallback, ignore_merges, prefixes/suffixes); post-processors
// TemplateProcessing / BertProcessing / RobertaProcessing / ByteLevel(trim_offsets) / Sequence; added tokens.
#pragma once
#include <cstdint>
#include <memory>
#include <string>
#include <utility>
#include <vector>

namespace srb {

struct Encoding {
  std::vector<int32_t> ids;
  std::vector<std::string> tokens;
  std::vector<std::pair<int, int>> offsets;  // byte offsets into the original text; (0,0) for special tokens
};

class TokenizerImpl;

class Tokenizer {
 public:
  ~Tokenizer();
  static Tokenizer* from_file(const std::string& path, std::string* err);
  // encode(text, add_special_tokens) with truncation {max_length, LongestFirst, Right, stride 0}
  // (core/tokenization.rs:218-247); max_length <= 0 disables truncation.
  Encoding encode(const std::string& text, bool add_special_tokens, int max_length) const;
  int pad_id() const;
  // "padding": {"strategy": {"Fixed": n}} of the tokenizer.json (0: none / BatchLongest), its direction and pad token.
  // encode() never pads; callers that mirror a reference path which keeps the file's padding (BertSimilarity,
  // core/similarity.rs:189-205) append the pads themselves.
  int pad_fixed() const;
  bool pad_left() const;
  const std::string& pad_token() const;
  int token_to_id(const std::string& tok) const;  // -1 if absent

 private:
  Tokenizer();
  std::unique_ptr<TokenizerImpl> impl_;
};

}  // namespace srb
