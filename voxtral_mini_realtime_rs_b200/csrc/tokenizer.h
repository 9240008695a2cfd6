#pragma once
#include <cstddef>
#include <cstdint>
#include <map>
#include <mutex>
#include <string>
#include <string_view>
#include <unordered_map>
#include <vector>

namespace vox {

class Tokenizer {
  public:
    static constexpr uint32_t kTextTokenOffset = 1000;  // tokenizer/mod.rs:66
    static Tokenizer *from_json(const char *json, size_t len);
    static Tokenizer *from_file(const std::string &path);
    std::string decode(const uint32_t *ids, size_t n) const;
    bool decode_token(uint32_t id, std::string *out) const;
    size_t vocab_size() const { return vocab_size_; }
    // Tekken encode (tiktoken's encode with no special tokens): UTF-8 text -> text ids (vocab position + 1000).
    // VOX_EINVAL for invalid UTF-8; VOX_EFORMAT for a pattern other than Tekken's or a rank table without the 256
    // single bytes.  Thread-safe: the rank table is built once, on the first call.
    std::vector<int32_t> encode(const char *text, size_t len) const;
    // the first code point of valid UTF-8 text is White_Space (\s of the pattern)
    static bool starts_with_white_space(const char *text, size_t len);

  private:
    void build_ranks() const;

    std::vector<std::string> vocab_bytes_;
    std::vector<uint8_t> has_bytes_;
    std::map<uint32_t, std::string> special_;
    size_t vocab_size_ = 0;
    std::string pattern_;
    // encoder state, built by the first encode(): byte string -> vocab position (views into vocab_bytes_)
    mutable std::once_flag ranks_once_;
    mutable std::unordered_map<std::string_view, uint32_t> ranks_;
    mutable int32_t ranks_err_ = 0;   // VOX_E* when the vocabulary cannot encode
    mutable std::string ranks_msg_;
};

}  // namespace vox
