// tokenizer.cpp -- Tekken tokenizer (reference src/tokenizer/mod.rs:70-214, decode only there).
// tekken.json -> per-vocab-index byte strings (base64 `token_bytes`, else UTF-8 of `token_str`);
// control entries (is_control) are kept in a rank->string map; decode() skips ids < 1000, maps
// id-1000 to the vocab *position*, silently skips unknown ids and returns lossy UTF-8.
// encode() is tiktoken's encode over the same positions (mistral_common's Tekkenizer.encode without BOS/EOS).
#include "tokenizer.h"

#include <algorithm>
#include <cstdlib>
#include <cctype>
#include <cstring>
#include <fstream>
#include <sstream>

#include "common.h"
#include "unicode_tables.h"

namespace vox {
namespace {

// ---- minimal JSON DOM ------------------------------------------------------------------
struct JVal {
    enum T { Null, Bool, Num, Str, Arr, Obj } t = Null;
    bool b = false;
    double num = 0;
    std::string s;
    std::vector<JVal> arr;
    std::vector<std::pair<std::string, JVal>> obj;
    const JVal *get(const char *k) const {
        for (auto &kv : obj)
            if (kv.first == k) return &kv.second;
        return nullptr;
    }
};

struct JParser {
    const char *p, *e;
    [[noreturn]] void err(const char *m) { fail(VOX_EIO, std::string("Failed to parse tekken JSON: ") + m); }
    void ws() { while (p < e && (*p == ' ' || *p == '\n' || *p == '\t' || *p == '\r')) ++p; }
    static void put_utf8(std::string &o, uint32_t c) {
        if (c < 0x80) o += (char)c;
        else if (c < 0x800) { o += (char)(0xC0 | (c >> 6)); o += (char)(0x80 | (c & 0x3F)); }
        else if (c < 0x10000) { o += (char)(0xE0 | (c >> 12)); o += (char)(0x80 | ((c >> 6) & 0x3F)); o += (char)(0x80 | (c & 0x3F)); }
        else { o += (char)(0xF0 | (c >> 18)); o += (char)(0x80 | ((c >> 12) & 0x3F)); o += (char)(0x80 | ((c >> 6) & 0x3F)); o += (char)(0x80 | (c & 0x3F)); }
    }
    uint32_t hex4() {
        if (e - p < 4) err("bad \\u escape");
        uint32_t v = 0;
        for (int i = 0; i < 4; ++i) {
            char c = *p++;
            v <<= 4;
            if (c >= '0' && c <= '9') v |= c - '0';
            else if (c >= 'a' && c <= 'f') v |= c - 'a' + 10;
            else if (c >= 'A' && c <= 'F') v |= c - 'A' + 10;
            else err("bad hex digit");
        }
        return v;
    }
    std::string str() {
        if (p >= e || *p != '"') err("expected string");
        ++p;
        std::string o;
        while (p < e && *p != '"') {
            char c = *p++;
            if (c != '\\') { o += c; continue; }
            if (p >= e) err("bad escape");
            char x = *p++;
            switch (x) {
                case '"': o += '"'; break;
                case '\\': o += '\\'; break;
                case '/': o += '/'; break;
                case 'b': o += '\b'; break;
                case 'f': o += '\f'; break;
                case 'n': o += '\n'; break;
                case 'r': o += '\r'; break;
                case 't': o += '\t'; break;
                case 'u': {
                    uint32_t c1 = hex4();
                    if (c1 >= 0xD800 && c1 < 0xDC00 && e - p >= 6 && p[0] == '\\' && p[1] == 'u') {
                        p += 2;
                        uint32_t c2 = hex4();
                        if (c2 >= 0xDC00 && c2 < 0xE000) c1 = 0x10000 + ((c1 - 0xD800) << 10) + (c2 - 0xDC00);
                        else { put_utf8(o, 0xFFFD); c1 = c2; }
                    }
                    if (c1 >= 0xD800 && c1 < 0xE000) c1 = 0xFFFD;  // lone surrogate
                    put_utf8(o, c1);
                    break;
                }
                default: err("unknown escape");
            }
        }
        if (p >= e) err("unterminated string");
        ++p;
        return o;
    }
    int depth = 0;
    struct Depth {   // recursion guard: a crafted "[[[[..." must be an error, not a stack overflow
        JParser &ps;
        explicit Depth(JParser &q) : ps(q) { if (++ps.depth > 64) ps.err("nesting deeper than 64"); }
        ~Depth() { --ps.depth; }
    };
    JVal val() {
        Depth guard(*this);
        ws();
        if (p >= e) err("unexpected end");
        JVal v;
        char c = *p;
        if (c == '{') {
            v.t = JVal::Obj;
            ++p; ws();
            if (p < e && *p == '}') { ++p; return v; }
            for (;;) {
                ws();
                std::string k = str();
                ws();
                if (p >= e || *p != ':') err("expected ':'");
                ++p;
                v.obj.emplace_back(std::move(k), val());
                ws();
                if (p < e && *p == ',') { ++p; continue; }
                if (p < e && *p == '}') { ++p; break; }
                err("expected ',' or '}'");
            }
        } else if (c == '[') {
            v.t = JVal::Arr;
            ++p; ws();
            if (p < e && *p == ']') { ++p; return v; }
            for (;;) {
                v.arr.push_back(val());
                ws();
                if (p < e && *p == ',') { ++p; continue; }
                if (p < e && *p == ']') { ++p; break; }
                err("expected ',' or ']'");
            }
        } else if (c == '"') {
            v.t = JVal::Str;
            v.s = str();
        } else if (c == 't' && e - p >= 4 && !strncmp(p, "true", 4)) { v.t = JVal::Bool; v.b = true; p += 4; }
        else if (c == 'f' && e - p >= 5 && !strncmp(p, "false", 5)) { v.t = JVal::Bool; v.b = false; p += 5; }
        else if (c == 'n' && e - p >= 4 && !strncmp(p, "null", 4)) { v.t = JVal::Null; p += 4; }
        else {
            // the buffer is length-delimited, not NUL-terminated: copy the numeric token into a bounded buffer
            // before strtod so that it cannot read past `e`
            char tmp[64];
            size_t n = 0;
            while (p + n < e && n + 1 < sizeof(tmp) && (isdigit((unsigned char)p[n]) || p[n] == '-' || p[n] == '+' || p[n] == '.' || p[n] == 'e' || p[n] == 'E')) {
                tmp[n] = p[n];
                ++n;
            }
            tmp[n] = '\0';
            char *end = nullptr;
            v.num = strtod(tmp, &end);
            if (n == 0 || end == tmp) err("bad number");
            v.t = JVal::Num;
            p += (end - tmp);
        }
        return v;
    }
};

// base64 STANDARD (with padding), strict like BASE64_STANDARD.decode: returns false on bad input.
bool b64_decode(const std::string &in, std::string &out) {
    static int8_t T[256];
    static bool init = false;
    if (!init) {
        memset(T, -1, sizeof(T));
        const char *A = "ABCDEFGHIJKLMNOPQRSTUVWXYZabcdefghijklmnopqrstuvwxyz0123456789+/";
        for (int i = 0; i < 64; ++i) T[(uint8_t)A[i]] = (int8_t)i;
        init = true;
    }
    out.clear();
    size_t n = in.size();
    if (n % 4 != 0) return false;
    for (size_t i = 0; i < n; i += 4) {
        int v[4];
        int pad = 0;
        for (int j = 0; j < 4; ++j) {
            char c = in[i + j];
            if (c == '=') {
                if (i + 4 != n || j < 2) return false;
                v[j] = 0;
                ++pad;
            } else {
                if (pad) return false;
                v[j] = T[(uint8_t)c];
                if (v[j] < 0) return false;
            }
        }
        uint32_t w = (v[0] << 18) | (v[1] << 12) | (v[2] << 6) | v[3];
        out += (char)(w >> 16);
        if (pad < 2) out += (char)((w >> 8) & 0xFF);
        if (pad < 1) out += (char)(w & 0xFF);
    }
    return true;
}

// String::from_utf8_lossy: invalid sequences -> U+FFFD (maximal-subpart replacement).
std::string utf8_lossy(const std::string &in) {
    std::string o;
    const uint8_t *s = (const uint8_t *)in.data();
    size_t n = in.size(), i = 0;
    auto rep = [&]() { o += "\xEF\xBF\xBD"; };
    while (i < n) {
        uint8_t c = s[i];
        if (c < 0x80) { o += (char)c; ++i; continue; }
        int need;
        uint8_t lo = 0x80, hi = 0xBF;
        if (c >= 0xC2 && c <= 0xDF) need = 1;
        else if (c == 0xE0) { need = 2; lo = 0xA0; }
        else if (c >= 0xE1 && c <= 0xEC) need = 2;
        else if (c == 0xED) { need = 2; hi = 0x9F; }
        else if (c >= 0xEE && c <= 0xEF) need = 2;
        else if (c == 0xF0) { need = 3; lo = 0x90; }
        else if (c >= 0xF1 && c <= 0xF3) need = 3;
        else if (c == 0xF4) { need = 3; hi = 0x8F; }
        else { rep(); ++i; continue; }
        size_t j = i + 1;
        bool ok = true;
        for (int k = 0; k < need; ++k, ++j) {
            if (j >= n) { ok = false; break; }
            uint8_t d = s[j];
            uint8_t l = k == 0 ? lo : 0x80, h = k == 0 ? hi : 0xBF;
            if (d < l || d > h) { ok = false; break; }
        }
        if (ok) { o.append(in, i, need + 1); i += need + 1; }
        else { rep(); i = j > i + 1 ? j : i + 1; }
    }
    return o;
}

// ---- Tekken encoder: pre-tokenizer over code points, then tiktoken's byte-pair merge inside each piece ----------
// The one pattern the encoder knows (config.pattern of every Tekken vocabulary), matched by match_piece() below.
const char kTekkenPattern[] =
    R"([^\r\n\p{L}\p{N}]?[\p{Lu}\p{Lt}\p{Lm}\p{Lo}\p{M}]*[\p{Ll}\p{Lm}\p{Lo}\p{M}]+|)"
    R"([^\r\n\p{L}\p{N}]?[\p{Lu}\p{Lt}\p{Lm}\p{Lo}\p{M}]+[\p{Ll}\p{Lm}\p{Lo}\p{M}]*|)"
    R"(\p{N}| ?[^\s\p{L}\p{N}]+[\r\n/]*|\s*[\r\n]+|\s+(?!\S)|\s+)";

// per-code-point flags: the pattern's classes
enum : uint8_t {
    fL = 1,      // \p{L}
    fN = 2,      // \p{N}
    fWS = 4,     // \s (White_Space)
    fU = 8,      // [\p{Lu}\p{Lt}\p{Lm}\p{Lo}\p{M}]
    fLw = 16,    // [\p{Ll}\p{Lm}\p{Lo}\p{M}]
    fCRLF = 32,  // [\r\n]
    fTail = 64,  // [\r\n/]
};

uint8_t char_flags(uint32_t c) {
    int lo = 0, hi = uni::kNumRanges - 1, cls = 0;
    while (lo <= hi) {
        const int mid = (lo + hi) / 2;
        if (c < uni::kUniRanges[mid].lo) hi = mid - 1;
        else if (c > uni::kUniRanges[mid].hi) lo = mid + 1;
        else { cls = uni::kUniRanges[mid].cls; break; }
    }
    uint8_t f = 0;
    switch (cls) {
        case uni::kLu: case uni::kLt: f = fL | fU; break;
        case uni::kLl: f = fL | fLw; break;
        case uni::kLm: case uni::kLo: f = fL | fU | fLw; break;
        case uni::kM: f = fU | fLw; break;
        case uni::kN: f = fN; break;
        default: break;
    }
    for (uint32_t w : uni::kWhiteSpace)
        if (c == w) f |= fWS;
    if (c == '\r' || c == '\n') f |= fCRLF | fTail;
    if (c == '/') f |= fTail;
    return f;
}

// [^\r\n\p{L}\p{N}] and [^\s\p{L}\p{N}]
bool is_lead(uint8_t f) { return !(f & (fL | fN | fCRLF)); }
bool is_punct(uint8_t f) { return !(f & (fL | fN | fWS)); }

// strict UTF-8 -> code points and their byte offsets (offs has one more entry: the end)
void utf8_decode(const uint8_t *s, size_t n, std::vector<uint32_t> &cps, std::vector<size_t> &offs) {
    size_t i = 0;
    while (i < n) {
        const uint8_t c = s[i];
        offs.push_back(i);
        if (c < 0x80) { cps.push_back(c); ++i; continue; }
        int need;
        uint8_t lo = 0x80, hi = 0xBF;
        uint32_t cp;
        if (c >= 0xC2 && c <= 0xDF) { need = 1; cp = c & 0x1F; }
        else if (c >= 0xE0 && c <= 0xEF) { need = 2; cp = c & 0x0F; if (c == 0xE0) lo = 0xA0; if (c == 0xED) hi = 0x9F; }
        else if (c >= 0xF0 && c <= 0xF4) { need = 3; cp = c & 0x07; if (c == 0xF0) lo = 0x90; if (c == 0xF4) hi = 0x8F; }
        else fail(VOX_EINVAL, fmt("encode: invalid UTF-8 byte 0x%02X at offset %zu", c, i));
        VOX_CHECK(n - i > (size_t)need, VOX_EINVAL, "encode: truncated UTF-8 sequence at offset %zu", i);
        for (int k = 1; k <= need; ++k) {
            const uint8_t d = s[i + k];
            VOX_CHECK(d >= (k == 1 ? lo : 0x80) && d <= (k == 1 ? hi : 0xBF), VOX_EINVAL,
                      "encode: invalid UTF-8 sequence at offset %zu", i);
            cp = (cp << 6) | (d & 0x3F);
        }
        cps.push_back(cp);
        i += need + 1;
    }
    offs.push_back(n);
}

// end of the maximal run of code points from k that have one of `mask`'s flags
size_t run_end(const std::vector<uint8_t> &f, size_t k, uint8_t mask) {
    while (k < f.size() && (f[k] & mask)) ++k;
    return k;
}

// The pattern's match at code point i (regex semantics: the first alternative that matches, greedy quantifiers that
// give back characters); returns its end.  Every code point starts a match, so pieces tile the text.
size_t match_piece(const std::vector<uint32_t> &cp, const std::vector<uint8_t> &f, size_t i) {
    const size_t n = f.size(), none = SIZE_MAX;
    // U* Lw+ from j: the star gives back characters (U and Lw overlap on Lm, Lo, M) until the plus can match
    auto upper_lower = [&](size_t j) -> size_t {
        const size_t kmax = run_end(f, j, fU);
        for (size_t k = kmax + 1; k-- > j;)
            if (k < n && (f[k] & fLw)) return run_end(f, k, fLw);
        return none;
    };
    // U+ Lw*
    auto upper_then = [&](size_t j) -> size_t {
        const size_t kmax = run_end(f, j, fU);
        return kmax > j ? run_end(f, kmax, fLw) : none;
    };
    const bool lead = is_lead(f[i]);   // the optional leading character: tried with it first, then without
    size_t e;
    if (lead && (e = upper_lower(i + 1)) != none) return e;                  // 1
    if ((e = upper_lower(i)) != none) return e;
    if (lead && (e = upper_then(i + 1)) != none) return e;                   // 2
    if ((e = upper_then(i)) != none) return e;
    if (f[i] & fN) return i + 1;                                              // 3
    const size_t p0 = (cp[i] == ' ' && i + 1 < n && is_punct(f[i + 1])) ? i + 1 : i;   // 4
    if (is_punct(f[p0])) {
        size_t k = p0;
        while (k < n && is_punct(f[k])) ++k;
        return run_end(f, k, fTail);
    }
    const size_t w = run_end(f, i, fWS);
    for (size_t k = w; k-- > i;)                                              // 5: \s* gives back to [\r\n]+
        if (f[k] & fCRLF) return run_end(f, k, fCRLF);
    if (w > i && w == n) return w;                                            // 6: \s+(?!\S)
    if (w > i + 1) return w - 1;                                              //    the last space goes to the next word
    if (w > i) return w;                                                      // 7
    return i + 1;   // unreachable: a code point is a letter, a number, White_Space or [^\s\p{L}\p{N}]
}

}  // namespace

bool Tokenizer::starts_with_white_space(const char *text, size_t len) {
    if (len == 0) return false;
    const size_t first = (uint8_t)text[0] < 0x80 ? 1 : (uint8_t)text[0] < 0xE0 ? 2 : (uint8_t)text[0] < 0xF0 ? 3 : 4;
    std::vector<uint32_t> cps;
    std::vector<size_t> offs;
    utf8_decode((const uint8_t *)text, std::min(first, len), cps, offs);
    return (char_flags(cps[0]) & fWS) != 0;
}

void Tokenizer::build_ranks() const {
    if (pattern_ != kTekkenPattern) {
        ranks_err_ = VOX_EFORMAT;
        ranks_msg_ = "encode: the tokenizer's pattern is not Tekken's; only decoding is available";
        return;
    }
    // text ranks below default_vocab_size - 1000, as mistral_common cuts them; the lowest position of a byte string wins
    const size_t cut = std::min(vocab_bytes_.size(), vocab_size_ > kTextTokenOffset ? vocab_size_ - kTextTokenOffset : 0);
    ranks_.reserve(cut);
    for (size_t p = 0; p < cut; ++p)
        if (has_bytes_[p] && !vocab_bytes_[p].empty()) ranks_.emplace(std::string_view(vocab_bytes_[p]), (uint32_t)p);
    for (int b = 0; b < 256; ++b) {
        const char c = (char)b;
        if (!ranks_.count(std::string_view(&c, 1))) {
            ranks_err_ = VOX_EFORMAT;
            ranks_msg_ = fmt("encode: the vocabulary (cut at %zu text ranks) has no token for byte 0x%02X", cut, b);
            ranks_.clear();
            return;
        }
    }
}

std::vector<int32_t> Tokenizer::encode(const char *text, size_t len) const {
    std::call_once(ranks_once_, [this] { build_ranks(); });
    if (ranks_err_) fail(ranks_err_, ranks_msg_);
    std::vector<uint32_t> cps;
    std::vector<size_t> offs;
    utf8_decode((const uint8_t *)text, len, cps, offs);
    std::vector<uint8_t> f(cps.size());
    for (size_t k = 0; k < cps.size(); ++k) f[k] = char_flags(cps[k]);
    std::vector<int32_t> out;
    std::vector<std::pair<size_t, uint32_t>> parts;   // (byte start, rank of the pair starting here)
    auto rank_of = [&](std::string_view v) -> uint32_t {
        auto it = ranks_.find(v);
        return it == ranks_.end() ? UINT32_MAX : it->second;
    };
    for (size_t i = 0; i < cps.size();) {
        const size_t e = match_piece(cps, f, i);
        const std::string_view piece(text + offs[i], offs[e] - offs[i]);
        i = e;
        const uint32_t whole = rank_of(piece);
        if (whole != UINT32_MAX) { out.push_back((int32_t)(whole + kTextTokenOffset)); continue; }
        // tiktoken's byte_pair_merge: merge the adjacent pair of lowest rank (the leftmost on a tie) until none is a token
        const size_t m = piece.size();
        parts.clear();
        for (size_t k = 0; k + 1 < m; ++k) parts.emplace_back(k, rank_of(piece.substr(k, 2)));
        parts.emplace_back(m - 1, UINT32_MAX);
        parts.emplace_back(m, UINT32_MAX);
        auto pair_rank = [&](size_t k) {
            return k + 3 < parts.size() ? rank_of(piece.substr(parts[k].first, parts[k + 3].first - parts[k].first)) : UINT32_MAX;
        };
        for (;;) {
            size_t best = SIZE_MAX;
            uint32_t r = UINT32_MAX;
            for (size_t k = 0; k + 1 < parts.size(); ++k)
                if (parts[k].second < r) { r = parts[k].second; best = k; }
            if (best == SIZE_MAX) break;
            if (best > 0) parts[best - 1].second = pair_rank(best - 1);
            parts[best].second = pair_rank(best);
            parts.erase(parts.begin() + best + 1);
        }
        for (size_t k = 0; k + 1 < parts.size(); ++k) {
            const uint32_t t = rank_of(piece.substr(parts[k].first, parts[k + 1].first - parts[k].first));
            out.push_back((int32_t)(t + kTextTokenOffset));   // every part is a token: the 256 bytes are
        }
    }
    return out;
}

Tokenizer *Tokenizer::from_json(const char *json, size_t len) {
    JParser jp{json, json + len};
    JVal root = jp.val();
    VOX_CHECK(root.t == JVal::Obj, VOX_EIO, "Failed to parse tekken JSON: root is not an object");
    const JVal *cfg = root.get("config");
    const JVal *vocab = root.get("vocab");
    VOX_CHECK(cfg && cfg->t == JVal::Obj, VOX_EIO, "Failed to parse tekken JSON: missing field `config`");
    VOX_CHECK(vocab && vocab->t == JVal::Arr, VOX_EIO, "Failed to parse tekken JSON: missing field `vocab`");
    const JVal *dvs = cfg->get("default_vocab_size");
    VOX_CHECK(dvs && dvs->t == JVal::Num, VOX_EIO, "Failed to parse tekken JSON: missing field `default_vocab_size`");
    Tokenizer *t = new Tokenizer();
    t->vocab_size_ = (size_t)dvs->num;
    const JVal *pat = cfg->get("pattern");
    if (pat && pat->t == JVal::Str) t->pattern_ = pat->s;
    t->vocab_bytes_.resize(vocab->arr.size());
    t->has_bytes_.assign(vocab->arr.size(), 0);
    for (size_t idx = 0; idx < vocab->arr.size(); ++idx) {
        const JVal &e = vocab->arr[idx];
        if (e.t != JVal::Obj) continue;
        const JVal *rank = e.get("rank");
        const JVal *tb = e.get("token_bytes");
        const JVal *ts = e.get("token_str");
        const JVal *ic = e.get("is_control");
        bool is_control = ic && ic->t == JVal::Bool && ic->b;
        if (is_control) {
            if (ts && ts->t == JVal::Str && rank && rank->t == JVal::Num) t->special_[(uint32_t)rank->num] = ts->s;
            continue;
        }
        if (tb && tb->t == JVal::Str) {
            std::string raw;
            if (b64_decode(tb->s, raw)) {
                t->vocab_bytes_[idx] = raw;
                t->has_bytes_[idx] = 1;
                continue;
            }
        }
        if (ts && ts->t == JVal::Str) {
            t->vocab_bytes_[idx] = ts->s;
            t->has_bytes_[idx] = 1;
        }
    }
    return t;
}

Tokenizer *Tokenizer::from_file(const std::string &path) {
    std::ifstream f(path, std::ios::binary);
    VOX_CHECK(f.good(), VOX_EIO, "Failed to open tokenizer file: %s", path.c_str());
    std::stringstream ss;
    ss << f.rdbuf();
    std::string s = ss.str();
    return from_json(s.data(), s.size());
}

std::string Tokenizer::decode(const uint32_t *ids, size_t n) const {
    std::string bytes;
    for (size_t i = 0; i < n; ++i) {
        uint32_t id = ids[i];
        if (id < kTextTokenOffset) continue;
        size_t v = id - kTextTokenOffset;
        if (v < vocab_bytes_.size() && has_bytes_[v]) bytes += vocab_bytes_[v];
    }
    return utf8_lossy(bytes);
}

bool Tokenizer::decode_token(uint32_t id, std::string *out) const {
    if (id < kTextTokenOffset) {
        auto it = special_.find(id);
        if (it == special_.end()) return false;
        *out = it->second;
        return true;
    }
    size_t v = id - kTextTokenOffset;
    if (v < vocab_bytes_.size() && has_bytes_[v]) {
        *out = utf8_lossy(vocab_bytes_[v]);
        return true;
    }
    return false;
}

}  // namespace vox
