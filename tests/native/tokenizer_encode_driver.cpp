// tests/native/tokenizer_encode_driver.cpp -- AddressSanitizer / UBSan exercise of the Tekken encoder (tokenizer.cpp):
// random bytes, random and truncated UTF-8, every prefix of multi-byte text, and vocabularies with missing or duplicated
// tokens or another pattern.  Invalid text must fail with VOX_EINVAL, an unusable vocabulary with VOX_EFORMAT, and valid
// text must decode back to itself -- never a memory error.  Built and run by tests/test_tokenizer_encode_sanitizers.py.
// argv: a synthetic BPE tekken.json, the same with byte tokens cut away, with a duplicated token, with another pattern.
#include <cstdio>
#include <fstream>
#include <random>
#include <sstream>
#include <string>
#include <thread>
#include <vector>
#include "common.h"
#include "tokenizer.h"
using namespace vox;

static std::string slurp(const char *p) { std::ifstream f(p, std::ios::binary); std::stringstream ss; ss << f.rdbuf(); return ss.str(); }

static void put_utf8(std::string &o, uint32_t c) {
    if (c < 0x80) o += (char)c;
    else if (c < 0x800) { o += (char)(0xC0 | (c >> 6)); o += (char)(0x80 | (c & 0x3F)); }
    else if (c < 0x10000) { o += (char)(0xE0 | (c >> 12)); o += (char)(0x80 | ((c >> 6) & 0x3F)); o += (char)(0x80 | (c & 0x3F)); }
    else { o += (char)(0xF0 | (c >> 18)); o += (char)(0x80 | ((c >> 12) & 0x3F)); o += (char)(0x80 | ((c >> 6) & 0x3F)); o += (char)(0x80 | (c & 0x3F)); }
}

static int failures = 0;
#define EXPECT(c) do { if (!(c)) { fprintf(stderr, "FAILED %s (line %d)\n", #c, __LINE__); ++failures; } } while (0)

// encode: returns the VOX_E* code (0 on success); on success decode must give the text back
static int try_encode(const Tokenizer *t, const std::string &s, bool check_roundtrip) {
    try {
        std::vector<int32_t> ids = t->encode(s.data(), s.size());
        std::vector<uint32_t> u(ids.begin(), ids.end());
        for (int32_t id : ids) EXPECT(id >= (int32_t)Tokenizer::kTextTokenOffset);
        if (check_roundtrip) EXPECT(t->decode(u.data(), u.size()) == s);
        return 0;
    } catch (const Error &e) {
        return e.code;
    }
}

int main(int argc, char **argv) {
    if (argc < 5) { fprintf(stderr, "usage: drv bpe.json cut.json dup.json pattern.json\n"); return 2; }
    std::string j = slurp(argv[1]);
    Tokenizer *t = Tokenizer::from_json(j.data(), j.size());
    std::mt19937 rng(7);
    // ---- random bytes: valid or VOX_EINVAL, never anything else
    int ok = 0, inval = 0;
    for (int i = 0; i < 20000; ++i) {
        std::string s(rng() % 24, '\0');
        for (auto &c : s) c = (char)(rng() % 4 ? rng() % 256 : 0x80 + rng() % 64);
        const int r = try_encode(t, s, true);
        EXPECT(r == 0 || r == VOX_EINVAL);
        (r == 0 ? ok : inval)++;
    }
    printf("random bytes: %d encoded, %d refused\n", ok, inval);
    // ---- random valid UTF-8 over the whole code space (surrogates excluded) and every truncation of it
    const uint32_t tops[] = {0x80, 0x800, 0x10000, 0x110000};
    int trunc_refused = 0;
    for (int i = 0; i < 4000; ++i) {
        std::string s;
        const int n = 1 + rng() % 10;
        for (int k = 0; k < n; ++k) {
            uint32_t c;
            do { c = rng() % tops[rng() % 4]; } while (c >= 0xD800 && c < 0xE000);
            if (rng() % 5 == 0) c = " \t\r\n/"[rng() % 5];
            put_utf8(s, c);
        }
        EXPECT(try_encode(t, s, true) == 0);
        for (size_t cut = 0; cut < s.size(); ++cut) {
            const std::string p = s.substr(0, cut);
            const int r = try_encode(t, p, true);
            EXPECT(r == 0 || r == VOX_EINVAL);
            trunc_refused += r == VOX_EINVAL;
        }
    }
    printf("truncated UTF-8: %d refused\n", trunc_refused);
    // ---- long runs (the quadratic merge loop and the whitespace alternatives over whole inputs)
    EXPECT(try_encode(t, std::string(3000, ' '), true) == 0);
    EXPECT(try_encode(t, std::string(2000, 'a') + "\r\n" + std::string(500, '\t') + "x", true) == 0);
    {
        std::string marks = "a";
        for (int k = 0; k < 500; ++k) put_utf8(marks, 0x0301);
        EXPECT(try_encode(t, marks, true) == 0);
    }
    // ---- two threads on one fresh handle (the rank table is built once)
    {
        Tokenizer *f = Tokenizer::from_json(j.data(), j.size());
        std::vector<int32_t> a, b;
        std::thread x([&] { a = f->encode("the transcription of Zurich", 27); });
        std::thread y([&] { b = f->encode("the transcription of Zurich", 27); });
        x.join(); y.join();
        EXPECT(!a.empty() && a == b);
        delete f;
    }
    delete t;
    // ---- vocabularies that cannot encode, and a duplicated token
    for (int v = 2; v <= 4; ++v) {
        std::string jv = slurp(argv[v]);
        Tokenizer *x = Tokenizer::from_json(jv.data(), jv.size());
        const int r1 = try_encode(x, "hello world", true), r2 = try_encode(x, "", true);
        if (v == 3) EXPECT(r1 == 0 && r2 == 0);
        else EXPECT(r1 == VOX_EFORMAT && r2 == VOX_EFORMAT);
        std::vector<uint32_t> ids = {1000 + 'h', 1000 + 'i'};
        EXPECT(x->decode(ids.data(), ids.size()).size() <= 2);   // decoding keeps working
        delete x;
    }
    printf("%s\n", failures ? "FAILED" : "done");
    return failures ? 1 : 0;
}
