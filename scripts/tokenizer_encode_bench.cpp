// tokenizer_encode_bench.cpp -- host figures of the Tekken encoder (DESIGN §9): JSON parse time, the one-time rank-table
// build (time and heap bytes, mallinfo2) and encoding a 256-word bias list with its leading-space forms.
// Build from the repository root, then run on a tekken.json:
//   g++ -O2 -std=c++17 -Ivoxtral_mini_realtime_rs_b200/csrc -Iinclude scripts/tokenizer_encode_bench.cpp
//       voxtral_mini_realtime_rs_b200/csrc/tokenizer.cpp -o /tmp/tokbench
//   /tmp/tokbench path/to/tekken.json
#include <chrono>
#include <cstdio>
#include <fstream>
#include <sstream>
#include <string>
#include <vector>
#include "tokenizer.h"
#include <malloc.h>
using namespace vox;
int main(int argc, char **argv) {
    std::ifstream f(argv[1], std::ios::binary); std::stringstream ss; ss << f.rdbuf(); std::string j = ss.str();
    auto t0 = std::chrono::steady_clock::now();
    Tokenizer *t = Tokenizer::from_json(j.data(), j.size());
    auto t1 = std::chrono::steady_clock::now();
    long r0 = (long)(mallinfo2().uordblks / 1024);
    auto t2 = std::chrono::steady_clock::now();
    t->encode("", 0);
    auto t3 = std::chrono::steady_clock::now();
    long r1 = (long)(mallinfo2().uordblks / 1024);
    // 256 words, each with its leading-space form, as set_bias_text expands them
    std::vector<std::string> words;
    const char *base[] = {"Kubernetes", "Zürich", "PyTorch", "transcription", "Genève", "phonograph", "Voxtral", "São Paulo"};
    for (int i = 0; i < 256; ++i) words.push_back(std::string(base[i % 8]) + (i >= 8 ? std::to_string(i) : ""));
    double best = 1e9; size_t total = 0;
    for (int rep = 0; rep < 20; ++rep) {
        auto a = std::chrono::steady_clock::now();
        total = 0;
        for (auto &w : words) { total += t->encode(w.data(), w.size()).size(); std::string s = " " + w; total += t->encode(s.data(), s.size()).size(); }
        auto b = std::chrono::steady_clock::now();
        best = std::min(best, std::chrono::duration<double, std::milli>(b - a).count());
    }
    printf("parse %.1f ms; rank table build %.2f ms, heap +%.1f MB; 256 words x 2 forms: %.3f ms (best of 20), %zu ids\n",
           std::chrono::duration<double, std::milli>(t1 - t0).count(), std::chrono::duration<double, std::milli>(t3 - t2).count(),
           (r1 - r0) / 1024.0, best, total);
}
