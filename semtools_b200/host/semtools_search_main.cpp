// semtools_b200_search: `semtools search` (reference src/bin/semtools.rs:52-83,
// src/cmds/search.rs:113-276, non-workspace path) on the C++ host layer.
//   semtools_b200_search --vocab vocab.txt --table table.f32 QUERY [FILES...]
//       [-n N|--n-lines N|--context N] [--top-k K] [-m D|--max-distance D|--threshold D]
//       [-i|--ignore-case] [-j|--json]
// The model comes as a WordLevel vocabulary (one token per line) + a raw V x 256 f32 table;
// real model2vec checkpoints are tokenised by the Python host (semtools_b200/model.py).
// `--selftest` exercises the pure host functions without a GPU.
#include <unistd.h>

#include <chrono>
#include <cmath>
#include <random>
#include <thread>

#include <cstdio>
#include <cstring>
#include <fstream>
#include <iostream>
#include <iterator>

#include <memory>

#include "semtools_store.hpp"
#include "semtools_tokenizer.hpp"

using namespace semtools;

// Synthetic ingestion batch of SURVEY 8d: V = 500k words, line lengths ~ LogNormal(2.5, 0.8)
// clipped to [0, 2048], word ranks ~ Zipf(1.1); reports lines/s and tokens/s of tokenize_to_csr.
static int tokenize_bench(size_t n_lines, unsigned threads, const std::string &tokenizer_json = "") {
  std::vector<std::string> words;
  words.reserve(500000);
  for (uint64_t i = 0; i < 500000; ++i) words.push_back("t" + std::to_string(i * 7919 % 1000003));
  // with a tokenizer.json: the same synthetic lines go through the Unigram pipeline (the words are
  // then segmented into whatever pieces its vocabulary offers); without: the WordLevel tokenizer
  std::unique_ptr<Tokenizer> owner;
  if (!tokenizer_json.empty()) owner.reset(new HfTokenizer(tokenizer_json));
  else owner.reset(new WordLevelTokenizer(words));
  const Tokenizer &tok = *owner;
  std::mt19937_64 rng(12345);
  std::lognormal_distribution<double> len(2.5, 0.8);
  std::vector<double> cdf(500000);
  double acc = 0;
  for (int r = 0; r < 500000; ++r) { acc += 1.0 / std::pow(r + 1.0, 1.1); cdf[r] = acc; }
  std::uniform_real_distribution<double> uni(0.0, acc);
  std::vector<std::string> lines(n_lines);
  for (auto &l : lines) {
    const int nt = (int)std::min(2048.0, std::max(0.0, std::round(len(rng))));
    for (int t = 0; t < nt; ++t) {
      const size_t r = std::lower_bound(cdf.begin(), cdf.end(), uni(rng)) - cdf.begin();
      if (t) l += ' ';
      l += words[std::min<size_t>(r, 499999)];
    }
  }
  std::vector<uint64_t> off; std::vector<uint32_t> ids;
  for (unsigned th : {1u, threads}) {
    double best = 1e30;
    for (int rep = 0; rep < 3; ++rep) {
      const auto t0 = std::chrono::steady_clock::now();
      tokenize_to_csr(lines, tok, 2048, off, ids, th);
      best = std::min(best, std::chrono::duration<double>(std::chrono::steady_clock::now() - t0).count());
    }
    printf("{\"threads\": %u, \"lines\": %zu, \"tokens\": %zu, \"seconds\": %.4f, \"lines_per_s\": %.0f, \"tokens_per_s\": %.0f}\n",
           th ? th : std::thread::hardware_concurrency(), n_lines, ids.size(), best, n_lines / best, ids.size() / best);
    if (th == threads) break;
  }
  return 0;
}

static int selftest() {
  int bad = 0;
  auto expect = [&](const std::string &got, const std::string &want) {
    if (got != want) { fprintf(stderr, "selftest: got '%s' want '%s'\n", got.c_str(), want.c_str()); ++bad; }
  };
  expect(rust_display_f64(0.0), "0");
  expect(rust_display_f64(1.0), "1");
  expect(rust_display_f64(0.25), "0.25");
  expect(rust_display_f64(0.1 + 0.2), "0.30000000000000004");
  expect(rust_display_f64(1e-7), "0.0000001");
  expect(rust_display_f64(1e21), "1000000000000000000000");
  expect(json_f64(1.0), "1.0");
  expect(json_f64(0.00001), "0.00001");
  expect(json_f64(0.000001), "1e-6");
  expect(json_f64(2.220446049250313e-16), "2.220446049250313e-16");
  expect(json_string("a\"b\n\t\x01"), "\"a\\\"b\\n\\t\\u0001\"");
  auto l = rust_lines("a\r\nb\n\nc");
  if (l.size() != 4 || l[0] != "a" || l[2] != "" || l[3] != "c") { fprintf(stderr, "selftest: rust_lines\n"); ++bad; }
  if (!rust_lines("").empty() || rust_lines("\n").size() != 1) { fprintf(stderr, "selftest: rust_lines edge\n"); ++bad; }
  SearchResult r{"f.txt", {"x", "y", "z"}, 4, 7, 5, 0.5};
  expect(format_search_results({r}, false), "f.txt:4::7 (0.5)\n   5: x\n   6: y\n   7: z\n\n");
  expect(search_output_json({}), "{\n  \"results\": []\n}");
  {  // tokenize_to_csr: every thread count gives the serial result
    std::vector<std::string> words;
    for (int i = 0; i < 5000; ++i) words.push_back("w" + std::to_string(i));
    WordLevelTokenizer tok(words);
    std::vector<std::string> lines;
    uint64_t h = 88172645463325252ull;
    for (int i = 0; i < 3000; ++i) {
      std::string l;
      h ^= h << 13; h ^= h >> 7; h ^= h << 17;
      const int nt = (int)(h % 40);
      for (int t = 0; t < nt; ++t) { h ^= h << 13; h ^= h >> 7; h ^= h << 17; l += (t ? " " : "") + ((h % 7) ? "w" + std::to_string(h % 6000) : std::string("\tunk ")); }
      lines.push_back(l);
    }
    std::vector<uint64_t> o1, oN; std::vector<uint32_t> i1, iN;
    tokenize_to_csr(lines, tok, 16, o1, i1, 1);
    for (unsigned th : {2u, 3u, 8u}) {
      tokenize_to_csr(lines, tok, 16, oN, iN, th);
      if (o1 != oN || i1 != iN) { fprintf(stderr, "selftest: tokenize_to_csr differs with %u threads\n", th); ++bad; }
    }
    if (o1.size() != 3001 || o1.back() != i1.size() || i1.empty()) { fprintf(stderr, "selftest: tokenize_to_csr shape\n"); ++bad; }
    for (size_t i = 0; i < 3000; ++i) if (o1[i + 1] - o1[i] > 16) { fprintf(stderr, "selftest: truncation\n"); ++bad; break; }
  }
  printf(bad ? "selftest FAILED\n" : "selftest ok\n");
  return bad ? 1 : 0;
}

static int real_main(int argc, char **argv) {
  std::string vocab, tokenizer_json, table, model_dir, query;
  uint32_t tok_flags = 0;                        // --gpu-tokenizer utf8: STB_TOKENIZER_UTF8
  std::vector<std::string> files;
  SearchConfig cfg;
  bool json = false, have_query = false;
  std::optional<std::string> workspace_name;
  for (int i = 1; i < argc; ++i) {
    std::string a = argv[i];
    auto next = [&]() -> std::string { if (i + 1 >= argc) { fprintf(stderr, "error: %s needs a value\n", a.c_str()); exit(2); } return argv[++i]; };
    if (a == "--selftest") return selftest();
    if (a == "--tokenize-bench") {                 // host tokenisation throughput (SURVEY 8f-2): LINES THREADS
      const size_t n_lines = i + 1 < argc ? std::stoul(argv[i + 1]) : 1000000;
      const unsigned threads = i + 2 < argc ? (unsigned)std::stoul(argv[i + 2]) : 0;
      return tokenize_bench(n_lines, threads, i + 3 < argc ? argv[i + 3] : "");
    }
    if (a == "--encode") {                         // test hook: --encode tokenizer.json: stdin lines -> "raw ids | ids without unk"
      HfTokenizer tk(next());
      std::string in;
      char buf[65536];
      size_t n;
      while ((n = fread(buf, 1, sizeof(buf), stdin)) > 0) in.append(buf, n);
      printf("median_token_length %zu vocab %zu\n", tk.median_token_length(), tk.vocab_size());
      for (const auto &l : rust_lines(in)) {
        try {
          std::string o;
          for (uint32_t id : tk.encode_raw(l)) o += std::to_string(id) + " ";
          o += "|";
          for (uint32_t id : tk.encode(l)) o += " " + std::to_string(id);
          puts(o.c_str());
        } catch (const std::exception &e) { printf("ERROR %s\n", e.what()); }
      }
      return 0;
    }
    if (a == "--normalize") {                      // test hook: --normalize tokenizer.json: stdin lines -> normalizer output, one per line
      HfTokenizer tk(next());
      std::string in;
      char buf[65536];
      size_t n;
      while ((n = fread(buf, 1, sizeof(buf), stdin)) > 0) in.append(buf, n);
      for (const auto &l : rust_lines(in)) {
        try { const std::string o = tk.normalize_str(l); fwrite(o.data(), 1, o.size(), stdout); fputc('\n', stdout); }
        catch (const std::exception &e) { printf("ERROR %s\n", e.what()); }
      }
      return 0;
    }
    if (a == "--graphemes") {                      // test hook: stdin lines -> byte lengths of the extended grapheme clusters
      std::string in;
      char buf[65536];
      size_t n;
      while ((n = fread(buf, 1, sizeof(buf), stdin)) > 0) in.append(buf, n);
      for (const auto &l : rust_lines(in)) {
        std::string o;
        size_t b = 0;
        for (size_t e : grapheme_ends(l)) { o += std::to_string(e - b) + " "; b = e; }
        puts(o.c_str());
      }
      return 0;
    }
    if (a == "--model-info") {                     // test hook: what load_model_dir read (no GPU needed)
      ModelDir m;
      try { m = load_model_dir(next()); } catch (const std::exception &e) { fprintf(stderr, "Error: %s\n", e.what()); return 1; }
      auto h = [](const void *p, size_t n) { return (unsigned long long)stb_fnv1a64(reinterpret_cast<const uint8_t *>(p), n); };
      printf("{\"V\": %llu, \"normalize\": %s, \"n_weights\": %zu, \"n_mapping\": %zu, \"fingerprint\": \"%s\", \"table_fnv\": \"%016llx\", "
             "\"weights_fnv\": \"%016llx\", \"mapping_fnv\": \"%016llx\"}\n",
             (unsigned long long)m.V, m.normalize ? "true" : "false", m.weights.size(), m.mapping.size(), m.fingerprint.c_str(),
             h(m.E.data(), m.E.size() * 4), h(m.weights.data(), m.weights.size() * 4), h(m.mapping.data(), m.mapping.size() * 4));
      return 0;
    }
    if (a == "--lines") {                          // test hook: stdin -> rust_lines -> one JSON string per line
      std::string in;
      char buf[65536];
      size_t n;
      while ((n = fread(buf, 1, sizeof(buf), stdin)) > 0) in.append(buf, n);
      for (const auto &l : rust_lines(in)) {
        std::string o = "\"";
        for (unsigned char ch : l) {
          if (ch == '"' || ch == '\\') { o.push_back('\\'); o.push_back((char)ch); }
          else if (ch < 0x20) { char e[8]; snprintf(e, sizeof(e), "\\u%04x", ch); o += e; }
          else o.push_back((char)ch);
        }
        o += "\"\n";
        fwrite(o.data(), 1, o.size(), stdout);
      }
      return 0;
    }
    if (a == "--lower") {                          // test hook: stdin -> to_lowercase -> stdout
      std::string in, line;
      char buf[65536];
      size_t n;
      while ((n = fread(buf, 1, sizeof(buf), stdin)) > 0) in.append(buf, n);
      const std::string out = to_lowercase(in);
      fwrite(out.data(), 1, out.size(), stdout);
      return 0;
    }
    else if (a == "--vocab") vocab = next();
    else if (a == "--tokenizer") tokenizer_json = next();
    else if (a == "--table") table = next();
    else if (a == "--model") model_dir = next();
    else if (a == "--gpu-tokenizer") {
      const std::string g = next();
      if (g != "ascii" && g != "utf8") { fprintf(stderr, "Error: --gpu-tokenizer takes ascii or utf8\n"); return 2; }
      tok_flags = g == "utf8" ? STB_TOKENIZER_UTF8 : 0;
    }
    else if (a == "-n" || a == "--n-lines" || a == "--context") cfg.n_lines = std::stoul(next());
    else if (a == "--top-k") cfg.top_k = std::stoul(next());
    else if (a == "-m" || a == "--max-distance" || a == "--threshold") cfg.max_distance = std::stod(next());
    else if (a == "-i" || a == "--ignore-case") cfg.ignore_case = true;
    else if (a == "-j" || a == "--json") json = true;
    else if (a == "-w" || a == "--workspace") workspace_name = next();
    else if (!have_query) { query = a; have_query = true; }
    else files.push_back(a);
  }
  if (model_dir.empty() && vocab.empty() && tokenizer_json.empty() && table.empty())
    if (const char *e = getenv("SEMTOOLS_B200_MODEL_DIR"); e && *e) model_dir = e;              // as the Python CLI (__main__.py)
  if (!model_dir.empty() && vocab.empty() && tokenizer_json.empty() && table.empty()) tokenizer_json = model_dir + "/tokenizer.json";
  else if (!model_dir.empty()) { fprintf(stderr, "Error: --model replaces --tokenizer / --vocab / --table\n"); return 2; }
  if (!have_query || (vocab.empty() == tokenizer_json.empty()) || (table.empty() && model_dir.empty())) {
    fprintf(stderr, "usage: semtools_b200_search (--model DIR | (--tokenizer tokenizer.json | --vocab V) --table T) QUERY [FILES...] [-n N] [--top-k K] [-m D] [-i] [-j] [-w WORKSPACE]\n"
                    "       [--gpu-tokenizer ascii|utf8]\n"
                    "  --model:     a local model2vec directory (tokenizer.json, model.safetensors, config.json), as StaticModel::from_pretrained reads it\n"
                    "               (default: $SEMTOOLS_B200_MODEL_DIR, like the Python CLI)\n"
                    "  --tokenizer: the model's HF tokenizer.json (Unigram + Metaspace subset, see semtools_tokenizer.hpp)\n"
                    "  --vocab:     whitespace WordLevel vocabulary, one token per line (synthetic models)\n"
                    "  --gpu-tokenizer: which lines the GPU tokenises -- ascii (printable ASCII lines, the default) or utf8\n"
                    "               (every valid UTF-8 line); the other lines are tokenised on the host, with the same ids\n");
    return 2;
  }
  try {
    if (cfg.ignore_case) query = to_lowercase(query);
    const bool stdin_tty = isatty(0);
    std::vector<std::pair<std::string, std::string>> inputs;      // (filename, content)
    if (files.empty() && !stdin_tty) {
      std::string content((std::istreambuf_iterator<char>(std::cin)), std::istreambuf_iterator<char>());
      if (!content.empty()) inputs.emplace_back("<stdin>", content);
    }
    if (files.empty() && inputs.empty()) {
      const char *msg = "No input provided. Either specify files as arguments or pipe input to stdin.";
      if (json) fprintf(stderr, "{\n  \"error\": %s,\n  \"error_type\": \"NoInput\"\n}\n", json_string(msg).c_str());
      else fprintf(stderr, "Error: %s\n", msg);
      return 1;
    }
    std::unique_ptr<Tokenizer> tok_owner;
    if (!tokenizer_json.empty()) tok_owner.reset(new HfTokenizer(tokenizer_json));
    else tok_owner.reset(new WordLevelTokenizer(vocab));
    const Tokenizer &tok = *tok_owner;
    ModelDir md;
    std::vector<char> raw;
    if (!model_dir.empty()) md = load_model_dir(model_dir);
    else {
      std::ifstream tf(table, std::ios::binary);
      raw.assign((std::istreambuf_iterator<char>(tf)), std::istreambuf_iterator<char>());
      if (raw.empty() || raw.size() % (STB_DIM * sizeof(float))) { fprintf(stderr, "Error: bad table file\n"); return 1; }
    }
    const float *tab_E = model_dir.empty() ? reinterpret_cast<const float *>(raw.data()) : md.E.data();
    const uint64_t tab_V = model_dir.empty() ? raw.size() / (STB_DIM * sizeof(float)) : md.V;
    const bool tab_norm = model_dir.empty() ? true : md.normalize;
    std::string tok_text;                          // a tokenizer.json also goes to the library: lines are embedded from text
    if (!tokenizer_json.empty()) {
      std::ifstream tf(tokenizer_json, std::ios::binary);
      tok_text.assign((std::istreambuf_iterator<char>(tf)), std::istreambuf_iterator<char>());
    }
    auto load = [&](Searcher &s) {
      s.load_table(tab_E, tab_V, tab_norm, md.weights.data(), md.weights.size(), md.mapping.data(), md.mapping.size());
      if (!tok_text.empty()) s.load_text_tokenizer(tok_text, tok_flags);
    };
    // identity of this host's embedder, recorded in the store so its vectors are never mixed with another
    // host's / model's (ADVICE r1): a model directory gets the Python host's fingerprint string, the
    // synthetic forms (vocabulary file / bare tokenizer.json + raw table) their own
    char fp_buf[96];
    if (!model_dir.empty()) snprintf(fp_buf, sizeof(fp_buf), "%s", md.fingerprint.c_str());
    else {
      std::ifstream vf(tokenizer_json.empty() ? vocab : tokenizer_json, std::ios::binary);
      std::vector<char> vraw((std::istreambuf_iterator<char>(vf)), std::istreambuf_iterator<char>());
      const uint64_t hv = stb_fnv1a64(reinterpret_cast<const uint8_t *>(vraw.data()), vraw.size());
      const uint64_t ht = stb_fnv1a64(reinterpret_cast<const uint8_t *>(raw.data()), std::min<size_t>(raw.size(), 1u << 20));
      snprintf(fp_buf, sizeof(fp_buf), "%s:%zux256:%016llx", tokenizer_json.empty() ? "wordlevel" : "hf-unigram", raw.size() / (STB_DIM * sizeof(float)), (unsigned long long)(hv ^ (ht * 0x9E3779B97F4A7C15ull)));
    }
    const std::string fingerprint = fp_buf;
    bool in_workspace = false;
    if (!files.empty()) { try { Workspace::active(workspace_name); in_workspace = true; } catch (const std::exception &) {} }
    if (in_workspace) {
      // cmds/search.rs:194-241: persisted line embeddings, only new/changed files are embedded
      Searcher s(0);
      load(s);
      auto ranked = search_with_workspace(
          files, s.encode_single(query, tok),
          [&](const std::vector<std::string> &lines) { return s.embed_lines(lines, tok, cfg.ignore_case); }, cfg, workspace_name,
          [](const std::string &m) { fprintf(stderr, "%s\n", m.c_str()); }, 0, fingerprint);
      if (json) printf("%s\n", workspace_output_json(ranked, cfg.n_lines).c_str());
      else fputs(format_workspace_search_results(ranked, cfg.n_lines, isatty(1)).c_str(), stdout);
      return 0;
    }
    for (const auto &f : files) {
      std::ifstream in(f, std::ios::binary);
      if (!in) { fprintf(stderr, "Error: %s: No such file or directory (os error 2)\n", f.c_str()); return 1; }
      inputs.emplace_back(f, std::string((std::istreambuf_iterator<char>(in)), std::istreambuf_iterator<char>()));
    }
    Searcher s(0);
    load(s);
    for (const auto &in : inputs) s.add_document(in.first, in.second, tok, cfg.ignore_case);
    auto results = s.search_documents(s.encode_single(query, tok), cfg);
    if (json) printf("%s\n", search_output_json(results).c_str());
    else fputs(format_search_results(results, isatty(1)).c_str(), stdout);
  } catch (const std::exception &e) {
    fprintf(stderr, "Error: %s\n", e.what());
    return 1;
  }
  return 0;
}

// nothing a bad input file can throw ends in std::terminate: every exit is a message + status
int main(int argc, char **argv) {
  try {
    return real_main(argc, argv);
  } catch (const std::exception &e) {
    fprintf(stderr, "Error: %s\n", e.what());
    return 1;
  } catch (...) {
    fprintf(stderr, "Error: unknown failure\n");
    return 1;
  }
}
