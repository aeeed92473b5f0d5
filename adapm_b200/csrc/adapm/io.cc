#include "io.h"

#include <algorithm>
#include <cerrno>
#include <cstdlib>
#include <cstring>
#include <fstream>

#include "log.h"

namespace adapm {

namespace {
std::string slurp(const std::string& path) {
  std::ifstream f(path, std::ios::binary);
  ADAPM_CHECK(f.good(), "cannot open '" << path << "'");
  f.seekg(0, std::ios::end);
  const std::streamoff n = f.tellg();
  f.seekg(0, std::ios::beg);
  std::string s((size_t)n, '\0');
  f.read(&s[0], n);
  return s;
}
inline const char* skip_ws(const char* p, const char* e) {
  while (p < e && (*p == ' ' || *p == '\t' || *p == '\r' || *p == '\n')) ++p;
  return p;
}
inline const char* line_end(const char* p, const char* e) {
  const void* q = memchr(p, '\n', (size_t)(e - p));
  return q ? (const char*)q : e;
}
}  // namespace

std::vector<int64_t> read_triples_file(const std::string& path) {
  const std::string buf = slurp(path);
  const char* p = buf.data();
  const char* e = p + buf.size();
  std::vector<int64_t> out;
  out.reserve(buf.size() / 4);
  while (true) {
    p = skip_ws(p, e);
    if (p >= e) break;
    char* q = nullptr;
    const long long v = strtoll(p, &q, 10);
    ADAPM_CHECK(q != p, path << ": not an integer near byte " << (p - buf.data()));
    out.push_back((int64_t)v);
    p = q;
  }
  ADAPM_CHECK(out.size() % 3 == 0, path << ": the number of values (" << out.size() << ") is not a multiple of 3");
  return out;
}

CooMatrix read_matrix_market_coo_file(const std::string& path) {
  const std::string buf = slurp(path);
  const char* p = buf.data();
  const char* e = p + buf.size();
  ADAPM_CHECK(buf.compare(0, 32, "%%MatrixMarket matrix coordinate") == 0, path << ": not a MatrixMarket coordinate file");
  // comment lines
  while (p < e && *p == '%') p = line_end(p, e) + 1;
  CooMatrix m;
  char* q = nullptr;
  m.rows = strtoll(p, &q, 10); p = q;
  m.cols = strtoll(p, &q, 10); p = q;
  const long long nnz = strtoll(p, &q, 10); p = q;
  ADAPM_CHECK(m.rows > 0 && m.cols > 0 && nnz >= 0, path << ": bad size line");
  m.i.reserve((size_t)nnz); m.j.reserve((size_t)nnz); m.x.reserve((size_t)nnz);
  for (long long k = 0; k < nnz; ++k) {
    p = skip_ws(p, e);
    ADAPM_CHECK(p < e, path << ": " << nnz << " entries announced, " << k << " found");
    const long long i = strtoll(p, &q, 10); p = q;
    const long long j = strtoll(p, &q, 10); p = q;
    const double x = strtod(p, &q);
    ADAPM_CHECK(q != p, path << ": malformed entry " << k);
    p = q;
    ADAPM_CHECK(i >= 1 && i <= m.rows && j >= 1 && j <= m.cols, path << ": entry " << k << " is outside the matrix");
    m.i.push_back(i - 1); m.j.push_back(j - 1); m.x.push_back((float)x);
  }
  return m;
}

EdgeList read_edge_list_file(const std::string& path) {
  const std::string buf = slurp(path);
  const char* p = buf.data();
  const char* e = p + buf.size();
  EdgeList g;
  int fields = 0;                      // 2 or 3, set by the first data line
  for (int64_t line = 1; p < e; ++line) {
    const char* le = line_end(p, e);
    const char* f[4];
    const char* fe[4];
    int nf = 0;
    for (const char* q = p; q < le;) {
      while (q < le && (*q == ' ' || *q == '\t' || *q == '\r')) ++q;
      if (q >= le) break;
      const char* s = q;
      while (q < le && *q != ' ' && *q != '\t' && *q != '\r') ++q;
      if (nf < 4) { f[nf] = s; fe[nf] = q; }
      ++nf;
    }
    p = le + 1;
    if (nf == 0 || *f[0] == '#') continue;
    ADAPM_CHECK(nf == 2 || nf == 3, path << ":" << line << ": expected 'src dst [weight]', found " << nf << " fields");
    if (fields == 0) fields = nf;
    ADAPM_CHECK(nf == fields, path << ":" << line << ": " << nf << " fields, but the first edge line has " << fields);
    for (int k = 0; k < 2; ++k) {
      char* q = nullptr;
      errno = 0;
      const long long v = strtoll(f[k], &q, 10);
      ADAPM_CHECK(q == fe[k] && errno == 0, path << ":" << line << ": '" << std::string(f[k], fe[k])
                                                  << "' is not an integer node id");
      ADAPM_CHECK(v >= 0, path << ":" << line << ": negative node id " << v);
      (k == 0 ? g.src : g.dst).push_back((int64_t)v);
    }
    if (nf == 3) {
      char* q = nullptr;
      const double w = strtod(f[2], &q);
      ADAPM_CHECK(q == fe[2], path << ":" << line << ": '" << std::string(f[2], fe[2]) << "' is not a number");
      g.weight.push_back(w);
    }
  }
  g.ids.reserve(2 * g.src.size());
  g.ids.insert(g.ids.end(), g.src.begin(), g.src.end());
  g.ids.insert(g.ids.end(), g.dst.begin(), g.dst.end());
  std::sort(g.ids.begin(), g.ids.end());
  g.ids.erase(std::unique(g.ids.begin(), g.ids.end()), g.ids.end());
  for (auto* v : {&g.src, &g.dst})
    for (int64_t& x : *v) x = std::lower_bound(g.ids.begin(), g.ids.end(), x) - g.ids.begin();
  return g;
}

}  // namespace adapm
