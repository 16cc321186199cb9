// C++ host mirror: ed25519::Curve::VerifyBatch (kyber_b200/host/kyber_b200.hpp) on cases read from a file, one per line:
// "<pk hex> <msg hex or -> <sig hex> <expected status>".  All cases go in one batch, then each in a batch of one.
#include <cstdio>
#include <fstream>
#include <sstream>
#include "../../kyber_b200/host/kyber_b200.hpp"

static std::vector<uint8_t> unhex(const std::string& s) {
  std::vector<uint8_t> out;
  if (s == "-") return out;
  for (size_t i = 0; i + 1 < s.size(); i += 2) out.push_back((uint8_t)std::stoul(s.substr(i, 2), nullptr, 16));
  return out;
}

int main(int argc, char** argv) {
  if (argc != 2) { fprintf(stderr, "usage: test_eddsa <cases file>\n"); return 2; }
  std::vector<b200::ed25519::PointBytes> pks;
  std::vector<std::vector<uint8_t>> msgs;
  std::vector<std::array<uint8_t, 64>> sigs;
  std::vector<int> want;
  std::ifstream f(argv[1]);
  std::string line;
  while (std::getline(f, line)) {
    std::istringstream ss(line);
    std::string pk, msg, sig;
    int code;
    if (!(ss >> pk >> msg >> sig >> code)) continue;
    auto p = unhex(pk), s = unhex(sig);
    if (p.size() != 32 || s.size() != 64) { fprintf(stderr, "bad case line\n"); return 2; }
    b200::ed25519::PointBytes pa;
    std::array<uint8_t, 64> sa;
    std::copy(p.begin(), p.end(), pa.begin());
    std::copy(s.begin(), s.end(), sa.begin());
    pks.push_back(pa); msgs.push_back(unhex(msg)); sigs.push_back(sa); want.push_back(code);
  }
  auto eng = std::make_shared<b200::Engine>(0);
  b200::ed25519::Curve curve(eng);
  int fails = 0;
  auto batch = curve.VerifyBatch(pks, msgs, sigs);
  for (size_t i = 0; i < want.size(); i++) {
    auto one = curve.VerifyBatch({pks[i]}, {msgs[i]}, {sigs[i]});
    bool ok = batch[i] == want[i] && one[0] == want[i];
    printf("%s case %zu: batch %d single %d want %d\n", ok ? "ok" : "FAIL", i, batch[i], one[0], want[i]);
    fails += !ok;
  }
  bool threw = false;
  try { curve.VerifyBatch(pks, msgs, {}); } catch (const std::logic_error&) { threw = true; }
  printf("%s length mismatch throws\n", threw ? "ok" : "FAIL");
  fails += !threw;
  printf(fails ? "FAILED\n" : "PASSED\n");
  return fails ? 1 : 0;
}
