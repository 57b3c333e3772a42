// CPU program of the .zkey / .wtns parser (ethrex_b200/csrc/zkey_parse.cpp), run by tests/test_zkey_host.py.
// One request per stdin line, one answer per stdout line:
//   zkey <path>           -> "<status> <message>": the parse, then zkey_coef_check over every section-4 record (the check
//                            the loader runs on the device); "0 ok <nVars> <nPublic> <log_n> <nCoefs>" when accepted
//   wtns <path> <nVars>   -> "<status> <message>"; "0 ok" when accepted
#include <cstdio>
#include <cstring>
#include <fstream>
#include <iostream>
#include <iterator>
#include <sstream>
#include <string>
#include <vector>

#include "zkey_parse.h"

using namespace b200zk;

static std::vector<uint8_t> slurp(const std::string& path) {
  std::ifstream f(path, std::ios::binary);
  return std::vector<uint8_t>(std::istreambuf_iterator<char>(f), std::istreambuf_iterator<char>());
}

int main() {
  std::string line;
  while (std::getline(std::cin, line)) {
    std::istringstream in(line);
    std::string kind, path;
    in >> kind >> path;
    std::vector<uint8_t> data = slurp(path);
    std::string err;
    if (kind == "zkey") {
      ZkeyLayout L;
      int rc = zkey_parse(data.data(), data.size(), &L, &err);
      for (size_t i = 0; rc == 0 && i < L.n_coefs; ++i) {
        uint32_t w[11];
        memcpy(w, L.coefs + kZkeyCoefBytes * i, sizeof w);
        const int code = zkey_coef_check(w, L.domain_size, L.n_vars);
        if (code != ZKEY_COEF_OK) rc = zkey_coef_error(code, i, &err);
      }
      if (rc) std::cout << rc << " " << err << "\n";
      else std::cout << "0 ok " << L.n_vars << " " << L.n_public << " " << L.log_n << " " << L.n_coefs << "\n";
    } else {
      uint32_t n_vars = 0;
      in >> n_vars;
      const uint8_t* values = nullptr;
      int rc = wtns_parse(data.data(), data.size(), n_vars, &values, &err);
      if (rc) std::cout << rc << " " << err << "\n";
      else std::cout << "0 ok\n";
    }
  }
  return 0;
}
