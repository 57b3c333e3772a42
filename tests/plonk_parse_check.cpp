// CPU program of the PLONK .zkey parser (plonk_zkey_parse in ethrex_b200/csrc/zkey_parse.cpp), run by
// tests/test_plonk_host.py.  One path per stdin line, one answer per stdout line: "<status> <message>", or
// "0 ok <nVars> <nPublic> <log_n> <nAdditions> <nConstraints>" when the key is accepted.
#include <fstream>
#include <iostream>
#include <iterator>
#include <string>
#include <vector>

#include "zkey_parse.h"

using namespace b200zk;

int main() {
  std::string path;
  while (std::getline(std::cin, path)) {
    std::ifstream f(path, std::ios::binary);
    std::vector<uint8_t> data((std::istreambuf_iterator<char>(f)), std::istreambuf_iterator<char>());
    std::string err;
    PlonkLayout L;
    const int rc = plonk_zkey_parse(data.data(), data.size(), &L, &err);
    if (rc) std::cout << rc << " " << err << "\n";
    else std::cout << "0 ok " << L.n_vars << " " << L.n_public << " " << L.log_n << " " << L.n_additions << " " << L.n_constraints << "\n";
  }
  return 0;
}
