// The C++ host mirror's SqrtInformation (voxgraph_b200/host/voxgraph_b200.hpp) on information matrices read from
// stdin, one per line: allow_semi_definite (0 or 1), then the 16 row-major entries (any strtod form, hex floats
// included).  Prints one line per matrix: "ok" and the 16 entries of the factor as the hex of their IEEE-754 bits,
// or "invalid_argument" and the exception's message.  No GPU needed.
#include <cinttypes>
#include <cstdio>
#include <cstring>
#include <iostream>
#include <sstream>
#include <string>

#include "voxgraph_b200.hpp"

using namespace voxgraph_b200;

int main() {
  std::string line;
  while (std::getline(std::cin, line)) {
    std::istringstream in(line);
    int semi = 0;
    std::string v;
    InformationMatrix info{};
    in >> semi;
    for (double& x : info) {
      in >> v;
      x = std::strtod(v.c_str(), nullptr);
    }
    try {
      const std::array<double, 16> S = SqrtInformation(info, semi != 0);
      std::printf("ok");
      for (double x : S) {
        uint64_t bits;
        std::memcpy(&bits, &x, sizeof bits);
        std::printf(" %016" PRIx64, bits);
      }
      std::printf("\n");
    } catch (const std::invalid_argument& e) {
      std::printf("invalid_argument %s\n", e.what());
    }
  }
  return 0;
}
