// Host driver for tests/test_key_numbers_host.py: the decimal grammar and conversion of mrhbm_map_key_numbers
// (csrc/mrhbm_decimal.cuh), host-compiled.  With "--table" it prints the power-of-five table, one "q hi lo" line per
// entry in hex.  Otherwise it reads one token per line from stdin and prints, per token, "bad" when the grammar
// refuses it, else "<path> <device bits> <host bits>": path E when dec_to_bits gives the value itself, H19 when it
// sends the token to the host for its digits, HEL for the ambiguous Eisel-Lemire case (device bits then 0); the host
// bits are dec_parse_host's (std::from_chars).  Both in hex, "x" if dec_parse_host refuses a token the grammar took.
#include <cinttypes>
#include <cstdio>
#include <iostream>
#include <string>
#include <vector>

#include "mrhbm_decimal.cuh"

using namespace mrhbm;

int main(int argc, char** argv) {
  std::vector<uint64_t> pow5(2 * kPow5Count);
  dec_pow5_table(pow5.data());
  if (argc > 1 && std::string(argv[1]) == "--table") {
    for (int q = kPow5Min; q <= kPow5Max; q++)
      std::printf("%d %016" PRIx64 " %016" PRIx64 "\n", q, pow5[2 * (q - kPow5Min)], pow5[2 * (q - kPow5Min) + 1]);
    return 0;
  }
  std::string tok;
  while (std::getline(std::cin, tok)) {
    const unsigned char* s = (const unsigned char*)tok.data();
    DecScan d;
    if (!dec_scan(s, tok.size(), &d)) {
      std::printf("bad\n");
      continue;
    }
    uint64_t dev = 0, host = 0;
    const int r = dec_to_bits(d, pow5.data(), &dev);
    const char* path = r == DEC_EXACT ? "E" : d.nd > (uint32_t)kDecMaxDigits ? "H19" : "HEL";
    if (r != DEC_EXACT) dev = 0;
    if (dec_parse_host(s, tok.size(), &host))
      std::printf("%s %016" PRIx64 " %016" PRIx64 "\n", path, dev, host);
    else
      std::printf("%s %016" PRIx64 " x\n", path, dev);
  }
  return 0;
}
