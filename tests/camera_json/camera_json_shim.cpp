// The camera JSON writer and the printed summary of the command line tools (icc_cli_common.hpp) on their own, for
// tests/test_camera_json.py:
//   camera_json_shim write <model name> k0 k1 ..  the `intrinsics` object write_intrinsics makes of k
//   camera_json_shim print <model name> k0 k1 ..  the lines print_camera prints for k
// Errors go to stderr with exit code 1.
#include "../../openimucameracalibrator_b200/csrc/icc_cli_common.hpp"

#include <iostream>

int main(int argc, char** argv) {
  try {
    if (argc < 3) throw std::runtime_error("usage: camera_json_shim write|print <model name> k0 k1 ..");
    const std::string cmd = argv[1];
    const icccli::CameraLayout* c = icccli::find_camera(argv[2]);
    if (!c) throw std::runtime_error(std::string("unknown model ") + argv[2]);
    std::vector<double> k;
    for (int i = 3; i < argc; ++i) k.push_back(std::stod(argv[i]));
    if ((int)k.size() != c->num_params) throw std::runtime_error("expected " + std::to_string(c->num_params) + " intrinsics");
    if (cmd == "write") std::cout << iccjson::dump(icccli::write_intrinsics(*c, k.data())) << std::endl;
    else if (cmd == "print") icccli::print_camera(std::cout, *c, k.data());
    else throw std::runtime_error("unknown command " + cmd);
  } catch (const std::exception& e) {
    std::cerr << e.what() << std::endl;
    return 1;
  }
  return 0;
}
