// rir_ref -- runs the reference's own RirGenerator (compiled in by path, see build.sh) and writes
// the float32 response to stdout: int32 rows, int32 cols, then rows x cols float32.
// Arguments are rir-simulate's options as --name=value.  TEST INFRASTRUCTURE ONLY.
#include <cstdio>
#include <cstring>
#include <map>
#include <string>

#include RIR_GENERATOR_CC

int main(int argc, char** argv) {
  using namespace kaldi;
  try {
    RirGeneratorOptions o;
    for (int i = 1; i < argc; ++i) {
      std::string a(argv[i]);
      const size_t eq = a.find('=');
      if (a.compare(0, 2, "--") != 0 || eq == std::string::npos) throw std::runtime_error("bad argument " + a);
      const std::string k = a.substr(2, eq - 2), v = a.substr(eq + 1);
      if (k == "sound-velocity") o.sound_velocity = std::stof(v);
      else if (k == "samp-frequency") o.samp_frequency = std::stof(v);
      else if (k == "hp-filter") o.hp_filter = v == "true";
      else if (k == "number-samples") o.num_samples = std::stoi(v);
      else if (k == "order") o.order = std::stoi(v);
      else if (k == "microphone-type") o.microphone_type = v;
      else if (k == "receiver-location") o.receiver_location = v;
      else if (k == "source-location") o.source_location = v;
      else if (k == "room-topo") o.room_topo = v;
      else if (k == "angle") o.orientation = v;
      else if (k == "beta") o.beta = v;
      else throw std::runtime_error("unknown option " + k);
    }
    RirGenerator gen(o);
    Matrix<BaseFloat> rir;
    gen.GenerateRir(&rir);
    const int32_t dims[2] = {rir.rows, rir.cols};
    fwrite(dims, sizeof(int32_t), 2, stdout);
    fwrite(rir.data.data(), sizeof(float), rir.data.size(), stdout);
  } catch (const std::exception& e) {
    fprintf(stderr, "%s\n", e.what());
    return 1;
  }
  return 0;
}
