// sim_test_pass.cpp -- TrainNet::TestPass in its two halves for several in-process ranks on the stream-order model.  On hardware each
// rank is its own process and b2h_tester_test_pass runs the whole pass; here one host thread drives every rank, so every rank's pass
// (forwards, score adds, score allreduce) has to be enqueued before any rank's closing read forces the collective.  TEST
// INFRASTRUCTURE ONLY (libtestpasssim.so, Makefile.testpass; tests/test_periodic_test_sim.py).
#include <cstring>
#include <memory>
#include <string>

#include "../../caffe_mpi_b200/host/train_net.hpp"

using namespace caffe;

// the layout of b2h_capi.cpp's tester handle, whose pointer the Python Tester holds
struct TesterHandle {
  std::unique_ptr<Net> desc;
  std::unique_ptr<TrainNet> net;
};

static thread_local std::string g_perr;

extern "C" {

const char* sim_pass_last_error() { return g_perr.c_str(); }
// returns the batches enqueued (= iterations), -1 on error
int sim_tester_enqueue_pass(void* hv, int iterations) {
  try { return static_cast<TesterHandle*>(hv)->net->EnqueueTestPass(iterations, nullptr); }
  catch (const std::exception& e) { g_perr = e.what(); return -1; }
}
int sim_tester_read_pass(void* hv, float* means, float* loss) {
  try {
    vector<float> m;
    static_cast<TesterHandle*>(hv)->net->ReadTestPass(&m, loss);
    std::memcpy(means, m.data(), sizeof(float) * m.size());
    return 0;
  } catch (const std::exception& e) { g_perr = e.what(); return -1; }
}

}  // extern "C"
