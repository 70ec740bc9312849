// TEST INFRASTRUCTURE (oracle/_ref) -- not part of the shipped product.
//
// The graph-label entry points of the reference, over the graph and the thread-local engine of libeuler_ref.so (built by
// oracle/Makefile; this file links against it, recipe oracle/graph_label.mk):
//   ref_graph_labels          Graph::GetGraphLabel (euler/core/graph/graph.cc:439-457) on the graph ref_graph_load loaded
//   ref_sample_graph_label    the loop of SampleGraphLabelOp::Compute (euler/core/kernels/sample_graph_label_op.cc), restated:
//                             that file needs the engine's op framework and protobuf, which are not built here
#include <stdint.h>
#include <string.h>
#include <math.h>

#include <string>
#include <vector>

#include "euler/common/random.h"
#include "euler/core/graph/graph.h"

extern "C" {

// the labels' bytes concatenated into buf (when their total fits cap) and their ends in ends[n]; returns n
int64_t ref_graph_labels(int64_t cap, char* buf, int64_t* ends, int64_t ends_cap) {
  const std::vector<std::string> v = euler::Graph::Instance().GetGraphLabel();
  int64_t total = 0;
  for (size_t i = 0; i < v.size(); ++i) {
    if (buf && total + (int64_t)v[i].size() <= cap) memcpy(buf + total, v[i].data(), v[i].size());
    total += (int64_t)v[i].size();
    if (ends && (int64_t)i < ends_cap) ends[i] = total;
  }
  return (int64_t)v.size();
}

// out[i] = the label index of draw i: floor(ThreadLocalRandom() * L), as SampleGraphLabelOp draws it
void ref_sample_graph_label(int32_t count, int64_t L, int32_t* out) {
  for (int32_t i = 0; i < count; ++i) out[i] = (int32_t)floor(euler::common::ThreadLocalRandom() * L);
}

}  // extern "C"
