// ORACLE — TEST INFRASTRUCTURE ONLY (see fo_math.h). C ABI of the closure nodes of fo_closure.h, built as a library of its own
// (oracle/_build/libfundsp_oracle_closure.so, by tests/oracle_closure.py). Its nodes are fo::Node objects like those of
// libfundsp_oracle.so, compiled from the same headers with the same flags, so the combinators there take them as children
// (they only call virtual functions of their children; the library stays loaded for the life of the process).
#include "fo_closure.h"

using namespace fo;

#define API extern "C" __attribute__((visibility("default")))

// null when the text does not parse
API Node* fo_map(int inputs, int outputs, const char* text, int ncaps, const char* const* names, const float* values) {
  cl::Closure c;
  return c.parse(text, 0, inputs, ncaps, names, values) ? new Map(inputs, outputs, c) : nullptr;
}
API Node* fo_shape_fn(const char* text, int ncaps, const char* const* names, const float* values) {
  cl::Closure c;
  return c.parse(text, 1, 1, ncaps, names, values) ? new ShapeFn(c) : nullptr;
}
API Node* fo_envelope_in(double interval, int inputs, int outputs, const char* text, int ncaps, const char* const* names, const float* values) {
  cl::Closure c;
  return c.parse(text, 2, inputs, ncaps, names, values) ? new EnvelopeIn((float)interval, inputs, outputs, c) : nullptr;
}
