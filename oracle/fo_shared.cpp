// ORACLE — TEST INFRASTRUCTURE ONLY (see fo_math.h). C ABI of the Shared nodes of fo_shared.h, built as a library of its own
// (oracle/_build/libfundsp_oracle_shared.so, by tests/oracle_shared.py). Its nodes are fo::Node objects like those of libfundsp_oracle.so,
// compiled from the same headers with the same flags, so the combinators there take them as children.
#include "fo_shared.h"

using namespace fo;

#define API extern "C" __attribute__((visibility("default")))

API Cell* fo_shared_new(float value) { Cell* c = new Cell(std::make_shared<std::atomic<uint32_t>>(0u)); cell_set(*c, value); return c; }
API void fo_shared_free(Cell* c) { delete c; }
API void fo_shared_set(Cell* c, float value) { cell_set(*c, value); }
API float fo_shared_get(const Cell* c) { return cell_get(*c); }
API Node* fo_var_shared(const Cell* c) { return new VarShared(*c); }
API Node* fo_monitor_shared(const Cell* c, int kind, double timescale) { return new MonitorShared(*c, kind, timescale); }
API Node* fo_var_fn(const Cell* c, int outputs, const char* text, int ncaps, const char* const* names, const float* values) {   // null: no parse
  cl::Closure f;
  return f.parse(text, 1, 1, ncaps, names, values) ? new VarFn(*c, outputs, f) : nullptr;
}
API Node* fo_timer(const Cell* c) { return new Timer(*c); }
