// fundsp_b200 closure parser: the text of a closure of the signal (map, shape_fn, envelope_in) -> the type expression the device
// compiles (the Ex:: templates of csrc/dsp/nodes.cuh). The text is a subset of Rust closure syntax (DESIGN.md §2); user text never
// reaches NVRTC, only the type expression generated from the parsed tree.
#pragma once
#include <string>
#include <vector>

namespace fdsp {
namespace host {

enum ClosureKind { CL_MAP = 0, CL_SHAPE_FN = 1, CL_ENVELOPE_IN = 2 };
constexpr int CLOSURE_MAX_TEXT = 4096;   // bytes
constexpr int CLOSURE_MAX_OPS = 256;     // operators, calls and literals: bounds the template depth NVRTC sees

struct Closure {
  std::string expr;                 // type expression of the body, e.g. Ex::Tanh<Ex::Mul<Ex::In<0>,Ex::Cap<0>>>
  std::vector<std::string> caps;    // captured identifiers in Cap<k> order (first occurrence in the text)
};

// Parses `text` as the closure of a node of `kind` with `inputs` inputs and `outputs` outputs. Returns "" or the reason; reasons
// that are arity mismatches start with "arity mismatch".
std::string parse_closure(const char* text, ClosureKind kind, int inputs, int outputs, Closure& out);

}  // namespace host
}  // namespace fdsp
