// fundsp_b200 closure parser: the text of a closure of the signal or of time (map, shape_fn, envelope_in, envelope) -> the type expression the device
// compiles (the Ex:: templates of csrc/dsp/nodes.cuh). The text is a subset of Rust closure syntax (DESIGN.md §2); user text never
// reaches NVRTC, only the type expression generated from the parsed tree.
#pragma once
#include <cstdint>
#include <string>
#include <vector>

namespace fdsp {
namespace host {

// CL_VAR_FN: var_fn's |x| of the Shared's value; CL_ENVELOPE: envelope / lfo's |t| of time alone; CL_UPDATE: update's |t, dt, x|,
// whose body is `let`s and unconditional `x.set(Setting::..)` statements
enum ClosureKind { CL_MAP = 0, CL_SHAPE_FN = 1, CL_ENVELOPE_IN = 2, CL_VAR_FN = 3, CL_ENVELOPE = 4, CL_UPDATE = 5 };
constexpr int CLOSURE_MAX_TEXT = 4096;   // bytes
constexpr int CLOSURE_MAX_OPS = 256;     // operators, calls and literals: bounds the template depth NVRTC sees

// One `x.set(Setting::kind(args).address..)` of an update function: `kind` numbered as the C ABI's settings (include/fundsp_b200.h),
// its arguments the values [arg, arg + nargs) of the body's tuple, `address` the Index values of .left() / .right() / .index(N) in order.
struct UpdateSet { int kind, arg, nargs, col; std::vector<uint64_t> address; };

struct Closure {
  std::string expr;                 // type expression of the body, e.g. Ex::Tanh<Ex::Mul<Ex::In<0>,Ex::Cap<0>>>
  std::vector<std::string> caps;    // captured identifiers in Cap<k> order (first occurrence in the text)
  std::vector<UpdateSet> sets;      // CL_UPDATE: the statements in order; `expr` is the tuple of all their arguments (t = In<0>, dt = In<1>)
};

// Parses `text` as the closure of a node of `kind` with `inputs` inputs and `outputs` outputs. Returns "" or the reason; reasons
// that are arity mismatches start with "arity mismatch".
std::string parse_closure(const char* text, ClosureKind kind, int inputs, int outputs, Closure& out);

}  // namespace host
}  // namespace fdsp
