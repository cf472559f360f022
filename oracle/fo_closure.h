// ORACLE — TEST INFRASTRUCTURE ONLY (see fo_math.h). Closures of the signal: an interpreter for the closure text the product
// compiles (DESIGN.md §2), written independently of csrc/host/closure.cpp — the two share the language, not the code. The text is
// parsed once into a tree (precedence climbing) that is walked per call, in f32, with the oracle's own libm restatements.
// Nodes: Map (src/audionode.rs:1328-1371, ID 5), Shaper<ShapeFn> (src/shape.rs:33-42, ID 42), EnvelopeIn<f32> (src/envelope.rs:185-358, ID 53).
#pragma once
#include "fo_nodes.h"
#include <cctype>
#include <cstring>
#include <string>

namespace fo {
namespace cl {

struct Expr {
  std::string op;            // "lit" "t" "in" "cap" "var" "neg" "not" "+" "-" "*" "/" "<" "<=" ">" ">=" "==" "!=" "&&" "||" "if" "let" "tuple" or a function name
  float lit = 0.0f; int idx = 0; bool method = false;
  std::vector<std::shared_ptr<Expr>> a;
};
typedef std::shared_ptr<Expr> E;

struct Ctx { const float* in; const float* caps; float t; std::vector<float> slots; };

inline float num(const std::string& s) {   // a Rust f32 literal: underscores and the f32 suffix dropped, rounded once to f32
  std::string d;
  for (char c : s) if (c != '_') d += c;
  if (d.size() > 3 && d.substr(d.size() - 3) == "f32") d.resize(d.size() - 3);
  return strtof(d.c_str(), nullptr);
}

struct Reader {
  std::string s; size_t i = 0; bool bad = false;
  std::vector<std::string> params;      // names; kinds below
  std::vector<int> pkind;               // 0 time, 1 frame, 2 scalar input pidx, 3 frame or scalar
  std::vector<int> pidx;
  std::vector<std::pair<std::string, int>> scope;   // let name -> slot
  int nslots = 0;
  std::vector<std::string> capnames;

  void ws() {
    for (;;) {
      while (i < s.size() && isspace((unsigned char)s[i])) i++;
      if (s.compare(i, 2, "//") == 0) { while (i < s.size() && s[i] != '\n') i++; continue; }
      if (s.compare(i, 2, "/*") == 0) { size_t e = s.find("*/", i + 2); i = e == std::string::npos ? s.size() : e + 2; continue; }
      return;
    }
  }
  bool peek(const char* t) { ws(); return s.compare(i, strlen(t), t) == 0; }
  bool eat(const char* t) { if (peek(t)) { i += strlen(t); return true; } return false; }
  void need(const char* t) { if (!eat(t)) bad = true; }
  std::string word() {
    ws(); size_t j = i;
    while (j < s.size() && (isalnum((unsigned char)s[j]) || s[j] == '_')) j++;
    std::string w = s.substr(i, j - i); i = j; return w;
  }
  static E node(const std::string& op, std::vector<E> a = {}) { E e = std::make_shared<Expr>(); e->op = op; e->a = std::move(a); return e; }

  void skip_type() { int depth = 0; while (i < s.size()) { char c = s[i]; if (depth == 0 && (c == ',' || c == '|' || c == '=')) return; if (c == '<' || c == '(') depth++; if (c == '>' || c == ')') depth--; i++; } }

  // binary operators by Rust precedence (higher binds tighter)
  static int prec(const std::string& o) {
    if (o == "||") return 1;
    if (o == "&&") return 2;
    if (o == "<" || o == "<=" || o == ">" || o == ">=" || o == "==" || o == "!=") return 3;
    if (o == "+" || o == "-") return 4;
    if (o == "*" || o == "/") return 5;
    return 0;
  }
  std::string binop() {
    ws();
    static const char* ops[] = {"||", "&&", "<=", ">=", "==", "!=", "<", ">", "+", "-", "*", "/"};
    for (const char* o : ops) if (s.compare(i, strlen(o), o) == 0) return o;
    return "";
  }
  E expr(int minp = 1) {
    E l = unary();
    for (;;) {
      std::string o = binop();
      int p = o.empty() ? 0 : prec(o);
      if (p < minp || bad) return l;
      i += o.size();
      E r = expr(p + 1);   // left-associative
      l = node(o, {l, r});
    }
  }
  E unary() {
    if (eat("-")) return node("neg", {unary()});
    if (peek("!") && !peek("!=")) { i++; return node("not", {unary()}); }
    return postfix(primary());
  }
  E postfix(E x) {
    for (;;) {
      ws();
      if (i < s.size() && s[i] == '.' && !(i + 1 < s.size() && isdigit((unsigned char)s[i + 1]))) {
        i++;
        std::string m = word();
        need("(");
        std::vector<E> args{x};
        if (!eat(")")) { do { args.push_back(expr()); } while (eat(",")); need(")"); }
        E c = node(m, args); c->method = true; x = c;
      } else return x;
    }
  }
  E primary() {
    ws();
    if (bad || i >= s.size()) { bad = true; return node("lit"); }
    if (isdigit((unsigned char)s[i])) {
      size_t j = i;
      while (j < s.size() && (isalnum((unsigned char)s[j]) || s[j] == '_' || (s[j] == '.' && !(j + 1 < s.size() && isalpha((unsigned char)s[j + 1]))) ||
                              ((s[j] == '-' || s[j] == '+') && (s[j - 1] == 'e' || s[j - 1] == 'E')))) j++;
      E e = node("lit"); e->lit = num(s.substr(i, j - i)); i = j; return e;
    }
    if (eat("(")) {
      std::vector<E> el{expr()};
      bool tuple = false;
      while (eat(",")) { tuple = true; if (peek(")")) break; el.push_back(expr()); }
      need(")");
      return tuple ? node("tuple", el) : el[0];
    }
    if (peek("{")) return block();
    std::string w = word();
    if (w.empty()) { bad = true; return node("lit"); }
    if (w == "if") {
      E c = expr(); E a = block(); E b;
      ws();
      if (word() != "else") { bad = true; return a; }
      ws();
      if (peek("if")) { i += 2; b = ifrest(); } else b = block();
      return node("if", {c, a, b});
    }
    if (eat("(")) {
      std::vector<E> args;
      if (!eat(")")) { do { args.push_back(expr()); } while (eat(",")); need(")"); }
      return node(w, args);
    }
    for (size_t k = scope.size(); k-- > 0;) if (scope[k].first == w) { E e = node("var"); e->idx = scope[k].second; return e; }
    for (size_t k = 0; k < params.size(); k++) {
      if (params[k] != w) continue;
      if (pkind[k] == 0) return node("t");
      if (eat("[")) { ws(); size_t j = i; while (j < s.size() && isdigit((unsigned char)s[j])) j++; E e = node("in"); e->idx = atoi(s.substr(i, j - i).c_str()); i = j; need("]"); return e; }
      E e = node("in"); e->idx = pkind[k] == 2 ? pidx[k] : 0; return e;
    }
    for (size_t k = 0; k < capnames.size(); k++) if (capnames[k] == w) { E e = node("cap"); e->idx = (int)k; return e; }
    bad = true; return node("lit");
  }
  E ifrest() {   // after `else if`
    E c = expr(); E a = block(); E b;
    ws();
    if (word() != "else") { bad = true; return a; }
    ws();
    if (peek("if")) { i += 2; b = ifrest(); } else b = block();
    return node("if", {c, a, b});
  }
  E block() {
    need("{");
    size_t depth = scope.size();
    std::vector<std::pair<int, E>> lets;
    for (;;) {
      ws();
      size_t save = i;
      if (word() != "let") { i = save; break; }
      std::string n = word();
      if (eat(":")) skip_type();
      need("=");
      E v = expr();
      need(";");
      int slot = nslots++;
      lets.push_back({slot, v});
      scope.push_back({n, slot});
    }
    E body = expr();
    need("}");
    scope.resize(depth);
    for (size_t k = lets.size(); k-- > 0;) { E l = node("let", {lets[k].second, body}); l->idx = lets[k].first; body = l; }
    return body;
  }
};

// value of a subtree; bools travel as 0 / 1
inline float ev(const Expr& e, Ctx& c);
inline float fn(const Expr& e, Ctx& c) {
  float x[5] = {0, 0, 0, 0, 0};
  for (size_t k = 0; k < e.a.size() && k < 5; k++) x[k] = ev(*e.a[k], c);
  const std::string& f = e.op;
  if (f == "abs") return fabsf(x[0]);
  if (f == "min") return fminf(x[0], x[1]);   // f32::min: a NaN operand is ignored
  if (f == "max") return fmaxf(x[0], x[1]);
  if (f == "clamp" && e.method) { float v = x[0]; if (v < x[1]) v = x[1]; if (v > x[2]) v = x[2]; return v; }   // std f32::clamp
  if (f == "clamp") return fminf(fmaxf(x[2], x[0]), x[1]);                                                      // fundsp clamp(x0, x1, x)
  if (f == "clamp01") return clamp01f(x[0]);
  if (f == "clamp11") return clamp11f(x[0]);
  if (f == "floor") return floorf(x[0]);
  if (f == "ceil") return ceilf(x[0]);
  if (f == "round") return roundf(x[0]);
  if (f == "sqrt") return sqrtf(x[0]);
  if (f == "signum") { if (e.method && std::isnan(x[0])) { float q; uint32_t u = 0x7fc00000u; memcpy(&q, &u, 4); return q; } return copysignf(1.0f, x[0]); }
  if (f == "lerp") return lerpf(x[0], x[1], x[2]);
  if (f == "lerp11") return lerpf(x[0], x[1], x[2] * 0.5f + 0.5f);
  if (f == "delerp") return delerpf(x[0], x[1], x[2]);
  if (f == "delerp11") return (x[2] - x[0]) / (x[1] - x[0]) * 2.0f - 1.0f;
  if (f == "softsign") return x[0] / (1.0f + fabsf(x[0]));
  if (f == "softexp") { float p = fmaxf(x[0], 0.0f); return p * p + p + 1.0f / (1.0f + p - x[0]); }
  if (f == "smooth3") return (3.0f - 2.0f * x[0]) * x[0] * x[0];
  if (f == "smooth5") return ((x[0] * 6.0f - 15.0f) * x[0] + 10.0f) * x[0] * x[0] * x[0];
  if (f == "smooth7") { float x2 = x[0] * x[0]; return x2 * x2 * (35.0f - 84.0f * x[0] + (70.0f - 20.0f * x[0]) * x2); }
  if (f == "smooth9") return smooth9f(x[0]);
  if (f == "spline") { float y0 = x[0], y1 = x[1], y2 = x[2], y3 = x[3], t = x[4];
    return y1 + t * 0.5f * (y2 - y0 + t * (2.0f * y0 - 5.0f * y1 + 4.0f * y2 - y3 + t * (3.0f * (y1 - y2) + y3 - y0))); }
  if (f == "sqr_hz") { float v = x[1] * x[0]; v = v - floorf(v); return v < 0.5f ? 1.0f : -1.0f; }
  if (f == "tri_hz") { float v = x[1] * x[0] - 0.25f; v = v - floorf(v); return fabsf(v - 0.5f) * 4.0f - 1.0f; }
  if (f == "bpm_hz") return x[0] * (1.0f / 60.0f);
  if (f == "squared") return x[0] * x[0];
  if (f == "sin") return m::sinf_(x[0]);
  if (f == "cos") return m::cosf_(x[0]);
  if (f == "tan") return m::tanf_(x[0]);
  if (f == "tanh") return m::tanhf_(x[0]);
  if (f == "exp") return m::expf_(x[0]);
  if (f == "pow" || f == "powf") return m::powf_(x[0], x[1]);
  const float ln10 = (float)2.302585092994045684, tau = (float)6.283185307179586477;
  if (f == "exp10") return m::expf_(x[0] * ln10);
  if (f == "db_amp") return m::expf_(x[0] / 20.0f * ln10);
  if (f == "sin_hz") return m::sinf_(x[1] * x[0] * tau);
  if (f == "cos_hz") return m::cosf_(x[1] * x[0] * tau);
  assert(false && "closure function");
  return 0.0f;
}
inline float ev(const Expr& e, Ctx& c) {
  const std::string& o = e.op;
  if (o == "lit") return e.lit;
  if (o == "t") return c.t;
  if (o == "in") return c.in[e.idx];
  if (o == "cap") return c.caps[e.idx];
  if (o == "var") return c.slots[e.idx];
  if (o == "neg") return -ev(*e.a[0], c);
  if (o == "not") return ev(*e.a[0], c) != 0.0f ? 0.0f : 1.0f;
  if (o == "if") return ev(*e.a[0], c) != 0.0f ? ev(*e.a[1], c) : ev(*e.a[2], c);
  if (o == "let") { c.slots[e.idx] = ev(*e.a[0], c); return ev(*e.a[1], c); }
  if (e.a.size() == 2 && Reader::prec(o)) {
    const float a = ev(*e.a[0], c), b = ev(*e.a[1], c);
    switch (o[0]) {
      case '+': return a + b;
      case '-': return a - b;
      case '*': return a * b;
      case '/': return a / b;
      case '<': return o.size() == 1 ? a < b : a <= b;
      case '>': return o.size() == 1 ? a > b : a >= b;
      case '=': return a == b;
      case '!': return a != b;
      case '&': return (a != 0.0f) && (b != 0.0f);
      default: return (a != 0.0f) || (b != 0.0f);
    }
  }
  return fn(e, c);
}
// the closure's frame value: a tuple (possibly under `let` / `if`) or one f32
inline void frame(const Expr& e, Ctx& c, float* out) {
  if (e.op == "tuple") { for (size_t k = 0; k < e.a.size(); k++) out[k] = ev(*e.a[k], c); return; }
  if (e.op == "let") { c.slots[e.idx] = ev(*e.a[0], c); frame(*e.a[1], c, out); return; }
  if (e.op == "if") { if (ev(*e.a[0], c) != 0.0f) frame(*e.a[1], c, out); else frame(*e.a[2], c, out); return; }
  out[0] = ev(e, c);
}

// kind 0 map |x|, 1 shape_fn |x|, 2 envelope_in |t, i| or |t, x1, .., xN|
struct Closure {
  E body; int nslots = 0; std::vector<float> caps;
  bool parse(const char* text, int kind, int inputs, int ncaps, const char* const* names, const float* values) {
    Reader r; r.s = text;
    for (int k = 0; k < ncaps; k++) { r.capnames.push_back(names[k]); caps.push_back(values[k]); }
    r.ws();
    if (r.s.compare(r.i, 4, "move") == 0) r.i += 4;
    std::vector<std::string> ps;
    if (!r.eat("||")) {
      r.need("|");
      while (!r.bad && !r.eat("|")) { ps.push_back(r.word()); if (r.eat(":")) r.skip_type(); r.eat(","); if (ps.back().empty()) return false; }
    }
    const int np = (int)ps.size();
    for (int k = 0; k < np; k++) {
      int kd, ix = 0;
      if (kind == 0) kd = 1;
      else if (kind == 1) kd = 2;
      else if (k == 0) kd = 0;
      else if (np == 2 && inputs == 1) kd = 3;
      else if (np == 2) kd = 1;
      else { kd = 2; ix = k - 1; }
      r.params.push_back(ps[k]); r.pkind.push_back(kd); r.pidx.push_back(ix);
    }
    body = r.expr();
    r.ws();
    nslots = r.nslots;
    return !r.bad && r.i == r.s.size();
  }
  void call(const float* in, float t, float* out) const {
    Ctx c{in, caps.data(), t, std::vector<float>((size_t)nslots + 1, 0.0f)};
    frame(*body, c, out);
  }
};

}  // namespace cl

// ---- src/audionode.rs:1328-1371 Map (ID 5): no process override, the default tick loop
struct Map : Node {
  int ni, no; cl::Closure f;
  Map(int i, int o, cl::Closure c) : ni(i), no(o), f(std::move(c)) {}
  int inputs() const override { return ni; } int outputs() const override { return no; }
  uint64_t id() const override { return 5; }
  void tick(const float* in, float* out) override { f.call(in, 0.0f, out); }
  FO_CLONE(Map)
};
// ---- src/shape.rs:33-42 Shaper<ShapeFn<S>> (ID 42): ShapeFn::simd is the default per-lane `shape`, so the block path is the tick loop
struct ShapeFn : Node {
  cl::Closure f;
  explicit ShapeFn(cl::Closure c) : f(std::move(c)) {}
  int inputs() const override { return 1; } int outputs() const override { return 1; }
  uint64_t id() const override { return 42; }
  void tick(const float* in, float* out) override { f.call(in, 0.0f, out); }
  FO_CLONE(ShapeFn)
};
// ---- src/envelope.rs:185-358 EnvelopeIn<f32, E, I, R> (ID 53)
struct EnvelopeIn : Node {
  int ni, no; cl::Closure f;
  float t = 0, t_0 = 0, t_1 = 0; uint64_t t_hash = 0;
  std::vector<float> value_0, value_1, value, value_d;
  float interval, sample_duration = 0; uint64_t hash = 0;
  EnvelopeIn(float iv, int i, int o, cl::Closure c) : ni(i), no(o), f(std::move(c)), value_0(o), value_1(o), value(o), value_d(o), interval(iv) {
    set_sample_rate(DEFAULT_SR); reset();
  }
  void next_segment(const float* input) {   // :251-278
    if (t_0 == 0.0f && t_1 == 0.0f) f.call(input, t_0, value_0.data());
    else { t_0 = t_1; value_0 = value_1; }
    const float next_interval = lerpf(0.75f, 1.25f, (float)rnd1(t_hash)) * interval;
    t_1 = t_0 + next_interval;
    f.call(input, t_1, value_1.data());
    t_hash = t_hash * 6364136223846793005ull + 1ull;
    const float u = delerpf(t_0, t_1, t);
    for (int k = 0; k < no; k++) value[k] = lerpf(value_0[k], value_1[k], u);
    const float samples = next_interval / sample_duration;
    for (int k = 0; k < no; k++) value_d[k] = (value_1[k] - value_0[k]) / samples;
  }
  int inputs() const override { return ni; } int outputs() const override { return no; }
  uint64_t id() const override { return 53; }
  void reset() override { t = 0; t_0 = 0; t_1 = 0; t_hash = hash; }
  void set_sample_rate(double sr) override { sample_duration = (float)(1.0 / sr); }
  void tick(const float* in, float* out) override {   // :305-313
    if (t >= t_1) next_segment(in);
    for (int k = 0; k < no; k++) { out[k] = value[k]; value[k] += value_d[k]; }
    t += sample_duration;
  }
  void process(int size, const float* in, float* out) override {   // :315-342
    if (size == 0) return;
    float fr[8] = {0, 0, 0, 0, 0, 0, 0, 0};
    auto at = [&](int j) { for (int c = 0; c < ni; c++) fr[c] = in[c * B + j]; return fr; };
    if (t >= t_1) next_segment(at(0));
    int i = 0;
    while (i < size) {
      const size_t left = (size_t)(int64_t)ceilf((t_1 - t) / sample_duration);
      const size_t loop = std::min<size_t>((size_t)(size - i), left);
      for (int c = 0; c < no; c++) {
        float v = value[c];
        for (size_t o = 0; o < loop; o++) { out[c * B + i + o] = v; v += value_d[c]; }
        value[c] = v;
      }
      i += (int)loop;
      t += (float)(int64_t)loop * sample_duration;
      if (loop == left && i < size) next_segment(at(i));
    }
  }
  void set(const Setting& s) override { if (s.kind == P_INTERVAL) interval = s.v[0]; }
  void set_hash(uint64_t h) override { hash = h; t_hash = h; }
  FO_CLONE(EnvelopeIn)
};

}  // namespace fo
