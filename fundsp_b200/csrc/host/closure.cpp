// fundsp_b200 closure parser — see closure.h. A recursive-descent parser for the subset of Rust closure syntax that DESIGN.md §2
// lists, with Rust's precedence and associativity; it type-checks as it goes (f32, bool, tuple) and emits the Ex:: type expression.
// Every refusal names the offending token and its column (1-based byte offset into the text).
//
// This file is compiled as part of graph.cpp's translation unit (see the end of graph.cpp), so every build of the host graph has it.
#include "closure.h"

#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <map>

namespace fdsp {
namespace host {
namespace {

enum TokKind { T_END, T_ID, T_NUM, T_INT, T_PUNCT };
struct Tok { TokKind k; std::string s; int col; };

struct ParseError { std::string why; };
[[noreturn]] void fail_at(const Tok& t, const std::string& what) {
  std::string tok = t.k == T_END ? "end of text" : "`" + t.s + "`";
  throw ParseError{what.empty() ? "unexpected " + tok + " at column " + std::to_string(t.col)
                                : tok + " at column " + std::to_string(t.col) + ": " + what};
}

bool id_start(char c) { return (c >= 'a' && c <= 'z') || (c >= 'A' && c <= 'Z') || c == '_'; }
bool id_char(char c) { return id_start(c) || (c >= '0' && c <= '9'); }
bool digit(char c) { return c >= '0' && c <= '9'; }

std::vector<Tok> lex(const std::string& src) {
  std::vector<Tok> out;
  size_t i = 0;
  const size_t n = src.size();
  static const char* two[] = {"||", "&&", "==", "!=", "<=", ">=", "+=", "-=", "*=", "/=", "%=", "->", "..", "::"};
  while (i < n) {
    const char c = src[i];
    if (c == ' ' || c == '\t' || c == '\n' || c == '\r') { i++; continue; }
    if (c == '/' && i + 1 < n && src[i + 1] == '/') { while (i < n && src[i] != '\n') i++; continue; }
    if (c == '/' && i + 1 < n && src[i + 1] == '*') {
      const size_t e = src.find("*/", i + 2);
      if (e == std::string::npos) fail_at(Tok{T_PUNCT, "/*", (int)i + 1}, "unterminated comment");
      i = e + 2; continue;
    }
    const int col = (int)i + 1;
    if (id_start(c)) {
      size_t j = i; while (j < n && id_char(src[j])) j++;
      out.push_back({T_ID, src.substr(i, j - i), col}); i = j; continue;
    }
    if (digit(c)) {
      size_t j = i; bool flt = false;
      while (j < n && (digit(src[j]) || src[j] == '_')) j++;
      if (j < n && src[j] == '.' && !(j + 1 < n && (src[j + 1] == '.' || id_start(src[j + 1])))) {
        flt = true; j++;
        while (j < n && (digit(src[j]) || src[j] == '_')) j++;
      }
      if (j < n && (src[j] == 'e' || src[j] == 'E')) {
        size_t k = j + 1;
        if (k < n && (src[k] == '+' || src[k] == '-')) k++;
        if (k < n && digit(src[k])) { flt = true; j = k; while (j < n && (digit(src[j]) || src[j] == '_')) j++; }
      }
      std::string suffix;
      if (j < n && id_start(src[j])) { size_t k = j; while (k < n && id_char(src[k])) k++; suffix = src.substr(j, k - j); j = k; }
      const Tok t{T_NUM, src.substr(i, j - i), col};
      if (suffix == "f32") flt = true;
      else if (!suffix.empty()) fail_at(t, "only f32 literals are accepted (the closure computes in f32)");
      out.push_back({flt ? T_NUM : T_INT, t.s, col}); i = j; continue;
    }
    bool done = false;
    for (const char* p : two) if (src.compare(i, 2, p) == 0) { out.push_back({T_PUNCT, p, col}); i += 2; done = true; break; }
    if (done) continue;
    if (strchr("|,:&<>()[]{};=+-*/!.%^?#@$'\"\\~`", c)) { out.push_back({T_PUNCT, std::string(1, c), col}); i++; continue; }
    fail_at(Tok{T_PUNCT, std::string(1, c), col}, "character not allowed in a closure");
  }
  out.push_back({T_END, "", (int)n + 1});
  return out;
}

enum Ty { F32 = 0, BOOL = 1, TUPLE = 2 };
struct V { std::string s; Ty ty; int n; };   // n: tuple arity

struct Fn { const char* name; const char* tmpl; int nargs; };
const Fn FREE_FNS[] = {
  {"abs", "Abs", 1}, {"min", "Min", 2}, {"max", "Max", 2}, {"clamp", "Clamp", 3}, {"clamp01", "Clamp01", 1}, {"clamp11", "Clamp11", 1},
  {"floor", "Floor", 1}, {"ceil", "Ceil", 1}, {"round", "Round", 1}, {"sqrt", "Sqrt", 1}, {"signum", "Signum", 1},
  {"lerp", "Lerp", 3}, {"lerp11", "Lerp11", 3}, {"delerp", "Delerp", 3}, {"delerp11", "Delerp11", 3}, {"softsign", "Softsign", 1},
  {"softexp", "Softexp", 1}, {"smooth3", "Smooth3", 1}, {"smooth5", "Smooth5", 1}, {"smooth7", "Smooth7", 1}, {"smooth9", "Smooth9", 1},
  {"spline", "Spline", 5}, {"sqr_hz", "SqrHz", 2}, {"tri_hz", "TriHz", 2}, {"bpm_hz", "BpmHz", 1}, {"squared", "Squared", 1},
  {"sin", "Sin", 1}, {"cos", "Cos", 1}, {"tan", "Tan", 1}, {"tanh", "Tanh", 1}, {"exp", "Exp", 1}, {"pow", "Pow", 2},
  {"exp10", "Exp10", 1}, {"db_amp", "DbAmp", 1}, {"sin_hz", "SinHz", 2}, {"cos_hz", "CosHz", 2},
};
// methods: the receiver is the first argument
const Fn METHODS[] = {
  {"abs", "Abs", 1}, {"min", "Min", 2}, {"max", "Max", 2}, {"clamp", "ClampM", 3}, {"floor", "Floor", 1}, {"ceil", "Ceil", 1},
  {"round", "Round", 1}, {"sqrt", "Sqrt", 1}, {"signum", "SignumM", 1}, {"sin", "Sin", 1}, {"cos", "Cos", 1}, {"tan", "Tan", 1},
  {"tanh", "Tanh", 1}, {"exp", "Exp", 1}, {"powf", "Pow", 2},
};
const char* NOT_RESTATED[] = {"log", "log2", "log10", "exp2", "atan", "xerp", "xerp11", "dexerp", "dexerp11", "amp_db", "midi_hz",
                              "semitone_ratio", "ln", "exp_m1", "ln_1p", "atan2"};
const char* KEYWORDS[] = {"as", "for", "while", "loop", "return", "mut", "match", "fn", "break", "continue", "in", "true", "false",
                          "self", "struct", "impl", "unsafe", "ref", "static", "const", "else", "let", "if", "move"};

enum PKind { PK_TIME, PK_FRAME, PK_SCALAR, PK_FRAME_OR_SCALAR, PK_NODE };   // PK_NODE: update's node parameter, the receiver of `.set(..)`

// the settings an update function may make (src/setting.rs:130-170), numbered as the C ABI's (include/fundsp_b200.h)
struct SettingKind { const char* name; int kind, nargs; };
const SettingKind UPDATE_SETTINGS[] = {{"center", 1, 1}, {"center_q", 2, 2}, {"center_q_gain", 3, 3}, {"value", 4, 1}, {"biquad", 6, 5}, {"pan", 11, 1}};
constexpr int MAX_ADDRESS = 6;   // Setting's ArrayVec<[Address; 6]>
struct Param { std::string name; PKind kind; int index; };

struct Parser {
  std::vector<Tok> t; size_t p = 0;
  int inputs, outputs, ops = 0;
  std::vector<Param> params;
  std::vector<std::pair<std::string, Ty>> lets;   // innermost last
  std::vector<std::string> caps;

  const Tok& cur() const { return t[p]; }
  bool is(const char* s) const { return t[p].k == T_PUNCT && t[p].s == s; }
  bool is_id(const char* s) const { return t[p].k == T_ID && t[p].s == s; }
  void expect(const char* s) { if (!is(s)) fail_at(cur(), std::string("expected `") + s + "`"); p++; }
  void op() { if (++ops > CLOSURE_MAX_OPS) fail_at(cur(), "the closure has more than " + std::to_string(CLOSURE_MAX_OPS) + " operations"); }

  static V f32v(const V& v, const Tok& at) {
    if (v.ty == BOOL) fail_at(at, "a bool where an f32 is expected");
    if (v.ty == TUPLE) fail_at(at, "a tuple can only be the closure's value");
    return v;
  }
  static V boolv(const V& v, const Tok& at) {
    if (v.ty != BOOL) fail_at(at, v.ty == TUPLE ? "a tuple can only be the closure's value" : "an f32 where a bool is expected");
    return v;
  }
  static V mk(const char* tmpl, std::initializer_list<std::string> args, Ty ty = F32) {
    std::string s = std::string("Ex::") + tmpl + "<";
    bool first = true;
    for (const std::string& a : args) { if (!first) s += ","; s += a; first = false; }
    return V{s + ">", ty, 0};
  }

  void refuse_keyword(const Tok& k) {
    const std::string& s = k.s;
    if (s == "as") fail_at(k, "`as` casts are not supported (the closure computes in f32)");
    if (s == "for" || s == "while" || s == "loop" || s == "break" || s == "continue") fail_at(k, "loops are not supported");
    if (s == "mut") fail_at(k, "mutation is not supported");
    if (s == "true" || s == "false") fail_at(k, "bool literals are not supported; write a comparison");
    fail_at(k, "not supported in a closure");
  }
  static bool in_list(const char* const* l, size_t n, const std::string& s) { for (size_t i = 0; i < n; i++) if (s == l[i]) return true; return false; }
  static bool keyword(const std::string& s) { return in_list(KEYWORDS, sizeof(KEYWORDS) / sizeof(*KEYWORDS), s); }

  // ---- grammar (Rust precedence, low to high): || , && , comparisons (non-associative), + - , * / , unary - ! , postfix . [] , primary
  V expr() { return or_(); }
  V or_() {
    V a = and_();
    while (is("||")) { const Tok o = cur(); p++; op(); V b = and_(); a = mk("Or", {boolv(a, o).s, boolv(b, o).s}, BOOL); }
    return a;
  }
  V and_() {
    V a = cmp();
    while (is("&&")) { const Tok o = cur(); p++; op(); V b = cmp(); a = mk("And", {boolv(a, o).s, boolv(b, o).s}, BOOL); }
    return a;
  }
  V cmp() {
    V a = add();
    static const std::pair<const char*, const char*> CMP[] = {{"<", "Lt"}, {"<=", "Le"}, {">", "Gt"}, {">=", "Ge"}, {"==", "Eq"}, {"!=", "Ne"}};
    for (auto& c : CMP) {
      if (!is(c.first)) continue;
      const Tok o = cur(); p++; op();
      V b = add();
      for (auto& d : CMP) if (is(d.first)) fail_at(cur(), "comparison operators cannot be chained");
      return mk(c.second, {f32v(a, o).s, f32v(b, o).s}, BOOL);
    }
    return a;
  }
  V add() {
    V a = mul();
    for (;;) {
      if (is("+") || is("-")) { const Tok o = cur(); p++; op(); V b = mul(); a = mk(o.s == "+" ? "Add" : "Sub", {f32v(a, o).s, f32v(b, o).s}); }
      else if (is("+=") || is("-=") || is("*=") || is("/=") || is("%=") || is("=")) fail_at(cur(), "assignment is not supported");
      else if (is("%")) fail_at(cur(), "operator not supported");
      else return a;
    }
  }
  V mul() {
    V a = unary();
    while (is("*") || is("/")) { const Tok o = cur(); p++; op(); V b = unary(); a = mk(o.s == "*" ? "Mul" : "Div", {f32v(a, o).s, f32v(b, o).s}); }
    if (is("%")) fail_at(cur(), "operator not supported");
    return a;
  }
  V unary() {
    if (is("-")) { const Tok o = cur(); p++; op(); V a = unary(); return mk("Neg", {f32v(a, o).s}); }
    if (is("!")) { const Tok o = cur(); p++; op(); V a = unary(); return mk("Not", {boolv(a, o).s}, BOOL); }
    return postfix();
  }
  std::vector<V> args() {   // after `(`
    std::vector<V> a;
    if (is(")")) { p++; return a; }
    for (;;) {
      const Tok at = cur();
      a.push_back(f32v(expr(), at));
      if (is(",")) { p++; if (is(")")) { p++; return a; } continue; }
      expect(")"); return a;
    }
  }
  V call(const Tok& name, const Fn& f, std::vector<V> a) {
    if ((int)a.size() != f.nargs)
      fail_at(name, "takes " + std::to_string(f.nargs) + " argument" + (f.nargs == 1 ? "" : "s") + ", given " + std::to_string(a.size()));
    op();
    std::string s = std::string("Ex::") + f.tmpl + "<";
    for (size_t i = 0; i < a.size(); i++) s += (i ? "," : "") + a[i].s;
    return V{s + ">", F32, 0};
  }
  V postfix() {
    V a = primary();
    for (;;) {
      if (is(".")) {
        p++;
        const Tok m = cur();
        if (m.k != T_ID) fail_at(m, "expected a method name");
        p++;
        if (!is("(")) fail_at(m, "fields are not supported");
        if (in_list(NOT_RESTATED, sizeof(NOT_RESTATED) / sizeof(*NOT_RESTATED), m.s))
          fail_at(m, "its musl source is not restated on the device yet (DESIGN.md §2)");
        const Fn* f = nullptr;
        for (const Fn& x : METHODS) if (m.s == x.name) f = &x;
        if (!f) fail_at(m, "method not supported");
        p++;
        std::vector<V> av = args();
        av.insert(av.begin(), f32v(a, m));
        a = call(m, *f, av);
      } else if (is("[")) {
        fail_at(cur(), "only a frame parameter can be indexed");
      } else if (is_id("as")) {
        refuse_keyword(cur());
      } else return a;
    }
  }
  const Param* param(const std::string& s) const { for (const Param& x : params) if (x.name == s) return &x; return nullptr; }
  V primary() {
    const Tok k = cur();
    if (k.k == T_NUM) {
      p++; op();
      std::string d; for (char c : k.s) if (c != '_') d += c;
      if (d.size() > 3 && d.compare(d.size() - 3, 3, "f32") == 0) d.resize(d.size() - 3);
      const float f = strtof(d.c_str(), nullptr);   // decimal straight to f32, rounded once, as rustc does
      uint32_t u; memcpy(&u, &f, 4);
      char b[32]; snprintf(b, sizeof b, "Ex::Lit<0x%08xu>", u);
      return V{b, F32, 0};
    }
    if (k.k == T_INT) fail_at(k, "integer literals are not supported; write `" + k.s + ".0`");
    if (is("(")) {
      p++;
      std::vector<V> el;
      bool tuple = false;
      for (;;) {
        const Tok at = cur();
        V e = expr();
        if (e.ty == TUPLE) fail_at(at, "tuples cannot nest");
        el.push_back(e);
        if (is(",")) { p++; tuple = true; if (is(")")) { p++; break; } continue; }
        expect(")"); break;
      }
      if (!tuple) return el[0];
      std::string s = "Ex::Out<";
      for (size_t i = 0; i < el.size(); i++) s += (i ? "," : "") + f32v(el[i], k).s;
      return V{s + ">", TUPLE, (int)el.size()};
    }
    if (is("{")) return block();
    if (k.k != T_ID) fail_at(k, "");
    if (k.s == "if") return if_();
    if (keyword(k.s)) refuse_keyword(k);
    p++;
    if (is("(")) {   // a call of a free function
      if (in_list(NOT_RESTATED, sizeof(NOT_RESTATED) / sizeof(*NOT_RESTATED), k.s))
        fail_at(k, "its musl source is not restated on the device yet (DESIGN.md §2)");
      const Fn* f = nullptr;
      for (const Fn& x : FREE_FNS) if (k.s == x.name) f = &x;
      if (!f) fail_at(k, "function not supported");
      p++;
      return call(k, *f, args());
    }
    if (is("::")) fail_at(cur(), "paths are not supported");
    for (size_t i = lets.size(); i-- > 0;) {
      if (lets[i].first != k.s) continue;
      const int idx = (int)(lets.size() - 1 - i);
      return V{std::string(lets[i].second == BOOL ? "Ex::BVar<" : "Ex::Var<") + std::to_string(idx) + ">", lets[i].second, 0};
    }
    if (const Param* q = param(k.s)) {
      if (q->kind == PK_NODE) fail_at(k, "the node parameter can only be the receiver of `.set(..)`");
      if (q->kind == PK_TIME) return V{"Ex::T", F32, 0};
      if (q->kind == PK_SCALAR) return V{"Ex::In<" + std::to_string(q->index) + ">", F32, 0};
      if (is("[")) {
        p++;
        const Tok ix = cur();
        if (ix.k != T_INT) fail_at(ix, "a frame is indexed with an integer literal");
        const long v = strtol(ix.s.c_str(), nullptr, 10);
        if (v < 0 || v >= inputs) fail_at(ix, "arity mismatch: index " + ix.s + " of a frame of " + std::to_string(inputs) + " input" + (inputs == 1 ? "" : "s"));
        p++; expect("]");
        return V{"Ex::In<" + std::to_string(v) + ">", F32, 0};
      }
      if (q->kind == PK_FRAME_OR_SCALAR) return V{"Ex::In<0>", F32, 0};
      fail_at(k, "a frame parameter is used as `" + k.s + "[k]`");
    }
    int ci = -1;
    for (size_t i = 0; i < caps.size(); i++) if (caps[i] == k.s) ci = (int)i;
    if (ci < 0) { ci = (int)caps.size(); caps.push_back(k.s); }
    return V{"Ex::Cap<" + std::to_string(ci) + ">", F32, 0};
  }
  V if_() {
    const Tok k = cur(); p++; op();
    const Tok ct = cur();
    V c = boolv(expr(), ct);
    if (!is("{")) fail_at(cur(), "expected `{`");
    V a = block();
    if (!is_id("else")) fail_at(cur(), "an `if` needs an `else` (the closure must have a value)");
    p++;
    V b = is_id("if") ? if_() : (is("{") ? block() : (fail_at(cur(), "expected `{` or `if`"), V{}));
    if (a.ty != b.ty || a.n != b.n) fail_at(k, "the arms of `if` have different types");
    return V{"Ex::If<" + c.s + "," + a.s + "," + b.s + ">", a.ty, a.n};
  }
  void let_(std::vector<std::string>& vals) {   // after `let`
    if (is_id("mut")) fail_at(cur(), "mutation is not supported");
    const Tok n = cur();
    if (n.k != T_ID || keyword(n.s)) fail_at(n, "expected a name");
    p++;
    if (is(":")) { p++; skip_type(); }
    expect("=");
    const Tok at = cur();
    V v = expr();
    if (v.ty == TUPLE) fail_at(at, "a tuple can only be the closure's value");
    expect(";");
    vals.push_back(v.s);
    lets.push_back({n.s, v.ty});
  }
  V block() {
    expect("{");
    std::vector<std::string> vals;
    const size_t depth = lets.size();
    while (is_id("let")) { p++; let_(vals); }
    const Tok at = cur();
    V body = expr();
    if (is(";")) fail_at(cur(), "only `let` statements are allowed; the block ends with its value");
    expect("}");
    (void)at;
    for (size_t i = vals.size(); i-- > 0;) body.s = "Ex::Let<" + vals[i] + "," + body.s + ">";
    lets.resize(depth);
    return body;
  }
  // update's body: `x.set(Setting::kind(args)[.left() | .right() | .index(N)]*)` statements after any `let`s, in braces or alone. Every
  // argument of every statement is one value of the tuple the body evaluates to, so the lets are evaluated once per update.
  V update_body(std::vector<UpdateSet>& sets) {
    const bool braces = is("{");
    if (braces) p++;
    std::vector<std::string> vals, argv;
    auto at_end = [&]() { return braces ? is("}") : cur().k == T_END; };
    while (!at_end()) {
      if (is_id("let")) {
        if (!sets.empty()) fail_at(cur(), "a `let` after a `set` is not supported; put the `let`s first");
        p++; let_(vals); continue;
      }
      if (is_id("if")) fail_at(cur(), "a `set` inside an `if` is not supported; put the `if` inside the setting's arguments");
      const Tok r = cur();
      const Param* q = r.k == T_ID ? param(r.s) : nullptr;
      if (!q || q->kind != PK_NODE) fail_at(r, "expected `let` or a `.set(..)` of the node parameter");
      p++; expect(".");
      if (!is_id("set")) fail_at(cur(), "only `.set(..)` can be called on the node parameter");
      p++; expect("(");
      if (!is_id("Setting")) fail_at(cur(), "expected `Setting::..`");
      p++; expect("::");
      const Tok kt = cur();
      const SettingKind* sk = nullptr;
      for (const SettingKind& x : UPDATE_SETTINGS) if (kt.k == T_ID && kt.s == x.name) sk = &x;
      if (!sk) fail_at(kt, "setting not supported in an update function (center, center_q, center_q_gain, value, pan, biquad)");
      p++; expect("(");
      std::vector<V> a = args();
      if ((int)a.size() != sk->nargs)
        fail_at(kt, "takes " + std::to_string(sk->nargs) + " argument" + (sk->nargs == 1 ? "" : "s") + ", given " + std::to_string(a.size()));
      UpdateSet st{sk->kind, (int)argv.size(), sk->nargs, r.col, {}};
      for (const V& v : a) argv.push_back(v.s);
      while (is(".")) {
        p++;
        const Tok m = cur();
        if (m.k == T_ID && (m.s == "left" || m.s == "right")) { p++; expect("("); expect(")"); st.address.push_back(m.s == "left" ? 0 : 1); }
        else if (m.k == T_ID && m.s == "index") {
          p++; expect("(");
          const Tok ix = cur();
          if (ix.k != T_INT) fail_at(ix, "`.index()` takes an integer literal");
          p++; expect(")");
          st.address.push_back(strtoull(ix.s.c_str(), nullptr, 10));
        } else if (m.k == T_ID && m.s == "node") fail_at(m, "`.node()` addressing is not supported in an update function");
        else fail_at(m, "expected `.left()`, `.right()` or `.index(N)`");
        if ((int)st.address.size() > MAX_ADDRESS) fail_at(m, "an address has at most " + std::to_string(MAX_ADDRESS) + " steps");
      }
      expect(")");
      op();
      sets.push_back(std::move(st));
      if (is(";")) { p++; continue; }
      if (!at_end()) fail_at(cur(), "expected `;`");
    }
    if (sets.empty()) fail_at(cur(), "the update function sets nothing; it needs at least one `.set(..)` of the node parameter");
    if (braces) p++;
    std::string body = "Ex::Out<";
    for (size_t i = 0; i < argv.size(); i++) body += (i ? "," : "") + argv[i];
    body += ">";
    for (size_t i = vals.size(); i-- > 0;) body = "Ex::Let<" + vals[i] + "," + body + ">";
    return V{body, TUPLE, (int)argv.size()};
  }
  void skip_type() {   // a type annotation, ignored: tokens up to `,` or `|` outside brackets
    int depth = 0;
    for (;;) {
      const Tok& k = cur();
      if (k.k == T_END) fail_at(k, "");
      if (depth == 0 && (is(",") || is("|") || is("=") || is(";"))) return;
      if (is("<") || is("(") || is("[")) depth++;
      else if (is(">") || is(")") || is("]")) depth--;
      p++;
    }
  }
};

}  // namespace

std::string parse_closure(const char* text, ClosureKind kind, int inputs, int outputs, Closure& out) {
  if (!text) return "null closure text";
  const std::string src(text);
  if ((int)src.size() > CLOSURE_MAX_TEXT) return "the closure text is " + std::to_string(src.size()) + " bytes; the limit is " + std::to_string(CLOSURE_MAX_TEXT);
  try {
    Parser ps;
    ps.t = lex(src);
    ps.inputs = inputs; ps.outputs = outputs;
    if (ps.is_id("move")) ps.p++;
    std::vector<std::string> names;
    if (ps.is("||")) ps.p++;
    else {
      ps.expect("|");
      while (!ps.is("|")) {
        const Tok n = ps.cur();
        if (n.k != T_ID || Parser::keyword(n.s)) fail_at(n, "expected a parameter name");
        ps.p++;
        names.push_back(n.s);
        if (ps.is(":")) { ps.p++; ps.skip_type(); }
        if (ps.is(",")) ps.p++;
        else if (!ps.is("|")) fail_at(ps.cur(), "expected `,` or `|`");
      }
      ps.p++;
    }
    const int np = (int)names.size();
    auto arity = [&](const std::string& want) -> std::string {
      return "arity mismatch: " + want + ", the text has " + std::to_string(np) + " parameter" + (np == 1 ? "" : "s");
    };
    if (kind == CL_MAP) {
      if (np != 1) return arity("map takes one frame parameter |x|");
      ps.params.push_back({names[0], PK_FRAME, 0});
    } else if (kind == CL_SHAPE_FN || kind == CL_VAR_FN) {
      if (np != 1) return arity(kind == CL_VAR_FN ? "var_fn takes one parameter |x|" : "shape_fn takes one parameter |x|");
      ps.params.push_back({names[0], PK_SCALAR, 0});
    } else if (kind == CL_ENVELOPE) {
      if (np != 1) return arity("envelope takes one time parameter |t|");
      ps.params.push_back({names[0], PK_TIME, 0});
    } else if (kind == CL_UPDATE) {
      if (np != 3) return arity("update takes |t, dt, x|");
      ps.params.push_back({names[0], PK_SCALAR, 0}); ps.params.push_back({names[1], PK_SCALAR, 1}); ps.params.push_back({names[2], PK_NODE, 0});
    } else {
      if (np == 2 && inputs != 1) { ps.params.push_back({names[0], PK_TIME, 0}); ps.params.push_back({names[1], PK_FRAME, 0}); }
      else if (np == 2 && inputs == 1) { ps.params.push_back({names[0], PK_TIME, 0}); ps.params.push_back({names[1], PK_FRAME_OR_SCALAR, 0}); }
      else if (np == 1 + inputs) { ps.params.push_back({names[0], PK_TIME, 0}); for (int k = 0; k < inputs; k++) ps.params.push_back({names[1 + k], PK_SCALAR, k}); }
      else return arity("envelope_in takes |t, frame| or |t, x1, .., x" + std::to_string(inputs) + "| for " + std::to_string(inputs) + " input" + (inputs == 1 ? "" : "s"));
    }
    for (size_t i = 0; i < names.size(); i++)
      for (size_t j = 0; j < i; j++) if (names[i] == names[j]) return "parameter `" + names[i] + "` appears twice";
    const Tok at = ps.cur();
    if (kind == CL_UPDATE) {
      V body = ps.update_body(out.sets);
      if (ps.cur().k != T_END) fail_at(ps.cur(), "");
      out.expr = body.s;
      out.caps = ps.caps;
      return "";
    }
    V body = ps.expr();
    if (ps.cur().k != T_END) fail_at(ps.cur(), "");
    if (body.ty == BOOL) fail_at(at, "the closure's value is a bool; it must be f32 or a tuple of f32");
    const int nv = body.ty == TUPLE ? body.n : 1;
    if (nv != outputs)
      return "arity mismatch: the closure returns " + std::to_string(nv) + " value" + (nv == 1 ? "" : "s") + ", the node has " + std::to_string(outputs) + " output" + (outputs == 1 ? "" : "s");
    out.expr = body.s;
    out.caps = ps.caps;
    return "";
  } catch (const ParseError& e) {
    return e.why;
  }
}

}  // namespace host
}  // namespace fdsp
