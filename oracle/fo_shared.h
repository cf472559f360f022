// ORACLE — TEST INFRASTRUCTURE ONLY (see fo_math.h). The reference's Shared controls over a real shared cell, restated from
// src/shared.rs:47-250 (Shared, Var, Timer) and src/dynamics.rs:329-520 (MeterState, Monitor): tick and process as written.
#pragma once
#include "fo_nodes.h"
#include "fo_closure.h"

#include <atomic>
#include <cstring>
#include <memory>

namespace fo {

// Shared: Arc<AtomicU32> holding an f32 bit pattern (src/shared.rs:15-81)
typedef std::shared_ptr<std::atomic<uint32_t>> Cell;
inline float cell_get(const Cell& c) { const uint32_t u = c->load(std::memory_order_relaxed); float f; memcpy(&f, &u, 4); return f; }
inline void cell_set(const Cell& c, float f) { uint32_t u; memcpy(&u, &f, 4); c->store(u, std::memory_order_relaxed); }

// ---- src/shared.rs:84-131 Var (ID 68)
struct VarShared : Node {
  Cell value;
  explicit VarShared(Cell c) : value(std::move(c)) {}
  int inputs() const override { return 0; } int outputs() const override { return 1; }
  uint64_t id() const override { return 68; }
  void tick(const float*, float* out) override { out[0] = cell_get(value); }
  void process(int size, const float*, float* out) override {
    const float sample = cell_get(value);
    for (int i = 0; i < simd_items(size) * 8; i++) out[i] = sample;
  }
  FO_CLONE(VarShared)
};

// ---- src/shared.rs:134-200 VarFn (ID 70): the closure (fo_closure.h's interpreter, one parameter |x|) of the cell's value
struct VarFn : Node {
  Cell value; int no; cl::Closure f;
  VarFn(Cell c, int o, cl::Closure fn) : value(std::move(c)), no(o), f(std::move(fn)) {}
  int inputs() const override { return 0; } int outputs() const override { return no; }
  uint64_t id() const override { return 70; }
  void tick(const float*, float* out) override { const float x = cell_get(value); f.call(&x, 0.0f, out); }
  void process(int size, const float*, float* out) override {
    const float x = cell_get(value);
    float frame[8];
    f.call(&x, 0.0f, frame);
    for (int c = 0; c < no; c++) for (int i = 0; i < simd_items(size) * 8; i++) out[c * B + i] = frame[c];
  }
  FO_CLONE(VarFn)
};

// ---- src/dynamics.rs:329-407 Meter / MeterState, :441-520 Monitor (ID 56)
struct MonitorShared : Node {
  int kind; double timescale; float smoothing = 0.0f, state = 0.0f; Cell shared;
  MonitorShared(Cell c, int k, double t) : kind(k), timescale(t), shared(std::move(c)) { set_sample_rate(DEFAULT_SR); }
  int inputs() const override { return 1; } int outputs() const override { return 1; }
  uint64_t id() const override { return 56; }
  void reset() override { state = 0.0f; }
  void set_sample_rate(double sr) override { if (kind != 0) smoothing = (float)pow(0.5, 1.0 / (timescale * sr)); }
  void meter_tick(float value) {
    if (kind == 0) state = value;
    else if (kind == 1) state = std::max(state * smoothing, std::fabs(value));
    else state = state * smoothing + (value * value) * (1.0f - smoothing);
  }
  float level() const { return kind == 2 ? std::sqrt(state) : state; }
  void tick(const float* in, float* out) override { meter_tick(in[0]); cell_set(shared, level()); out[0] = in[0]; }
  void process(int size, const float* in, float* out) override {
    if (size == 0) return;
    if (kind == 0) meter_tick(in[size - 1]);   // Meter::latest_only
    else for (int i = 0; i < size; i++) meter_tick(in[i]);
    cell_set(shared, level());
    for (int i = 0; i < simd_items(size) * 8; i++) out[i] = in[i];
  }
  FO_CLONE(MonitorShared)
};

// ---- src/shared.rs:203-250 Timer (ID 57)
struct Timer : Node {
  Cell shared; double time = 0.0, sample_duration = 1.0 / DEFAULT_SR;
  explicit Timer(Cell c) : shared(std::move(c)) { cell_set(shared, 0.0f); }
  int inputs() const override { return 0; } int outputs() const override { return 0; }
  uint64_t id() const override { return 57; }
  void reset() override { time = 0.0; cell_set(shared, 0.0f); }
  void set_sample_rate(double sr) override { sample_duration = 1.0 / sr; }
  void tick(const float*, float*) override { time += sample_duration; cell_set(shared, (float)time); }
  void process(int size, const float*, float*) override { time += (double)size * sample_duration; cell_set(shared, (float)time); }
  FO_CLONE(Timer)
};

}  // namespace fo
