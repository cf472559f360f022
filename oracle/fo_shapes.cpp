// ORACLE — TEST INFRASTRUCTURE ONLY (see fo_math.h). C ABI of the shapes of fo_shapes.h, built as a library of its own
// (oracle/_build/libfundsp_oracle_shapes.so, by tests/oracle_shapes.py). Its nodes are fo::Node objects like those of
// libfundsp_oracle.so, compiled from the same headers with the same flags, so the combinators there take them as children.
#include "fo_shapes.h"

using namespace fo;

#define API extern "C" __attribute__((visibility("default")))

API float fo_atanf(float x) { return m::atanf_(x); }
API float fo_wide_atanf(float x) { return wide_atanf(x); }
// kind 0..6 as Shaper; null for any other kind
API Node* fo_shaper_x(int kind, float p0, float p1) { return (kind < 0 || kind > 6) ? nullptr : new XShaper(XShape(kind, p0, p1)); }
API Node* fo_shaper_adaptive(double timescale, int inner, float p0, float p1) {
  return (inner < 0 || inner > 6) ? nullptr : new XShaper(XShape::make_adaptive((float)timescale, inner, p0, p1));
}
API Node* fo_nl_biquad_x(int fb, int mode, int kind, float p0, float p1, int inputs, float center, float q, float gain) {
  return (kind < 0 || kind > 6) ? nullptr : new XNlBiquad(fb != 0, mode, XShape(kind, p0, p1), inputs, center, q, gain);
}
API Node* fo_nl_biquad_adaptive(int fb, int mode, double timescale, int inner, float p0, float p1, int inputs, float center, float q, float gain) {
  return (inner < 0 || inner > 6) ? nullptr : new XNlBiquad(fb != 0, mode, XShape::make_adaptive((float)timescale, inner, p0, p1), inputs, center, q, gain);
}
