// TEST INFRASTRUCTURE ONLY — the wrapper of ref_filter_shim.cpp around the UNMODIFIED reference class Filter, plus
// Filter::setSlope, so that mid-stream slope and frequency switches (onSlider, src/PluginProcessor.cpp:837-848) can be
// pinned.  Compiled from the reference's sources where they lie (oracle/params.mk, target `ref`).
#include "ref_filter_shim.cpp"

extern "C" void ref_filter_set_slope(void* f, int slope) { static_cast<Filter*>(f)->setSlope((FilterSlope)slope); }
