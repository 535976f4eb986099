// TEST INFRASTRUCTURE ONLY — the project header src/dsp/Impulse.{h,cpp} and SVF.{h,cpp} of the reference include, for
// compiling them unmodified into oracle/_ref/librefimpulse.so against the JUCE modules they use (oracle/recalc.mk).
#pragma once
#include <juce_core/juce_core.h>
#include <juce_audio_basics/juce_audio_basics.h>
#include <juce_audio_formats/juce_audio_formats.h>
using namespace juce;
namespace BinaryData { extern const char* Hall_Quad_flac; extern const int Hall_Quad_flacSize; }
