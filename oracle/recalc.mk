# TEST INFRASTRUCTURE ONLY — the checkers of the IR recalculation (b200conv_ir_recalc), built by oracle/recalc.py:
#   make -C oracle -f recalc.mk all [REF=...]
#  librecalc.so           : plain-C restatement of Impulse::recalcImpulse (recalc_oracle.c, on top of chain_oracle.c and
#                           partconv_oracle.c)
#  _ref/librefimpulse.so  : the UNMODIFIED src/dsp/Impulse.cpp + SVF.cpp, libs/FFTConvolver/AudioFFT.cpp and the JUCE
#                           modules juce_core, juce_audio_basics, juce_audio_formats, compiled where they lie under $(REF)
#                           (never copied into this repo; objects in _ref/) against juce_impulse/JuceHeader.h, plus
#                           ref_impulse_shim.cpp.
# `make ref` is a no-op (keeps a prebuilt _ref/) when $(REF) does not exist (GPU box).
REF ?= /root/reference
REFLIB := $(REF)/libs/FFTConvolver
JUCE := $(REF)/libs/JUCE/modules
CC ?= gcc
CXX ?= g++

all: librecalc.so ref

librecalc.so: recalc_oracle.c chain_oracle.c partconv_oracle.c
	$(CC) -O2 -std=c11 -fPIC -shared -ffp-contract=off -o $@ recalc_oracle.c chain_oracle.c partconv_oracle.c -lm

ref:
	@if [ -f "$(REF)/src/dsp/Impulse.cpp" ] && [ -d "$(JUCE)" ]; then $(MAKE) --no-print-directory -f recalc.mk _ref/librefimpulse.so; \
	else echo "reference sources absent; librefimpulse.so not rebuilt"; fi

# JUCE_USE_CURL=0: juce_core's web-input stream is not needed and its curl headers need not be installed
JUCE_FLAGS := -DJUCE_GLOBAL_MODULE_SETTINGS_INCLUDED=1 -DJUCE_STANDALONE_APPLICATION=0 -DJUCE_USE_CURL=0 \
  -DJUCE_MODULE_AVAILABLE_juce_core=1 -DJUCE_MODULE_AVAILABLE_juce_audio_basics=1 -DJUCE_MODULE_AVAILABLE_juce_audio_formats=1
IMP_CXX := $(CXX) -O2 -std=c++17 -fPIC -w $(JUCE_FLAGS) -I$(JUCE) -Ijuce_impulse -I$(REF)/src/dsp -I$(REFLIB)
IMP_OBJS := _ref/juce_core.o _ref/juce_core_CompilationTime.o _ref/juce_audio_basics.o _ref/juce_audio_formats.o \
  _ref/Impulse.o _ref/SVF.o _ref/AudioFFT.o _ref/ref_impulse_shim.o

_ref/juce_core.o:
	@mkdir -p _ref && $(IMP_CXX) -c $(JUCE)/juce_core/juce_core.cpp -o $@
_ref/juce_core_CompilationTime.o:
	@mkdir -p _ref && $(IMP_CXX) -c $(JUCE)/juce_core/juce_core_CompilationTime.cpp -o $@
_ref/juce_audio_basics.o:
	@mkdir -p _ref && $(IMP_CXX) -c $(JUCE)/juce_audio_basics/juce_audio_basics.cpp -o $@
_ref/juce_audio_formats.o:
	@mkdir -p _ref && $(IMP_CXX) -c $(JUCE)/juce_audio_formats/juce_audio_formats.cpp -o $@
_ref/Impulse.o: juce_impulse/JuceHeader.h
	@mkdir -p _ref && $(IMP_CXX) -c $(REF)/src/dsp/Impulse.cpp -o $@
_ref/SVF.o: juce_impulse/JuceHeader.h
	@mkdir -p _ref && $(IMP_CXX) -c $(REF)/src/dsp/SVF.cpp -o $@
_ref/AudioFFT.o:
	@mkdir -p _ref && $(IMP_CXX) -c $(REFLIB)/AudioFFT.cpp -o $@
_ref/ref_impulse_shim.o: ref_impulse_shim.cpp juce_impulse/JuceHeader.h
	@mkdir -p _ref && $(IMP_CXX) -c ref_impulse_shim.cpp -o $@
_ref/librefimpulse.so: $(IMP_OBJS)
	$(CXX) -shared -o $@ $(IMP_OBJS) -lpthread -ldl -lrt && echo "built _ref/librefimpulse.so"

clean:
	rm -f librecalc.so _ref/librefimpulse.so $(IMP_OBJS)
.PHONY: all ref clean
