# TEST INFRASTRUCTURE ONLY — the oracle of b200conv_chain_update (chain parameter changes), built by oracle/params.py:
#   make -C oracle -f params.mk all
#  libparams.so                 : plain-C restatement of onSlider's filter re-init, the per-block parameter reads and
#                                 the delay-line growth of processBlock (params_oracle.c, one translation unit with
#                                 hotswap_oracle.c, chain_oracle.c and partconv_oracle.c)
#  _ref/libreffilterswitch.so   : the UNMODIFIED src/dsp/Filter.cpp compiled where it lies under $(REF), with
#                                 ref_filter_switch_shim.cpp (adds Filter::setSlope); a no-op when $(REF) is absent
REF ?= /root/reference
CC ?= gcc
CXX ?= g++

all: libparams.so ref

libparams.so: params_oracle.c hotswap_oracle.c chain_oracle.c partconv_oracle.c
	$(CC) -O2 -std=c11 -fPIC -shared -ffp-contract=off -o $@ params_oracle.c -lm

ref:
	@if [ -d "$(REF)/src/dsp" ]; then \
	  mkdir -p _ref && \
	  $(CXX) -O2 -std=c++17 -fPIC -shared -Ijuce_min -I$(REF)/src/dsp -o _ref/libreffilterswitch.so \
	    ref_filter_switch_shim.cpp $(REF)/src/dsp/Filter.cpp && echo "built _ref/libreffilterswitch.so"; \
	else echo "reference sources absent; keeping prebuilt _ref/ (if any)"; fi

clean:
	rm -f libparams.so _ref/libreffilterswitch.so
.PHONY: all ref clean
