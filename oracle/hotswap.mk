# TEST INFRASTRUCTURE ONLY — the oracle of the IR hot swap inside the device chain (b200conv_chain_swap), built by
# oracle/hotswap.py:
#   make -C oracle -f hotswap.mk all
#  libhotswap.so : plain-C restatement of the warmer / warm-up / crossfade / swap of processBlock (hotswap_oracle.c,
#                  one translation unit with chain_oracle.c and partconv_oracle.c)
CC ?= gcc

all: libhotswap.so

libhotswap.so: hotswap_oracle.c chain_oracle.c partconv_oracle.c
	$(CC) -O2 -std=c11 -fPIC -shared -ffp-contract=off -o $@ hotswap_oracle.c -lm

clean:
	rm -f libhotswap.so
.PHONY: all clean
