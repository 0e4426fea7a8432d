# ORACLE build of the source decimator (SPEC_L.md; test infrastructure): decimate.c as its own library over the parity
# build libsdoracle.so, whose SPEC I.3 tap design it calls.  Same parity flags as Makefile.
#   make -C oracle -f decimate.mk
CC      := gcc
CFLAGS  ?= -O2 -ffp-contract=off -fno-fast-math -mfma -fPIC -Wall -Wextra -std=gnu11
OUT     := _build/libsddecim.so

all: $(OUT)

$(OUT): decimate.c decimate.h sd_oracle.h _build/libsdoracle.so
	$(CC) $(CFLAGS) -shared -o $@ decimate.c -L _build -lsdoracle -Wl,-rpath,'$$ORIGIN' -lm

_build/libsdoracle.so:
	$(MAKE) -f Makefile _build/libsdoracle.so

.PHONY: all
