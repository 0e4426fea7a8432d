# ORACLE build of the FAC tab (SPEC_FC.md; test infrastructure): fac.c with the SPEC transforms of fft_spec.c as its
# own library.  Same parity flags as Makefile.
#   make -C oracle -f fac.mk
CC      := gcc
CFLAGS  ?= -O2 -ffp-contract=off -fno-fast-math -mfma -fPIC -fopenmp -Wall -Wextra -std=gnu11
OUT     := _build/libsdfac.so

all: $(OUT)

$(OUT): fac.c fac.h fft_spec.c fft_fast.c sd_oracle.h
	mkdir -p _build
	$(CC) $(CFLAGS) -shared -o $@ fac.c fft_spec.c fft_fast.c -lm

.PHONY: all
