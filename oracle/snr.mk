# ORACLE build of the inspector's SNR meter (SPEC_SN.md; test infrastructure): snr.c with the SPEC Y.7 step of tasks.c
# and what tasks.c links against, as its own library.  Same parity flags as Makefile.
#   make -C oracle -f snr.mk
CC      := gcc
CFLAGS  ?= -O2 -ffp-contract=off -fno-fast-math -mfma -fPIC -fopenmp -Wall -Wextra -std=gnu11
OUT     := _build/libsdsnr.so
SRCS    := snr.c tasks.c math.c fft.c fft_spec.c fft_fast.c dsp.c

all: $(OUT)

$(OUT): $(SRCS) snr.h sd_oracle.h
	mkdir -p _build
	$(CC) $(CFLAGS) -shared -o $@ $(SRCS) -lm

.PHONY: all
