# ORACLE build of the inspector's Analog TV tab (SPEC_TI.md; test infrastructure): tvinsp.c with the TV processor of
# tvproc.c and what it links against, as its own library.  Same parity flags as Makefile.
#   make -C oracle -f tvinsp.mk
CC      := gcc
CFLAGS  ?= -O2 -ffp-contract=off -fno-fast-math -mfma -fPIC -fopenmp -Wall -Wextra -std=gnu11
OUT     := _build/libsdtvinsp.so
SRCS    := tvinsp.c tvproc.c math.c

all: $(OUT)

$(OUT): $(SRCS) tvinsp.h sd_oracle.h
	mkdir -p _build
	$(CC) $(CFLAGS) -shared -o $@ $(SRCS) -lm

.PHONY: all
