# ORACLE build of the power inspector (SPEC_PW.md; test infrastructure): power.c as its own library.  Same parity
# flags as Makefile.
#   make -C oracle -f power.mk
CC      := gcc
CFLAGS  ?= -O2 -ffp-contract=off -fno-fast-math -mfma -fPIC -Wall -Wextra -std=gnu11
OUT     := _build/libsdpower.so

all: $(OUT)

$(OUT): power.c power.h sd_oracle.h
	mkdir -p _build
	$(CC) $(CFLAGS) -shared -o $@ power.c

.PHONY: all
