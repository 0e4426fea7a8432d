# ORACLE build of channel tracking (SPEC_KT.md; test infrastructure): chtrack.c as its own library.  Same parity
# flags as Makefile.
#   make -C oracle -f chtrack.mk
CC      := gcc
CFLAGS  ?= -O2 -ffp-contract=off -fno-fast-math -mfma -fPIC -Wall -Wextra -std=gnu11
OUT     := _build/libsdchtrack.so

all: $(OUT)

$(OUT): chtrack.c chtrack.h sd_oracle.h
	mkdir -p _build
	$(CC) $(CFLAGS) -shared -o $@ chtrack.c

.PHONY: all
