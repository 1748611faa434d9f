# Builds the LZ4 / LZ4s converter oracle (orc_lz4.c) as its own library (test infrastructure only; never linked into the
# product).  make -C oracle -f lz4.mk
CC ?= gcc
CFLAGS ?= -O3 -g -fPIC -Wall -Wextra -Wno-unused-parameter -fvisibility=hidden -std=gnu11

all: liboracle_lz4.so

liboracle_lz4.so: orc_lz4.c orc_common.h
	$(CC) $(CFLAGS) -shared -o $@ orc_lz4.c

clean:
	rm -f liboracle_lz4.so
