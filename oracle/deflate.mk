# Builds the StatelessDeflate / gzip StatelessCompression oracle (orc_deflate.c) as its own library (test infrastructure
# only; never linked into the product).  -ffp-contract=off keeps every float32 / float64 operation rounded on its own, as
# the reference computes them on amd64.  make -C oracle -f deflate.mk
CC ?= gcc
CFLAGS ?= -O3 -g -fPIC -Wall -Wextra -Wno-unused-parameter -fvisibility=hidden -std=gnu11

all: liboracle_deflate.so

liboracle_deflate.so: orc_deflate.c orc_common.h
	$(CC) $(CFLAGS) -ffp-contract=off -shared -o $@ orc_deflate.c

clean:
	rm -f liboracle_deflate.so
