# Builds the raw DEFLATE / zlib / gzip decoder oracle (orc_flate.c) as its own library (test infrastructure only; never
# linked into the product).  make -C oracle -f flate.mk
CC ?= gcc
CFLAGS ?= -O3 -g -fPIC -Wall -Wextra -Wno-unused-parameter -fvisibility=hidden -std=gnu11

all: liboracle_flate.so

liboracle_flate.so: orc_flate.c orc_common.h
	$(CC) $(CFLAGS) -shared -o $@ orc_flate.c

clean:
	rm -f liboracle_flate.so
