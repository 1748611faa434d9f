# Builds the HuffmanOnly / NoCompression oracle (orc_flate_nolz.c, which compiles orc_deflate.c's bit writer into the same
# unit) as its own library (test infrastructure only; never linked into the product).  -ffp-contract=off as for
# deflate.mk.
# make -C oracle -f flate_nolz.mk
CC ?= gcc
CFLAGS ?= -O3 -g -fPIC -Wall -Wextra -Wno-unused-parameter -fvisibility=hidden -std=gnu11

all: liboracle_flate_nolz.so

liboracle_flate_nolz.so: orc_flate_nolz.c orc_deflate.c orc_common.h
	$(CC) $(CFLAGS) -ffp-contract=off -shared -o $@ orc_flate_nolz.c

clean:
	rm -f liboracle_flate_nolz.so
