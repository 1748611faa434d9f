# Builds the S2 oracle with the "best" block encoders (orc_s2best.c, which compiles in orc_s2.c) as its own library (test
# infrastructure only; never linked into the product).  make -C oracle -f s2best.mk
CC ?= gcc
CFLAGS ?= -O3 -g -fPIC -Wall -Wextra -Wno-unused-parameter -fvisibility=hidden -std=gnu11

all: liboracle_s2best.so

liboracle_s2best.so: orc_s2best.c orc_s2.c orc_common.h
	$(CC) $(CFLAGS) -shared -o $@ orc_s2best.c

clean:
	rm -f liboracle_s2best.so
