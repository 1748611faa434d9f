# Builds the SIMT-emulated copy of the S2 best block encoders (test infrastructure only).  make -C tests/emu -f s2best.mk
CXX ?= g++
CXXFLAGS ?= -O1 -g -fPIC -std=c++17 -Wall -Wno-unused-function -Wno-unused-variable -Wno-unknown-pragmas -I.
all: libb2c_emu_s2best.so
libb2c_emu_s2best.so: simt_emu.cpp emu_s2best.cpp simt_emu.h $(wildcard ../../compress_b200/csrc/*.cuh)
	$(CXX) $(CXXFLAGS) -shared -o $@ simt_emu.cpp emu_s2best.cpp
clean:
	rm -f libb2c_emu_s2best.so
