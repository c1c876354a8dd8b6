# Builds the validation oracle (test infrastructure: validation.cc) next to liboracle.so and linked to it.
# make -C oracle -f validation.mk   (after `make -C oracle`)
CXX ?= g++
CXXFLAGS ?= -O2 -std=c++17 -fPIC -Wall -Wextra -Wno-unused-parameter
OUT := _build

all: $(OUT)/libvalidation_oracle.so

$(OUT)/libvalidation_oracle.so: validation.cc validation.h oracle.h requirements.h ../karpenter-core_b200/host/model.h $(OUT)/liboracle.so
	$(CXX) $(CXXFLAGS) -shared -o $@ validation.cc -L$(OUT) -loracle -Wl,-rpath,'$$ORIGIN'

$(OUT)/liboracle.so:
	$(MAKE) -f Makefile
