# The bag-of-words assembly oracle's library (TEST INFRASTRUCTURE ONLY), with oracle/Makefile's compiler and flags:
#     make -C oracle -f bow_assembly.mk          (oracle/pybow.py runs this before loading it)
BW_HERE := $(dir $(abspath $(lastword $(MAKEFILE_LIST))))
include $(BW_HERE)Makefile
BOWA_LIB := $(BW_HERE)libbow_assembly_oracle.so
.DEFAULT_GOAL := $(BOWA_LIB)

# written aside and renamed, so that a process loading the library never sees a half-written file
$(BOWA_LIB): $(BW_HERE)bow_assembly_oracle.cpp
	$(CXX) $(CXXFLAGS) -fvisibility=hidden -shared -o $@.$$$$.tmp $< && mv -f $@.$$$$.tmp $@
