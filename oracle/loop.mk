# The loop-closure oracle's library (TEST INFRASTRUCTURE ONLY), with oracle/Makefile's compiler and flags:
#     make -C oracle -f loop.mk          (oracle/pyloop.py runs this before loading it)
LP_HERE := $(dir $(abspath $(lastword $(MAKEFILE_LIST))))
include $(LP_HERE)Makefile
LOOP_LIB := $(LP_HERE)libloop_oracle.so
.DEFAULT_GOAL := $(LOOP_LIB)

# written aside and renamed, so that a process loading the library never sees a half-written file
$(LOOP_LIB): $(LP_HERE)loop_oracle.cpp
	$(CXX) $(CXXFLAGS) -fvisibility=hidden -shared -o $@.$$$$.tmp $< && mv -f $@.$$$$.tmp $@
