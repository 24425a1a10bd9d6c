# The tracking oracle's library (TEST INFRASTRUCTURE ONLY), with oracle/Makefile's compiler and flags:
#     make -C oracle -f track.mk          (oracle/pytrack.py runs this before loading it)
TR_HERE := $(dir $(abspath $(lastword $(MAKEFILE_LIST))))
include $(TR_HERE)Makefile
TR_LIB := $(TR_HERE)libtrack_oracle.so
.DEFAULT_GOAL := $(TR_LIB)

# written aside and renamed, so that a process loading the library never sees a half-written file
$(TR_LIB): $(TR_HERE)track_oracle.cpp
	$(CXX) $(CXXFLAGS) -fvisibility=hidden -shared -o $@.$$$$.tmp $< && mv -f $@.$$$$.tmp $@
