# The localization oracle's library (TEST INFRASTRUCTURE ONLY), with oracle/Makefile's compiler and flags:
#     make -C oracle -f loc.mk          (oracle/pyloc.py runs this before loading it)
LO_HERE := $(dir $(abspath $(lastword $(MAKEFILE_LIST))))
include $(LO_HERE)Makefile
LO_LIB := $(LO_HERE)libloc_oracle.so
.DEFAULT_GOAL := $(LO_LIB)

# written aside and renamed, so that a process loading the library never sees a half-written file
$(LO_LIB): $(LO_HERE)loc_oracle.cpp
	$(CXX) $(CXXFLAGS) -fvisibility=hidden -shared -o $@.$$$$.tmp $< && mv -f $@.$$$$.tmp $@
