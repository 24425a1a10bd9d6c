# The map-point oracle's library (TEST INFRASTRUCTURE ONLY), with oracle/Makefile's compiler and flags:
#     make -C oracle -f mappoint.mk          (oracle/pymappoint.py runs this before loading it)
MP_HERE := $(dir $(abspath $(lastword $(MAKEFILE_LIST))))
include $(MP_HERE)Makefile
MP_LIB := $(MP_HERE)libmappoint_oracle.so
.DEFAULT_GOAL := $(MP_LIB)

# mappoint_oracle.cpp #includes geom_oracle.cpp: one translation unit that exports only its visibility("default") entries;
# written aside and renamed, so that a process loading the library never sees a half-written file
$(MP_LIB): $(MP_HERE)mappoint_oracle.cpp $(MP_HERE)geom_oracle.cpp
	$(CXX) $(CXXFLAGS) -fvisibility=hidden -shared -o $@.$$$$.tmp $< -lpthread && mv -f $@.$$$$.tmp $@
