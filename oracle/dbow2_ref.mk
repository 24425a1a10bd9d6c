# DBoW2's L1 score compiled from the reference's own sources (TEST INFRASTRUCTURE ONLY) into oracle/_ref/libdbow2_l1.so,
# which oracle/pin_l1_score_against_dbow2.py pins tests/golden/l1_score_golden.npz against:
#     make -C oracle -f dbow2_ref.mk REF=<reference source tree>
# ScoringObject.cpp includes TemplatedVocabulary.h, which needs OpenCV; defining its include guard skips it, and the two
# -include flags supply what it would have brought in. -O3 without -march: the library may run on another host, and the
# score is additions and subtractions only, which no instruction set changes.
DB_HERE := $(dir $(abspath $(lastword $(MAKEFILE_LIST))))
REF ?= $(error set REF to the reference source tree)
DBOW2 := $(REF)/Thirdparty/DBoW2/DBoW2
DBOW2_LIB := $(DB_HERE)_ref/libdbow2_l1.so
.DEFAULT_GOAL := $(DBOW2_LIB)

$(DBOW2_LIB): $(DB_HERE)dbow2_l1_shim.cpp $(DBOW2)/ScoringObject.cpp $(DBOW2)/BowVector.cpp
	mkdir -p $(dir $@)
	g++ -O3 -std=c++11 -fPIC -ffp-contract=off -fno-fast-math -w -shared -I$(DBOW2) -D__D_T_TEMPLATED_VOCABULARY__ \
	    -include cmath -include $(DBOW2)/ScoringObject.h -o $@.$$$$.tmp $^ && mv -f $@.$$$$.tmp $@
