# oracle/inertialization.mk -- builds the inertialization oracles with the flags of oracle/blend.mk. TEST INFRASTRUCTURE ONLY.
#   liboracle_inertialization.so            the capture and the apply restated in C (inertialization_oracle.c over acl_oracle.c)
#   _ref/libaclref_inertialization.so       the same built from the unmodified reference's rtm (ref_inertialization.cpp), only where the
#                                           reference tree exists
ACL_REF ?= /root/reference
CC      ?= gcc
CXX     ?= g++
HERE    := $(dir $(abspath $(lastword $(MAKEFILE_LIST))))
PORT_FLAGS := -std=c11 -O2 -msse4.1 -ffp-contract=off -fno-fast-math -fPIC -shared -Wall -Wextra
REF_FLAGS  := -std=c++14 -O2 -msse4.1 -ffp-contract=off -fno-fast-math -fPIC -shared -pthread \
              -static-libstdc++ -static-libgcc \
              -I$(ACL_REF)/includes -I$(ACL_REF)/external/rtm/includes

all: port ref

port: $(HERE)liboracle_inertialization.so
$(HERE)liboracle_inertialization.so: $(HERE)inertialization_oracle.c $(HERE)acl_oracle.c $(HERE)acl_oracle.h
	$(CC) $(PORT_FLAGS) -o $@ $(HERE)inertialization_oracle.c -lm

ifneq ($(wildcard $(ACL_REF)/includes/acl/version.h),)
ref: $(HERE)_ref/libaclref_inertialization.so
$(HERE)_ref/libaclref_inertialization.so: $(HERE)ref_inertialization.cpp
	mkdir -p $(HERE)_ref
	$(CXX) $(REF_FLAGS) -o $@ $(HERE)ref_inertialization.cpp
else
ref:
	@echo "reference tree $(ACL_REF) not present: keeping the prebuilt oracle/_ref/libaclref_inertialization.so (if any)"
endif

.PHONY: all port ref
