# oracle/feature_search.mk -- builds the motion matching oracle with the flags of oracle/Makefile. TEST INFRASTRUCTURE ONLY.
#   liboracle_feature_search.so   the pack and the search restated on the CPU (feature_search_oracle.c over acl_oracle.c); fmaf is C's
#                                 correctly rounded fused multiply add
CC      ?= gcc
HERE    := $(dir $(abspath $(lastword $(MAKEFILE_LIST))))
PORT_FLAGS := -std=c11 -O2 -msse4.1 -ffp-contract=off -fno-fast-math -fPIC -shared -Wall -Wextra

all: port

port: $(HERE)liboracle_feature_search.so
$(HERE)liboracle_feature_search.so: $(HERE)feature_search_oracle.c $(HERE)acl_oracle.c $(HERE)acl_oracle.h
	$(CC) $(PORT_FLAGS) -o $@ $(HERE)feature_search_oracle.c -lm

.PHONY: all port
