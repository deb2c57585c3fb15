# tests/native/coalesce.mk -- TEST INFRASTRUCTURE: the coalesced Send model (B200_SEND_COALESCE) and the
# b200_pair_ops tables over it.  make -C tests/native -f coalesce.mk
ROOT := ../..
all: libcoalesce_oracle.so
liboracle_pair_ops.so: oracle_pair_ops.c $(ROOT)/include/b200_endpoint.h $(ROOT)/oracle/liboracle.so
	$(MAKE) -f Makefile $@
libcoalesce_oracle.so: coalesce_oracle.c liboracle_pair_ops.so $(ROOT)/include/b200_endpoint.h $(ROOT)/oracle/liboracle.so
	gcc -O2 -g -std=gnu11 -fPIC -shared -Wall -o $@ coalesce_oracle.c -L. -loracle_pair_ops -L$(ROOT)/oracle -loracle -Wl,-rpath,'$$ORIGIN' -Wl,-rpath,'$$ORIGIN/$(ROOT)/oracle'
.PHONY: all
