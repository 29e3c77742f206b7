# ORACLE — test infrastructure.  oracle/libsora_oracle_tx11a44.so: the legacy 802.11a transmitter at 40 and 44 Msps (tx11a_legacy44.cpp) with the
# oracle sources it uses (tables, the rate-1/2 encoder of tx11a.cpp), built apart from libsora_oracle.so.   usage: make -C oracle -f tx11a_legacy44.mk
CXX ?= g++
CXXFLAGS ?= -O2 -msse4.1 -std=c++17 -ffp-contract=off -fPIC -Wall -Wno-unused-function -pthread
SRC = tables.cpp tx11a.cpp tx11a_legacy44.cpp
HDR = ops.h tables.h tx11a.h rx11a.h viterbi.h
# linked under a temporary name and renamed, as oracle/Makefile does
libsora_oracle_tx11a44.so: $(SRC) $(HDR)
	$(CXX) $(CXXFLAGS) -shared -Wl,--no-undefined -o $@.tmp.$$$$ $(SRC) && mv -f $@.tmp.$$$$ $@
clean:
	rm -f libsora_oracle_tx11a44.so
