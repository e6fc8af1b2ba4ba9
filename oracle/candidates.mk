# CPU oracle of the per-candidate breakdown (test infrastructure only).  Carries its own copy of apo_oracle.c so that it
# loads on its own; same flags as the main oracle (no FMA contraction).
CC ?= gcc
CFLAGS = -O2 -std=c11 -fPIC -ffp-contract=off -fno-fast-math -Wall -Wextra -pthread
all: libcand_oracle.so
libcand_oracle.so: cand_oracle.c cand_oracle.h apo_oracle.c apo_oracle.h
	$(CC) $(CFLAGS) -shared -o $@ cand_oracle.c apo_oracle.c -lm -lpthread
clean:
	rm -f libcand_oracle.so
