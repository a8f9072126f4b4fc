# TEST INFRASTRUCTURE ONLY.  Builds oracle/_ref/{qauto,lsd,pview,plambda}: the four tools of the weight maps of
# algo == 'mgm_multi_lsd' (s2p/block_matching.py:199-217), compiled where they lie (never copied into this repo).
# c/qauto.c and c/pview.c get the flags and the PFM-only iio_c.o that oracle/Makefile gives `plambda`;
# 3rdparty/lsd/{lsd.c,lsd_cmd.c} get the flags of 3rdparty/lsd/Makefile (-O3), as the reference's makefile:38-40 builds it.
# __graft_entry__.build() runs it next to oracle/Makefile:  make -C oracle -f lsd.mk lsd

include Makefile

LREF ?= /root/reference/3rdparty/lsd

.PHONY: lsd
ifneq ($(and $(wildcard $(CREF)/qauto.c),$(wildcard $(LREF)/lsd.c)),)
lsd: $(OUT)/qauto $(OUT)/lsd $(OUT)/pview $(OUT)/plambda
else
lsd:
	@echo "oracle: $(CREF) or $(LREF) absent -- using prebuilt $(OUT)/qauto, lsd and pview if present"
endif

$(OUT)/qauto: $(CREF)/qauto.c $(OUT)/iio_c.o | $(OUT)
	$(CC) $(CFLAGS) -std=gnu99 -w -I$(CREF) -o $@ $^ -lm
$(OUT)/pview: $(CREF)/pview.c $(OUT)/iio_c.o | $(OUT)
	$(CC) $(CFLAGS) -std=gnu99 -w -I$(CREF) -o $@ $^ -lm
$(OUT)/lsd: $(LREF)/lsd_cmd.c $(LREF)/lsd.c $(LREF)/lsd.h | $(OUT)
	$(CC) -O3 -w -o $@ $(LREF)/lsd_cmd.c $(LREF)/lsd.c -lm
