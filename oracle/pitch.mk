# oracle/pitch.mk -- TEST INFRASTRUCTURE ONLY: the reference's unmodified pitch tracker program,
# programs/pocketsphinx_pitch.c, linked against the same reference objects as _ref/libpsref.so into
# _ref/pocketsphinx_pitch (the checker of the device pitch tracker's printed lines).  Uses Makefile's
# variables and object rules; like the rest of _ref/ it is built only where $(REF) exists, and travels
# to the GPU box with the snapshot.
#
#   make -C oracle -f pitch.mk pitch

include Makefile

ifneq ($(wildcard $(REF)/programs/pocketsphinx_pitch.c),)
pitch: $(REFOUT)/pocketsphinx_pitch
else
pitch:
	@echo "oracle: $(REF) not present; keeping prebuilt $(REFOUT)/pocketsphinx_pitch if any"
endif

$(REFOUT)/pocketsphinx_pitch: $(REF)/programs/pocketsphinx_pitch.c $(REF_OBJS)
	$(CC) $(REF_CFLAGS) -o $@ $^ -lm

.PHONY: pitch
