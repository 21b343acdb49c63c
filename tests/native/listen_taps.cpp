/*
 * tests/native/listen_taps.cpp -- TEST-ONLY host build of the lane machine with the staged-tap check compiled in
 * (nfc_core.h NFCB200_CHECK_TAPS): every staged ring tap the machine uses is compared with a direct read of the ring.
 * tests/test_listen_staging.py builds it with the flags of host_sim.cpp and reads the counts through hostsim_taps().
 */
#define NFCB200_CHECK_TAPS 1
#include "host_sim.cpp"

extern "C" {

/* out[0] staged taps used, out[1] those that differed from the ring, out[2 + kind] used taps by stage kind (Machine::KIND_*) */
void hostsim_taps(unsigned long long *out)
{
   out[0] = nfcb200_taps_used;
   out[1] = nfcb200_taps_differ;
   for (int k = 0; k < 8; k++)
      out[2 + k] = nfcb200_taps_kind[k];
}

/* stage kinds of the locked NFC-A decoders at 106 kbps (rate 0) */
int hostsim_kind_poll106(void)
{
   return (int) Machine<1, Sink, 2>::KIND_POLL;
}

int hostsim_kind_listen106(void)
{
   return (int) Machine<1, Sink, 2>::KIND_LISTEN_ASK;
}

void hostsim_taps_clear(void)
{
   nfcb200_taps_used = nfcb200_taps_differ = 0;
   for (int k = 0; k < 8; k++)
      nfcb200_taps_kind[k] = 0;
}

}
