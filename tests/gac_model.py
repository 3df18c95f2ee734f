"""A bit-serial CPU model of the two machines behind noaa_gac_decoder and dmsp_rtd_decoder, written from their documented behaviour
(include/b200dsp.h, DESIGN §9), so that the tests can check the case streams' expectations without the reference: BPSK_CCSDS_Deframer
(33270 bits, 32-bit sync, states 2 / 6 / 12) and DMSP_Deframer (150 bits, 13-bit sync, states 0 / 2 / 6). Each state's number is also its
error threshold; NOSYNC needs an exact match of the sync or its complement."""
import numpy as np

from satdump_b200 import synth


class Machine:
    def __init__(self, dmsp, backward=False):
        self.dmsp = dmsp
        if dmsp:
            self.nbits, self.width, self.sync, self.states, self.nbytes = 150, 13, synth.DMSP_ASM, (0, 2, 6), 19
        else:
            self.nbits, self.width, self.nbytes = 33270, 32, 4159
            self.sync, self.states = (synth.GAC_SYNC_BACKWARD if backward else synth.GAC_SYNC), (2, 6, 12)
        self.backward = backward
        self.mask = (1 << self.width) - 1
        self.state, self.inv, self.good, self.bad = self.states[0], 0, 0, 0
        self.shifter, self.in_frame, self.bit_of_frame, self.frame = 0, False, 0, []
        self.frames, self.done = [], []  # frames written, and the stream bit that completed each
        self.pos = 0

    def _accept(self):
        self.in_frame = True
        self.frame = [(self.sync >> (self.width - 1 - k)) & 1 for k in range(self.width)]

    def push(self, bits):
        nosync, syncing, synced = self.states
        for b in np.asarray(bits, np.uint8).tolist():
            self.shifter = ((self.shifter << 1) | b) & self.mask
            p = self.pos
            self.pos += 1
            if self.in_frame:
                self.frame.append(b ^ self.inv)
                if len(self.frame) == self.nbits:
                    self.frames.append(list(self.frame))
                    self.done.append(p)
                elif len(self.frame) == self.nbits + self.width - 1:
                    self.in_frame = False
                continue
            want = self.sync ^ (self.mask if self.inv else 0)
            if self.state == nosync:
                if self.shifter in (self.sync, self.sync ^ self.mask):
                    self.inv = int(self.shifter != self.sync)
                    self.state, self.good, self.bad = syncing, 0, 0
                    self._accept()
            elif self.state == syncing:
                if bin(self.shifter ^ want).count("1") < syncing:
                    self.bad, self.good = 0, self.good + 1
                    if self.good > 10:
                        self.state = synced
                    self._accept()
                else:
                    self.bad, self.good = self.bad + 1, 0
                    if self.bad > 2:
                        self.state = nosync
            else:
                if bin(self.shifter ^ want).count("1") < synced:
                    self._accept()
                else:
                    self.state, self.good, self.bad = nosync, 0, 0
        return self

    def output(self):
        """the frames as the decoder writes them (GAC: reversed when backward, then the PN)"""
        img = synth.frame_image(np.array(self.frames, np.uint8).reshape(-1, self.nbits), self.nbytes)
        return img if self.dmsp else synth.gac_post(img, self.backward)


def run(soft, dmsp, backward=False):
    """frames, the completion bit of each and the final state of a whole stream (hard bits soft > 0)"""
    m = Machine(dmsp, backward).push((np.asarray(soft, np.int8) > 0).astype(np.uint8))
    return dict(out=m.output(), done=np.array(m.done, np.int64), state=m.state)
