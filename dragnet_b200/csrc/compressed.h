/*
 * compressed.h: what the rest of a scan sees of its compressed input
 * (compressed.cu): gzip and bzip2 files queued, decoded and fed in batches.
 */
#ifndef DNG_COMPRESSED_H
#define DNG_COMPRESSED_H

struct dng_scan;
struct CzState;		/* the queue, decoder buffers and stats of a scan */

/* decode and feed the queued files, in the order they were fed; the scan's
 * error code */
int cz_flush(dng_scan *s);
/* free the state, once the scan's streams are idle */
void cz_free(CzState *cz);

#endif
